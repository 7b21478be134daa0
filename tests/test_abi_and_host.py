"""CPU: the C-ABI library loads and exports every symbol the header declares (no compute calls
without a GPU), and the host-side logic of the drop-in (constructor, state dict, plan, sharding)."""
import os
import re

import pytest
import torch

from helpers import build_dropin
from raindrop_b200 import functional as RF
from raindrop_b200 import lib as L
from raindrop_b200.synth import make_batch, model_config, used_param_keys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ensure_built():
    if not os.path.isfile(L.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()


def test_library_exports_every_declared_symbol():
    _ensure_built()
    header = open(os.path.join(ROOT, "include", "raindrop_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    declared = set(re.findall(r"\b(rd_[a-z0-9_]+)\s*\(", header))
    assert declared == set(L.SIGNATURES), declared ^ set(L.SIGNATURES)
    lib = L.load()
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.rd_abi_version() == L.ABI_VERSION


def test_struct_layout_matches_header_sizes():
    import ctypes as C
    assert C.sizeof(L.RdDims) == 4 * 10 + 4 * 2 + 4 * 8 + 4 * 3
    assert C.sizeof(L.RdParams) == 8 * 11 + 8 * 12 * L.RD_MAX_LAYERS
    assert C.sizeof(L.RdGrads) == 8 * 10 + 8 * 12 * L.RD_MAX_LAYERS


def test_workspace_queries_are_pure_host_code():
    _ensure_built()
    import ctypes as C
    lib = L.load()
    plan = RF.Plan(34, 4, 2, 272, 2, 6, 2, 60, 0.2, True)
    d = plan.dims(128, True)
    ws, sc = lib.rd_workspace_bytes(C.byref(d)), lib.rd_backward_scratch_bytes(C.byref(d))
    assert ws > 0 and sc > 0 and ws % 256 == 0
    n = C.c_int64(0)
    off = lib.rd_workspace_offset(C.byref(d), L.WS_ENC_IN, C.byref(n))
    assert off > 0 and n.value == 60 * 128 * 152
    d.nhead = 7          # 152 % 7 != 0 -> rejected with a message, not a crash
    assert lib.rd_workspace_bytes(C.byref(d)) == 0
    assert b"divisible" in lib.rd_last_error_string()


# (N, d_ob, nhead, nhid, nlayers, d_static, T, B, training): P19, PAM, a model with D, nhid and Df not multiples of 4
@pytest.mark.parametrize("dims", [(34, 4, 2, 272, 2, 6, 60, 128, True), (17, 4, 2, 136, 2, 0, 600, 3, False),
                                  (10, 1, 2, 37, 3, 2, 130, 5, True), (8, 2, 8, 64, 8, 0, 48, 1, True)])
def test_workspace_views_are_disjoint_and_sized(dims):
    """Every named workspace view (rd_ws_buffer, the per-layer FFN activations included) lies inside the workspace, has
    its documented size, and overlaps no other view; RD_WS_FFN + nlayers and a negative id are rejected."""
    _ensure_built()
    import ctypes as C
    lib = L.load()
    N, d_ob, H, nhid, nl, ds, T, B, training = dims
    d = RF.Plan(N, d_ob, H, nhid, nl, ds, 2, T, 0.2, ds > 0).dims(B, training)
    total = lib.rd_workspace_bytes(C.byref(d))
    D = N * d_ob + 16
    Df = D + (N if ds > 0 else 0)
    want = {L.WS_X0: B * N * T * d_ob, L.WS_H1: B * N * T * d_ob, L.WS_ENC_IN: T * B * D, L.WS_ENC_OUT: T * B * D,
            L.WS_FEAT: B * Df, L.WS_RNG: 4, L.WS_HEAD_HIDDEN: B * Df}
    want.update({L.WS_FFN + l: T * B * nhid for l in range(nl)})
    spans = []
    for which, n_want in want.items():
        n = C.c_int64(0)
        off = lib.rd_workspace_offset(C.byref(d), which, C.byref(n))
        assert n.value == n_want, (which, n.value, n_want)
        assert off >= 0 and off % 256 == 0 and off + 4 * n.value <= total, (which, off, total)
        spans.append((off, off + 4 * n.value, which))
    spans.sort()
    for (a0, a1, wa), (b0, b1, wb) in zip(spans, spans[1:]):
        assert a1 <= b0, (wa, wb)
    for bad in (L.WS_FFN + nl, -1):
        assert lib.rd_workspace_offset(C.byref(d), bad, None) == -1
        assert b"unknown buffer" in lib.rd_last_error_string()


@pytest.mark.parametrize("name", ["P19", "PAM", "TINY"])
def test_dropin_state_dict_contract(name):
    """Same keys/shapes as the reference (via the oracle, which is key-identical to it), R_u absent."""
    from oracle.raindrop_oracle import build_oracle_model
    cfg = model_config(name)
    model = build_dropin(cfg, 3, device="cpu")
    sd, ref = model.state_dict(), build_oracle_model(cfg).state_dict()
    assert list(sd.keys()) == list(ref.keys())
    assert all(sd[k].shape == ref[k].shape for k in sd)
    assert "R_u" not in sd and not isinstance(model.R_u, torch.nn.Parameter)
    assert [k for k, _ in model._plan.fields] == [k for k in _order(used_param_keys(cfg), model)]
    assert len(sd) == (64 if cfg["static"] else 62)


def _order(keys, model):
    field_keys = [k for k, _ in model._plan.fields]
    assert sorted(field_keys) == sorted(keys)
    return field_keys


def test_seeded_construction_matches_reference_init():
    """torch.manual_seed(1) + construct draws the same initial weights as the reference does
    (same module creation order), so a seeded run of code/Raindrop.py starts from the same point."""
    from oracle.raindrop_oracle import build_oracle_model
    from raindrop_b200.models_rd import Raindrop_v2
    cfg = model_config("TINY")
    torch.manual_seed(1)
    m = Raindrop_v2(cfg["d_inp"], cfg["d_model"], cfg["nhead"], cfg["nhid"], cfg["nlayers"], cfg["dropout"],
                    cfg["max_len"], cfg["d_static"], cfg["MAX"], 0.5, "mean", cfg["n_classes"],
                    torch.ones(cfg["d_inp"], cfg["d_inp"]))
    o = build_oracle_model(cfg, seed=1)
    for (k1, a), (k2, b) in zip(m.state_dict().items(), o.state_dict().items()):
        assert k1 == k2 and torch.equal(a, b), k1
    assert torch.equal(m.R_u, o.R_u)


def test_forward_fails_loudly_without_cuda():
    if torch.cuda.is_available():
        pytest.skip("CPU-only check")
    cfg = model_config("TINY")
    model = build_dropin(cfg, 3, device="cpu")
    batch = make_batch(cfg, 2, seed=0)
    with pytest.raises(L.RaindropB200Error):
        model.forward(batch["src"], batch["static"], batch["times"], batch["lengths"])


def test_unbuilt_configurations_raise():
    from raindrop_b200.models_rd import Observation_progation, Raindrop_v2
    with pytest.raises(NotImplementedError):
        Raindrop_v2(5, 20, 2, 40, 2, 0.2, 12, 3, 100, 0.5, "mean", 2, torch.ones(5, 5), sensor_wise_mask=True)
    with pytest.raises(NotImplementedError):
        Observation_progation(20, 20, n_nodes=5, ob_dim=4, heads=2)


def test_synthetic_batch_conventions():
    cfg = model_config("P19")
    b = make_batch(cfg, 16, seed=3)
    T, N = cfg["max_len"], cfg["d_inp"]
    assert b["src"].shape == (T, 16, 2 * N) and b["times"].shape == (T, 16)
    assert torch.equal(b["lengths"], (b["times"] > 0).sum(0))
    m = b["src"][:, :, N:]
    assert set(m.unique().tolist()) <= {0.0, 1.0}
    assert torch.all(b["src"][:, :, :N][m == 0] == 0)                     # unobserved values are zero
    pad = torch.arange(T)[:, None] >= b["lengths"][None, :]
    assert torch.all(b["src"][pad] == 0)                                   # padding rows are all zero
    t0 = make_batch(cfg, 4, seed=3, first_time_zero=True)
    assert torch.all(t0["times"][0] == 0) and torch.all(t0["lengths"] == (t0["times"] > 0).sum(0))
    z = make_batch(cfg, 4, seed=3, zero_sensors=10)
    assert int((z["src"][:, 0, :N].abs().sum(0) == 0).sum()) >= 10
    again = make_batch(cfg, 16, seed=3)
    assert all(torch.equal(b[k], again[k]) for k in ("src", "times", "lengths", "y", "static"))


def test_shard_slices_partition_the_batch():
    from raindrop_b200.train import shard_slice
    for n in (1, 7, 128, 3880):
        for world in (1, 2, 3, 8):
            parts = [shard_slice(n, r, world) for r in range(world)]
            assert parts[0].start == 0 and parts[-1].stop == n
            assert all(a.stop == b.start for a, b in zip(parts, parts[1:]))
            sizes = [p.stop - p.start for p in parts]
            assert max(sizes) - min(sizes) <= 1


def test_root_module_is_the_drop_in():
    """`from models_rd import *` (code/Raindrop.py:19) with this repository's root on sys.path."""
    import importlib
    import sys
    sys.modules.pop("models_rd", None)
    mod = importlib.import_module("models_rd")
    assert mod.__file__.startswith(ROOT)
    ns = {}
    exec("from models_rd import *", ns)
    for name in ("Raindrop_v2", "Raindrop", "PositionalEncodingTF", "Observation_progation", "TransformerConv"):
        assert name in ns, name
    import inspect
    sig = inspect.signature(ns["Raindrop_v2"].__init__)
    assert list(sig.parameters)[1:] == ["d_inp", "d_model", "nhead", "nhid", "nlayers", "dropout", "max_len", "d_static",
                                        "MAX", "perc", "aggreg", "n_classes", "global_structure", "sensor_wise_mask",
                                        "static"]          # code/models_rd.py:208-209
    assert list(inspect.signature(ns["Raindrop_v2"].forward).parameters)[1:] == ["src", "static", "times", "lengths"]


def test_launcher_beats_a_competing_models_rd(tmp_path):
    """`python -m raindrop_b200.launch code/Raindrop.py` must import THIS implementation even though the script's
    own directory holds a competing models_rd.py (sys.path[0] precedes PYTHONPATH) -- ADVICE r1."""
    import subprocess
    import sys
    code = tmp_path / "code"
    code.mkdir()
    (code / "models_rd.py").write_text("WHO = 'reference'\n")
    (code / "utils_x.py").write_text("HELPER = 41\n")
    (code / "script.py").write_text(
        "import os, sys\nfrom models_rd import *\nimport models_rd, utils_x\n"
        "print('MODULE', os.path.abspath(models_rd.__file__))\nprint('HAS', 'Raindrop_v2' in globals(), utils_x.HELPER + 1)\n"
        "print('CWD', os.getcwd())\nprint('ARGV', sys.argv[1:])\n")
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "raindrop_b200.launch", str(code / "script.py"), "--dataset", "P19"],
                       capture_output=True, text=True, env=env, cwd=str(tmp_path), timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    out = dict(ln.split(" ", 1) for ln in r.stdout.strip().splitlines() if " " in ln)
    assert out["MODULE"] == os.path.join(ROOT, "raindrop_b200", "models_rd.py"), out
    assert out["HAS"] == "True 42" and out["CWD"] == str(code) and out["ARGV"] == "['--dataset', 'P19']", out
    # and the naive recipe indeed picks the competing file (the bug the launcher exists for)
    r2 = subprocess.run([sys.executable, str(code / "script.py")], capture_output=True, text=True, env=env, timeout=300)
    assert "MODULE " + str(code / "models_rd.py") in r2.stdout or r2.returncode != 0
