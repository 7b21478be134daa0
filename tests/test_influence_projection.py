"""TracIn-RP (raindrop_b200.influence.project / tracin_sketch): random projections of the gradient rows."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from helpers import build_dropin, to_dev
from oracle.projection_signs import project_rows, projection_matrix
from raindrop_b200 import influence as IF
from raindrop_b200 import lib as L
from raindrop_b200 import privacy as PV
from raindrop_b200.synth import make_batch, model_config

EXACT = 2
HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "raindrop_b200.h")


def _cpu_model(name="TINY"):
    cfg = model_config(name, dropout=0.0)
    return cfg, build_dropin(cfg, 21, device="cpu")


def _qt(d, y=True):
    return dict(src=d["src"], static=d["static"], times=d["times"], lengths=d["lengths"], y=d["y"] if y else None)


def _sketch(**kw):
    base = dict(features=torch.zeros(1, 3, 128), lrs=(1.0,), dim=128, seed=3, fields=None,
                layout=(("a", (2, 3)), ("b", (4,))), fingerprints=("f0",))
    base.update(kw)
    return IF.GradientSketch(**base)


# ---- host ------------------------------------------------------------------------------------------------------------------
def test_signs_are_balanced_and_a_function_of_seed_column_and_dimension():
    big = projection_matrix(400, 384, seed=11, col0=100)
    assert big.shape == (400, 384) and set(np.unique(big).tolist()) == {-1.0, 1.0}
    assert abs(big.mean()) < 0.02 and np.all(np.abs(big.mean(axis=0)) < 0.3)
    np.testing.assert_array_equal(projection_matrix(50, 128, seed=11, col0=230), big[130:180, :128])
    np.testing.assert_array_equal(projection_matrix(3, 384, seed=11, col0=499)[0], big[399])
    np.testing.assert_array_equal(projection_matrix(1, 256, seed=11, col0=101)[0], big[1, :256])
    assert (projection_matrix(400, 384, seed=12, col0=100) != big).mean() > 0.4
    far = projection_matrix(64, 128, seed=2 ** 40 + 3, col0=2 ** 33)
    assert abs(far.mean()) < 0.05
    # columns apart from each other and dims apart from each other are uncorrelated at this size
    assert np.abs(big.T @ big / 400 - np.eye(384)).max() < 0.3


def test_project_rows_restates_segment_sums():
    rng = np.random.default_rng(1)
    G = rng.normal(size=(3, 300))
    full = project_rows(G, 128, 5)
    split = project_rows(G, 128, 5, [0, 100, 204], [100, 104, 96])
    np.testing.assert_allclose(split, full, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(full, G @ projection_matrix(300, 128, 5) / math.sqrt(128), rtol=1e-12)


def test_argument_errors_raise_on_the_host():
    cfg, m = _cpu_model()
    m.eval()
    b = make_batch(cfg, 3, seed=1)
    q = _qt(b)
    for dim in (0, 100, 64, 4000, 32768 + 128, 2.5, True):
        with pytest.raises(ValueError):
            IF.project(m, q, dim=dim)
    for seed in (-1, 2 ** 64, 1.5):
        with pytest.raises(ValueError):
            IF.project(m, q, seed=seed)
    with pytest.raises(ValueError):
        IF.project(m, q, internal_batch_size=0)
    with pytest.raises(ValueError):
        IF.project(m, q, fields=["no.such.field"])
    m.train()
    with pytest.raises(ValueError):
        IF.project(m, q)


@pytest.mark.parametrize("field,value", [("dim", 256), ("seed", 4), ("fields", ("a",)), ("layout", (("a", (2, 3)),)),
                                         ("lrs", (0.5,)), ("fingerprints", ("f1",))])
def test_mismatched_sketches_are_refused_on_the_host(field, value):
    kw = {field: value}
    if field == "dim":
        kw["features"] = torch.zeros(1, 3, 256)
    with pytest.raises(ValueError):
        IF.tracin_sketch(_sketch(), _sketch(**kw))
    with pytest.raises(ValueError):
        IF.tracin_sketch(_sketch(**kw), _sketch())


def test_entry_points_raise_without_cuda():
    if torch.cuda.is_available():
        pytest.skip("checks the CPU-only behaviour")
    cfg, m = _cpu_model()
    m.eval()
    b = make_batch(cfg, 3, seed=1)
    with pytest.raises(L.RaindropB200Error):
        IF.project(m, _qt(b), dim=128)
    with pytest.raises(L.RaindropB200Error):
        IF.tracin_sketch(_sketch(), _sketch())


def test_sketch_save_load_round_trip(tmp_path):
    s = _sketch(features=torch.randn(2, 5, 128), lrs=(0.25, 1e-4), seed=2 ** 63 + 9, fields=("a", "b"),
                fingerprints=("x" * 64, "y" * 64))
    p = str(tmp_path / "s.pt")
    s.save(p)
    r = IF.GradientSketch.load(p)
    assert torch.equal(r.features, s.features) and r.features.dtype == torch.float32
    for f in ("lrs", "dim", "seed", "fields", "layout", "fingerprints"):
        assert getattr(r, f) == getattr(s, f), f
    s2 = _sketch(fields=None)
    s2.save(p)
    assert IF.GradientSketch.load(p, map_location="cpu").fields is None


def test_new_symbols_are_exported():
    header = open(HEADER).read()
    for name in ("rd_grad_projection_scratch_bytes", "rd_grad_projection", "rd_debug_projection_signs"):
        assert name in L.SIGNATURES and name + "(" in header
    lib = L.load()
    for name in ("rd_grad_projection_scratch_bytes", "rd_grad_projection", "rd_debug_projection_signs"):
        assert hasattr(lib, name)
    assert lib.rd_grad_projection_scratch_bytes(3, 1000, 100, 1) == 0          # dim refused
    assert lib.rd_grad_projection_scratch_bytes(3, 1000, 256, 2) > 4 * 3 * 1000


# ---- GPU -------------------------------------------------------------------------------------------------------------------
def _device_signs(seed, col0, n_cols, dim):
    out = torch.empty(n_cols, dim, dtype=torch.float32, device="cuda")
    L.check(L.load().rd_debug_projection_signs(seed, col0, n_cols, dim, out.data_ptr(), L.stream_ptr()),
            "rd_debug_projection_signs")
    return out


def _project_raw(G, segs, dim, seed):
    lib = L.load()
    off = (C.c_int64 * len(segs))(*[o for o, _ in segs])
    ln = (C.c_int64 * len(segs))(*[n for _, n in segs])
    rows, ldg = G.shape
    nb = lib.rd_grad_projection_scratch_bytes(rows, ldg, dim, len(segs))
    sc = torch.empty((nb + 3) // 4, dtype=torch.float32, device="cuda")
    out = torch.full((rows, dim), float("nan"), dtype=torch.float32, device="cuda")
    L.check(lib.rd_grad_projection(G.data_ptr(), rows, ldg, off, ln, len(segs), dim, seed, out.data_ptr(), dim,
                                   sc.data_ptr(), L.stream_ptr()), "rd_grad_projection")
    return out


def _device_reference(G, dim, seed, seg_off, seg_len, chunk=1 << 18):
    """float64 [rows, dim] on the device: G's segment columns times the signs of rd_debug_projection_signs (checked
    against the host restatement bitwise by test_device_signs_equal_the_host_restatement), over sqrt(dim)."""
    G = G.double()
    out = torch.zeros(G.shape[0], dim, dtype=torch.float64, device=G.device)
    for o, n in zip(seg_off.tolist(), seg_len.tolist()):
        for c0 in range(o, o + n, chunk):
            c1 = min(o + n, c0 + chunk)
            out += G[:, c0:c1] @ _device_signs(seed, c0, c1 - c0, dim).double()
    return out / math.sqrt(dim)


def _rowwise(got, ref):
    got, ref = got.double(), ref.double()
    return ((got - ref).abs().amax(1) / ref.abs().amax(1).clamp_min(1e-300)).max().item()


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [0, 7, 2 ** 32 + 5, 2 ** 64 - 1])
def test_device_signs_equal_the_host_restatement(seed):
    for col0 in (0, 4, 2 ** 24 + 36, 2 ** 33 + 100):
        for dim in (128, 384):
            got = _device_signs(seed, col0, 300, dim).cpu().numpy()
            np.testing.assert_array_equal(got, projection_matrix(300, dim, seed, col0=col0).astype(np.float32))


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [128, 384])
def test_projection_kernel_against_float64_and_bitwise_per_row(dim):
    g = torch.Generator().manual_seed(dim)
    ldg = 12004
    segs = [(0, 1), (4, 37), (44, 4095), (4140, 4096), (8236, 33), (8272, 3731)]
    G = torch.randn(130, ldg, generator=g) * torch.exp2(torch.randint(-20, 21, (130, ldg), generator=g).float())
    Gd = G.cuda()
    off, ln = np.array([o for o, _ in segs]), np.array([n for _, n in segs])
    ref = torch.as_tensor(project_rows(G.numpy(), dim, 99, off, ln))
    for rows in (1, 7, 37, 130):
        got = _project_raw(Gd[:rows].contiguous(), segs, dim, 99).cpu()
        err = _rowwise(got, ref[:rows])
        assert err <= 1e-5, (rows, err)
    full = _project_raw(Gd, segs, dim, 99)
    alone = torch.cat([_project_raw(Gd[r:r + 1].contiguous(), segs, dim, 99) for r in (0, 63, 64, 129)])
    assert torch.equal(alone, full[[0, 63, 64, 129]])
    perm = torch.randperm(130, generator=g).cuda()
    assert torch.equal(_project_raw(Gd[perm].contiguous(), segs, dim, 99), full[perm])
    sub = torch.tensor([129, 3, 77, 64, 65, 5, 0]).cuda()
    assert torch.equal(_project_raw(Gd[sub].contiguous(), segs, dim, 99), full[sub])


CASES = {"tiny_b6": ("TINY", 6, 1024), "p19_b37": ("P19", 37, 1024), "p12_b3": ("P12", 3, 512),
         "pam_b2": ("PAM", 2, 256)}


def _setup(name, B=None, seed=None):
    cfg_name, B0, dim = CASES[name]
    B = B0 if B is None else B
    cfg = model_config(cfg_name, dropout=0.2)
    batch = make_batch(cfg, B, seed=700 + B if seed is None else seed)
    model = build_dropin(cfg, 21)
    model._prepare(torch.device("cuda")).obprop_mode = EXACT
    model.eval()
    return cfg, to_dev(batch), model, dim


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_project_against_float64_restatement(name):
    cfg, d, model, dim = _setup(name)
    keys = PV.sqnorm_fields(model)
    layout = IF.grad_layout(model)
    with torch.no_grad():
        logits, _, _ = model.forward(d["src"], d["static"], d["times"], d["lengths"])
    G = IF.per_sample_grads(model, d["src"], d["static"], d["times"], d["lengths"], d["y"])
    Gp = IF.per_sample_grads(model, d["src"], d["static"], d["times"], d["lengths"], logits.argmax(1))
    params0 = [p.detach().clone() for p in model.used_parameters()]
    rng0 = model._plan.rng_state.clone()
    for fields in (None, [keys[0], keys[3], keys[-1]]):
        seg_off, seg_len = IF.plan_segments(layout, fields)
        for data, rows in ((_qt(d), G), (_qt(d, y=False), Gp)):
            sk = IF.project(model, data, dim=dim, seed=2 ** 40 + 17, fields=fields)
            assert sk.features.shape == (1, d["src"].shape[1], dim) and sk.features.dtype == torch.float32
            assert sk.fields == (None if fields is None else tuple(fields)) and sk.dim == dim
            ref = _device_reference(rows, dim, 2 ** 40 + 17, seg_off, seg_len)
            err = _rowwise(sk.features[0], ref)
            assert err <= 1e-5, (fields, err)
    assert all(torch.equal(p, q) for p, q in zip(model.used_parameters(), params0))
    assert torch.equal(model._plan.rng_state, rng0) and not model.training


@pytest.mark.gpu
def test_project_bitwise_across_chunking_sources_and_runs():
    from raindrop_b200.data import DeviceDataset
    cfg, d, model, _ = _setup("p19_b37", B=300, seed=5)
    keys = PV.sqnorm_fields(model)
    sd0 = model.state_dict()
    torch.manual_seed(9)
    ck = [({k: sd0[k] + 0.01 * torch.randn_like(sd0[k]) for k in keys}, 0.3), ({k: sd0[k].clone() for k in keys}, 1.7)]
    ref = IF.project(model, _qt(d), checkpoints=ck, dim=512, seed=3)
    assert ref.lrs == (0.3, 1.7) and len(set(ref.fingerprints)) == 2
    assert torch.equal(IF.project(model, _qt(d), checkpoints=ck, dim=512, seed=3).features, ref.features)
    for ibs in (1, 129, 300):
        got = IF.project(model, _qt(d), checkpoints=ck, dim=512, seed=3, internal_batch_size=ibs)
        assert torch.equal(got.features, ref.features), ibs
    ds = DeviceDataset(d["src"], d["static"], d["times"], d["y"])
    assert torch.equal(IF.project(model, ds, checkpoints=ck, dim=512, seed=3, internal_batch_size=100).features,
                       ref.features)
    got = IF.project(model, (ds, torch.arange(300)), checkpoints=ck, dim=512, seed=3)
    assert torch.equal(got.features, ref.features)
    assert got.fingerprints == ref.fingerprints


@pytest.mark.gpu
def test_tracin_sketch_equals_the_product_of_the_features():
    cfg, d, model, _ = _setup("p19_b37", B=200, seed=5)
    _, dq, _, _ = _setup("p19_b37", B=70, seed=6)
    keys = PV.sqnorm_fields(model)
    sd0 = model.state_dict()
    torch.manual_seed(4)
    ck = [({k: sd0[k] + 0.01 * torch.randn_like(sd0[k]) for k in keys}, 0.5), ({k: sd0[k].clone() for k in keys}, 2.0)]
    sq = IF.project(model, _qt(dq, y=False), checkpoints=ck, dim=4096 + 128, seed=8)
    st = IF.project(model, _qt(d), checkpoints=ck, dim=4096 + 128, seed=8)
    S = IF.tracin_sketch(sq, st)
    assert S.dtype == torch.float64 and S.shape == (70, 200)
    ref = torch.as_tensor(IF.tracin_from_grads(sq.features.cpu(), st.features.cpu(), sq.lrs))
    bound = sum(abs(lr) * sq.features[c].double().norm(dim=1)[:, None] * st.features[c].double().norm(dim=1)[None, :]
                for c, lr in enumerate(sq.lrs)).cpu()
    assert ((S.cpu() - ref).abs() <= 1e-5 * bound).all()
    with pytest.raises(ValueError):
        IF.tracin_sketch(sq, IF.project(model, _qt(d), checkpoints=ck[:1] + [(ck[1][0], 2.0)], dim=4096 + 128, seed=9))
    with pytest.raises(ValueError):
        IF.tracin_sketch(sq, IF.project(model, _qt(d), checkpoints=ck[1:], dim=4096 + 128, seed=8))


@pytest.mark.gpu
def test_sketch_scores_lie_within_six_sigma_of_exact_tracin():
    cfg = model_config("P19", dropout=0.2)
    model = build_dropin(cfg, 21)
    model.eval()
    dq = to_dev(make_batch(cfg, 16, seed=61))
    dt = to_dev(make_batch(cfg, 64, seed=62))
    exact = IF.tracin(model, _qt(dq), _qt(dt))
    sk = IF.tracin_sketch(IF.project(model, _qt(dq), dim=4096, seed=1234),
                          IF.project(model, _qt(dt), dim=4096, seed=1234))
    nq = IF.self_influence(model, _qt(dq)).sqrt()
    nt = IF.self_influence(model, _qt(dt)).sqrt()
    sigma = ((nq[:, None] * nt[None, :]) ** 2 + exact ** 2).div(4096).sqrt()
    z = ((sk - exact).abs() / sigma).max().item()
    assert z <= 6.0, z


@pytest.mark.gpu
@pytest.mark.parametrize("name,n", [("PAM", 24), ("LARGE", 24)])
def test_large_shapes_complete_within_the_scratch_plan(name, n):
    cfg = model_config(name, dropout=0.2)
    model = build_dropin(cfg, 21)
    model.eval()
    d = to_dev(make_batch(cfg, n, seed=52))
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    sk = IF.project(model, _qt(d), dim=4096, seed=1)
    assert sk.features.shape == (1, n, 4096) and torch.isfinite(sk.features).all()
    assert sk.features.abs().amax().item() > 0
    assert torch.cuda.max_memory_allocated() - base < 4 * (1 << 30)
