"""Gradients of Raindrop_v2 (and legacy Raindrop v1) with respect to the model INPUTS src, static and times: what
saliency maps, integrated gradients and adversarial training need.  Reference values: tests/golden/input_grads.npz,
produced by the reference's own files (tools/make_input_grad_golden.py), eval mode, cross-entropy loss.

Tolerances are normwise max|delta| / max|ref| as in test_gpu_parity.py.  d_src runs through the transpose of the first
ob-prop layer, so in the single-pass TF32 mode its ReLU-gate flips (DESIGN.md "Precision") are bounded in relative L2."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import build_dropin, case_setup, check_against_golden, load_golden, normwise, rel_l2, to_dev
from raindrop_b200.synth import make_batch, model_config, synth_weights

EXACT, FAST = 2, 1
TOL_EXACT, TOL_EXACT_WIDE = 2e-3, 1e-2          # C = T*d_ob >= 1024: K = 1024..2400 dot products flip a rare gate
TOL_FAST, SRC_L2_FAST = 2e-2, 5e-2
FULL = ["tiny_dense", "tiny_t0", "tiny_sparse", "tiny8_nostatic"]
FINGERPRINT = ["p19_b5_leave10", "p12_b2", "pam_b2"]
ORACLE_CASES = [("P19", 1, {}), ("P19", 37, {}), ("P19", 100, {"first_time_zero": True}), ("P19", 128, {"zero_sensors": 10}),
                ("P12", 5, {}), ("PAM", 3, {}), ("TINY", 7, {"full_length": True}), ("TINY8", 9, {}), ("LARGE", 2, {})]


def _exact_tol(cfg):
    return TOL_EXACT_WIDE if cfg["max_len"] * cfg["d_ob"] >= 1024 else TOL_EXACT


def _leaves(batch, device):
    d = to_dev(batch, device)
    out = {"d_src": d["src"].clone().requires_grad_(True), "d_times": d["times"].clone().requires_grad_(True)}
    if d["static"] is not None:
        out["d_static"] = d["static"].clone().requires_grad_(True)
    return out, d


def _run(model, batch, device="cuda"):
    """Cross-entropy input gradients {d_src, d_times[, d_static]} of `model` on `batch`."""
    x, d = _leaves(batch, device)
    logits, _, _ = model.forward(x["d_src"], x.get("d_static"), x["d_times"], d["lengths"])
    g = torch.autograd.grad(F.cross_entropy(logits, d["y"]), list(x.values()))
    return dict(zip(x, g))


def _dropin(cfg, batch, wseed, mode, train=False):
    model = build_dropin(cfg, wseed).train(train)
    model._plan.obprop_mode = mode
    return _run(model, batch)


def _check(got, ref, mode, cfg, ref_tf32=None):
    """Exact mode: normwise everywhere.  Fast mode: relative L2 for src and times against the fp32 oracle -- the forward's
    TF32 error (3e-4) flips the odd ReLU gate of the encoder, which moves single tokens' d_times by a few percent of
    max|d_times| (per-token gradients do not average such flips out the way parameter gradients do) -- and normwise
    for static and times against the oracle evaluated under the kernels' TF32 rounding model."""
    for k, v in got.items():
        if mode == EXACT:
            e = normwise(v, ref[k])
            assert e < _exact_tol(cfg), (k, "normwise", e)
            continue
        if k in ("d_src", "d_times"):
            e = rel_l2(v, ref[k])
            assert e < SRC_L2_FAST, (k, "rel_l2", e)
        if k in ("d_static", "d_times"):
            e = normwise(v, ref_tf32[k] if ref_tf32 is not None else ref[k])
            assert e < TOL_FAST, (k, "normwise", e)


# ---- CPU: the oracle reproduces the reference's input gradients --------------------------------------------------
@pytest.mark.parametrize("name", FULL)
def test_oracle_reproduces_input_grad_fixture(golden_dir, name):
    from oracle.raindrop_oracle import build_oracle_model
    z = np.load(golden_dir + "/input_grads.npz")
    _, meta = load_golden(golden_dir, name)
    cfg, batch = case_setup(meta)
    oracle = build_oracle_model(cfg).eval()
    synth_weights(oracle, cfg, seed=meta["weight_seed"])
    x, d = _leaves(batch, "cpu")
    logits, _, _ = oracle.forward_dense(x["d_src"], x.get("d_static"), x["d_times"], d["lengths"])
    got = dict(zip(x, torch.autograd.grad(F.cross_entropy(logits, d["y"]), list(x.values()))))
    assert sorted(got) == sorted(k[len(name) + 1:] for k in z.files if k.startswith(name + "."))
    for k, v in got.items():
        assert normwise(v, z[name + "." + k]) < 1e-4, (k, normwise(v, z[name + "." + k]))
    N = cfg["d_inp"]
    assert np.all(z[name + ".d_src"][:, :, N:] == 0)          # the mask half takes no part without sensor_wise_mask


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
@pytest.mark.parametrize("name", FULL + FINGERPRINT)
def test_golden_input_grads(golden_dir, name, mode):
    z = np.load(golden_dir + "/input_grads.npz")
    _, meta = load_golden(golden_dir, name)
    cfg, batch = case_setup(meta)
    got = _dropin(cfg, batch, meta["weight_seed"], mode)
    full = name in FULL
    errs = {}
    for k, v in got.items():
        if mode == EXACT:
            check_against_golden(z, full, "%s.%s" % (name, k), v, _exact_tol(cfg), errs)
        elif k == "d_src":
            check_against_golden(z, full, "%s.%s" % (name, k), v, SRC_L2_FAST, errs, metric=rel_l2)
        else:
            check_against_golden(z, full, "%s.%s" % (name, k), v, TOL_FAST, errs)
    print(name, mode, errs)


@pytest.mark.gpu
def test_legacy_v1_input_grads(golden_dir):
    from raindrop_b200.models_rd import Raindrop
    from raindrop_b200.synth import CONFIGS
    z = np.load(golden_dir + "/v1_p12_b3.npz")
    zg = np.load(golden_dir + "/input_grads.npz")
    cfg = dict(CONFIGS["P12"]); cfg["name"] = "P12"
    batch = make_batch(dict(cfg, d_ob=2), 3, seed=77)
    model = Raindrop(36, 72, 2, 144, 2, 0.2, 215, 9, 100, 0.5, "mean", 2, torch.from_numpy(z["global_structure"]))
    model.load_state_dict({k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd.")})
    model = model.cuda().eval()
    d = to_dev(batch)
    static = d["static"].clone().requires_grad_(True)
    times = d["times"].clone().requires_grad_(True)
    logits, _, _ = model.forward(d["src"], static, times, d["lengths"])
    F.cross_entropy(logits, d["y"]).backward()
    for k, g in (("d_static", static.grad), ("d_times", times.grad)):
        e = normwise(g, zg["v1_p12_b3." + k])
        assert e < TOL_EXACT, (k, e)
    assert model.emb.weight.grad is not None and model.mlp_static[0].weight.grad is not None


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name,B,opts", ORACLE_CASES)
def test_input_grads_against_oracle(cfg_name, B, opts):
    from oracle.raindrop_oracle import build_oracle_model
    cfg = model_config(cfg_name, dropout=0.2)
    batch = make_batch(cfg, B, seed=100 + B, **opts)
    oracle = build_oracle_model(cfg).eval()
    synth_weights(oracle, cfg, seed=21)
    x, d = _leaves(batch, "cpu")
    logits, _, _ = oracle.forward_dense(x["d_src"], x.get("d_static"), x["d_times"], d["lengths"])
    ref = dict(zip(x, torch.autograd.grad(F.cross_entropy(logits, d["y"]), list(x.values()))))
    x, d = _leaves(batch, "cpu")
    logits, _, _ = oracle.forward_dense(x["d_src"], x.get("d_static"), x["d_times"], d["lengths"], tf32_model=True)
    ref_tf32 = dict(zip(x, torch.autograd.grad(F.cross_entropy(logits, d["y"]), list(x.values()))))
    for mode in (EXACT, FAST):
        got = _dropin(cfg, batch, 21, mode)
        print(cfg_name, B, mode, {k: (normwise(v, ref[k]), rel_l2(v, ref[k]), normwise(v, ref_tf32[k])) for k, v in got.items()})
        _check(got, ref, mode, cfg, ref_tf32)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
def test_exact_zeros(mode):
    """Bitwise zeros where the reference has them: the mask half of d_src, d_src wherever the value is 0 (unobserved or
    padded; relu'(0) = 0) and d_times on padded rows -- in train mode too."""
    cfg = model_config("P19", dropout=0.2)
    batch = make_batch(cfg, 24, seed=5, first_time_zero=True, zero_sensors=10)
    N = cfg["d_inp"]
    for train in (False, True):
        got = _dropin(cfg, batch, 3, mode, train=train)
        src = batch["src"].cuda()
        assert torch.all(got["d_src"][:, :, N:] == 0)
        assert torch.all(got["d_src"][:, :, :N][src[:, :, :N] == 0] == 0)
        assert torch.count_nonzero(got["d_src"]) > 0
        T = src.shape[0]
        padded = torch.arange(T, device="cuda")[:, None] >= batch["lengths"].cuda()[None, :]
        assert padded.any() and torch.all(got["d_times"][padded] == 0)
        assert torch.count_nonzero(got["d_times"][~padded]) > 0


def _launches(fn):
    from raindrop_b200 import lib as L
    lib = L.load()
    torch.cuda.synchronize()
    n0 = lib.rd_launch_count()
    fn()
    torch.cuda.synchronize()
    return int(lib.rd_launch_count() - n0)


@pytest.mark.gpu
def test_frozen_parameters():
    """model.requires_grad_(False): identical input gradients, no parameter gradient, fewer kernel launches."""
    cfg = model_config("P19", dropout=0.2)
    batch = make_batch(cfg, 32, seed=8)
    res = {}
    for frozen in (False, True):
        model = build_dropin(cfg, 6).eval()
        if frozen:
            model.requires_grad_(False)
        x, d = _leaves(batch, "cuda")
        logits, _, _ = model.forward(x["d_src"], x["d_static"], x["d_times"], d["lengths"])
        loss = F.cross_entropy(logits, d["y"])
        n = _launches(loss.backward)
        res[frozen] = (n, {k: v.grad for k, v in x.items()})
        with_grad = [k for k, p in model.named_parameters() if p.grad is not None]
        assert (with_grad == []) == frozen, with_grad
    (n_full, g_full), (n_frozen, g_frozen) = res[False], res[True]
    for k in g_full:
        assert torch.equal(g_full[k], g_frozen[k]), k
    print("backward launches: parameters trainable %d, frozen %d" % (n_full, n_frozen))
    assert n_frozen < n_full


@pytest.mark.gpu
def test_backward_without_input_grads_launches_unchanged():
    """A backward with no input requiring grad makes exactly the one rd_raindrop_v2_bwd call (same launches as calling
    the C ABI directly), and asking for input gradients adds the one input-gradient call on top."""
    from raindrop_b200 import lib as L
    lib = L.load()
    cfg = model_config("P19", dropout=0.2)
    batch = make_batch(cfg, 32, seed=9)
    model = build_dropin(cfg, 6).train()
    model._plan.debug_keep_workspace = True
    d = to_dev(batch)
    logits, _, _ = model.forward(d["src"], d["static"], d["times"], d["lengths"])
    n_module = _launches(F.cross_entropy(logits, d["y"]).backward)
    plan = model._plan
    G = plan._grad_struct[1]
    scratch = next(iter(plan._scratch.values()))
    d_logits = torch.zeros_like(logits)

    def direct():
        L.check(lib.rd_raindrop_v2_bwd(C.byref(plan.last_dims), C.byref(plan._param_struct[1]), d["static"].data_ptr(),
                                       d["lengths"].data_ptr(), plan.node_scale.data_ptr(), plan.last_workspace.data_ptr(),
                                       d_logits.data_ptr(), C.byref(G), scratch.data_ptr(), L.BWD_ALL, L.stream_ptr()), "bwd")
    assert n_module == _launches(direct)
    x, d2 = _leaves(batch, "cuda")
    logits, _, _ = model.forward(x["d_src"], x["d_static"], x["d_times"], d2["lengths"])
    n_input = _launches(F.cross_entropy(logits, d2["y"]).backward)
    assert n_input == n_module + 3, (n_input, n_module)      # weight split + dX0 GEMM + lift/PE/static backward


def _fd_check(model, batch, rng0, which, eps=1e-3):
    """Central difference of the loss along a random direction v vs <d_which, v>, dropout masks replayed."""
    x, d = _leaves(batch, "cuda")

    def loss_at(inputs):
        model._plan.rng_state.copy_(rng0)
        logits, _, _ = model.forward(inputs["d_src"], inputs.get("d_static"), inputs["d_times"], d["lengths"])
        return F.cross_entropy(logits, d["y"])
    g = torch.autograd.grad(loss_at(x), [x[which]])[0]
    gen = torch.Generator(device="cuda").manual_seed(3)
    v = torch.randn(x[which].shape, generator=gen, device="cuda")
    base = x[which].detach()
    if which == "d_src":
        N = base.shape[2] // 2
        support = torch.zeros_like(base, dtype=torch.bool)
        support[:, :, :N] = base[:, :, :N].abs() > 1e-2        # no ReLU kink of the lift within eps
        v = v * support
    elif which == "d_times":
        v = v * (torch.arange(base.shape[0], device="cuda")[:, None] < d["lengths"][None, :])
    with torch.no_grad():
        plus = {k: t.detach() for k, t in x.items()}
        minus = dict(plus)
        plus[which] = base + eps * v
        minus[which] = base - eps * v
        fd = (loss_at(plus).double() - loss_at(minus).double()) / (2 * eps)
    an = float((g.double() * v.double()).sum())
    return float(fd), an


@pytest.mark.gpu
def test_train_mode_finite_difference():
    """Train mode (dropout 0.2, exact ob-prop mode): the backward replays the forward's lift / encoder dropout masks, so
    the input gradient is the derivative of the very function the forward computed."""
    cfg = model_config("TINY", dropout=0.2)
    batch = make_batch(cfg, 6, seed=17)
    model = build_dropin(cfg, 4).train()
    model._plan.obprop_mode = EXACT
    x, d = _leaves(batch, "cuda")
    model.forward(x["d_src"], x["d_static"], x["d_times"], d["lengths"])      # creates the rng state
    rng0 = model._plan.rng_state.clone()
    for which in ("d_src", "d_times", "d_static"):
        fd, an = _fd_check(model, batch, rng0, which)
        print(which, "finite difference %.6e analytic %.6e" % (fd, an))
        assert abs(fd - an) <= 2e-2 * abs(an) and abs(an) > 0, (which, fd, an)


@pytest.mark.gpu
def test_autograd_grad_fp64_noncontiguous():
    """torch.autograd.grad through the module's .to(float32).contiguous(): fp64 and non-contiguous inputs get the same
    gradients as contiguous fp32 ones (in their own dtype)."""
    cfg = model_config("P19", dropout=0.2)
    batch = make_batch(cfg, 8, seed=12)
    model = build_dropin(cfg, 5).eval()
    d = to_dev(batch)
    src = d["src"].double().permute(1, 0, 2).contiguous().requires_grad_(True)        # [B, T, 2N], used transposed
    static = d["static"].double().t().contiguous().requires_grad_(True)               # [ds, B], used transposed
    times = d["times"].double().t().contiguous().requires_grad_(True)
    logits, _, _ = model.forward(src.transpose(0, 1), static.t(), times.t(), d["lengths"])
    g = torch.autograd.grad(logits[:, 1].sum(), [src, static, times])
    assert [t.dtype for t in g] == [torch.float64] * 3 and [t.shape for t in g] == [src.shape, static.shape, times.shape]
    x, _ = _leaves(batch, "cuda")
    logits32, _, _ = model.forward(x["d_src"], x["d_static"], x["d_times"], d["lengths"])
    g32 = torch.autograd.grad(logits32[:, 1].sum(), [x["d_src"], x["d_static"], x["d_times"]])
    assert torch.equal(g[0].transpose(0, 1).float(), g32[0])
    assert torch.equal(g[1].t().float(), g32[1])
    assert torch.equal(g[2].t().float(), g32[2])


@pytest.mark.gpu
def test_flat_adam_bound_model():
    """A FlatAdam-bound model takes the general path when inputs need gradients; its update equals torch.optim.Adam's."""
    from raindrop_b200.optim import FlatAdam
    cfg = model_config("P19", dropout=0.0)
    B = 16
    m1 = build_dropin(cfg, 8).train(); m2 = build_dropin(cfg, 8).train()
    o1 = torch.optim.Adam(m1.parameters(), lr=1e-3); o2 = FlatAdam(m2, lr=1e-3)
    for it in range(3):          # plain fast-path step first, then two with input gradients
        batch = make_batch(cfg, B, seed=60 + it)
        srcg = []
        for m, o in ((m1, o1), (m2, o2)):
            x, d = _leaves(batch, "cuda")
            if it == 0:
                x = {k: t.detach() for k, t in x.items()}
            logits, _, _ = m.forward(x["d_src"], x["d_static"], x["d_times"], d["lengths"])
            o.zero_grad()
            F.cross_entropy(logits, d["y"]).backward()
            o.step()
            srcg.append(x["d_src"].grad)
        if it > 0:
            assert normwise(srcg[1], srcg[0]) < 1e-3, normwise(srcg[1], srcg[0])
    p1, p2 = dict(m1.named_parameters()), dict(m2.named_parameters())
    for k, _ in m2._plan.fields:
        assert normwise(p2[k].grad, p1[k].grad) < 2e-2, k          # overwritten, not accumulated onto the last step
        assert rel_l2(p2[k], p1[k]) < 5e-3, k


@pytest.mark.gpu
@pytest.mark.parametrize("d_pe,max_len", [(16, 60), (16, 215), (36, 215)])
def test_positional_encoding_module_gradient(d_pe, max_len):
    from raindrop_b200.models_rd import PositionalEncodingTF
    g = torch.Generator().manual_seed(d_pe + max_len)
    t = (torch.rand(max_len, 7, generator=g) * 50)
    w = torch.randn(max_len, 7, d_pe, generator=g)
    tc = t.cuda().requires_grad_(True)
    (PositionalEncodingTF(d_pe, max_len, 100)(tc) * w.cuda()).sum().backward()
    tr = t.clone().requires_grad_(True)
    ts = torch.from_numpy((float(max_len) ** np.linspace(0, 1, d_pe // 2)).astype(np.float32))
    scaled = tr[:, :, None] / ts
    (torch.cat([torch.sin(scaled), torch.cos(scaled)], -1) * w).sum().backward()
    assert normwise(tc.grad, tr.grad) < 1e-5, normwise(tc.grad, tr.grad)
