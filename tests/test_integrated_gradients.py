"""Integrated-gradients attribution of Raindrop_v2 (raindrop_b200.attribution, rd_raindrop_v2_integrated_gradients).
Reference values: tests/golden/integrated_gradients.npz, produced by the reference's own files in eval mode with zero
baselines (tools/make_ig_golden.py).  Tolerances follow test_input_grads.py: normwise max|delta| / max|ref| in the
error-compensated ob-prop mode, relative L2 for attr_src in the single-pass TF32 mode."""
import json

import numpy as np
import pytest
import torch

from helpers import build_dropin, case_setup, check_against_golden, load_golden, normwise, rel_l2, to_dev
from raindrop_b200 import attribution as A
from raindrop_b200.synth import make_batch, model_config, synth_weights

EXACT, FAST = 2, 1
TOL_EXACT, TOL_EXACT_WIDE = 2e-3, 1e-2
TOL_FAST, SRC_L2_FAST = 2e-2, 5e-2
FULL = ["tiny_dense", "tiny_t0", "tiny_sparse", "tiny8_nostatic"]
FINGERPRINT = ["p19_b5_leave10", "p12_b2", "pam_b2"]


def _exact_tol(cfg):
    return TOL_EXACT_WIDE if cfg["max_len"] * cfg["d_ob"] >= 1024 else TOL_EXACT


def _fixture(golden_dir):
    z = np.load(golden_dir + "/integrated_gradients.npz")
    meta = json.loads(bytes(z["meta"]).decode())
    return z, dict(meta["full"], **meta["fingerprint"])


def ig_loop(forward, src, static, times, lengths, target, n_steps, method):
    """Integrated gradients by the hand-written loop (zero baselines): one forward and one torch.autograd.grad of
    sum_b logits[b, target[b]] per quadrature node, at the fp32 nodes the device path reads.  Returns (attr_src,
    attr_static | None) in fp64."""
    N = src.shape[2] // 2
    a32, w32 = (torch.from_numpy(v.astype(np.float32)) for v in A.quadrature(n_steps, method))
    g_src = torch.zeros(src.shape, dtype=torch.float64, device=src.device)
    g_st = None if static is None else torch.zeros(static.shape, dtype=torch.float64, device=src.device)
    for a, w in zip(a32.to(src.device), w32.tolist()):
        xs = src.clone()
        xs[:, :, :N] = a * src[:, :, :N]
        xs.requires_grad_(True)
        leaves = [xs]
        ss = None
        if static is not None:
            ss = (a * static).requires_grad_(True)
            leaves.append(ss)
        logits = forward(xs, ss, times, lengths)
        g = torch.autograd.grad(logits.gather(1, target[:, None]).sum(), leaves)
        g_src += w * g[0].double()
        if static is not None:
            g_st += w * g[1].double()
    attr_src = src.double() * g_src
    attr_src[:, :, N:] = 0
    return attr_src, None if static is None else static.double() * g_st


# ---- CPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", FULL)
def test_oracle_reproduces_ig_fixture(golden_dir, name):
    """The CPU oracle (forward_dense + autograd over the same nodes) reproduces the reference's attributions."""
    from oracle.raindrop_oracle import build_oracle_model
    z, spec = _fixture(golden_dir)
    method, n_steps, _ = spec[name]
    _, meta = load_golden(golden_dir, name)
    cfg, batch = case_setup(meta)
    oracle = build_oracle_model(cfg).eval()
    synth_weights(oracle, cfg, seed=meta["weight_seed"])

    def fwd(s, st, t, ln):
        return oracle.forward_dense(s, st, t, ln)[0]
    target = torch.from_numpy(z[name + ".target"])
    attr_src, attr_st = ig_loop(fwd, batch["src"], batch["static"], batch["times"], batch["lengths"], target, n_steps, method)
    assert normwise(attr_src, z[name + ".attr_src"]) < 1e-4, normwise(attr_src, z[name + ".attr_src"])
    if attr_st is not None:
        assert normwise(attr_st, z[name + ".attr_static"]) < 1e-4
    else:
        assert name + ".attr_static" not in z.files
    with torch.no_grad():
        f_x = fwd(batch["src"], batch["static"], batch["times"], batch["lengths"])
    assert normwise(f_x, z[name + ".endpoint_logits"][1]) < 1e-4
    if meta["case"] == "tiny_t0":               # target None: the argmax class at x
        assert torch.equal(target, f_x.argmax(dim=1))
    N = cfg["d_inp"]
    assert np.all(z[name + ".attr_src"][:, :, N:] == 0)


@pytest.mark.parametrize("n", [1, 2, 7, 16, 50])
def test_quadrature_tables(n):
    a, w = A.quadrature(n, "gausslegendre")
    x, v = np.polynomial.legendre.leggauss(n)
    assert abs(w.sum() - 1.0) < 1e-12
    np.testing.assert_allclose(a, (x + 1) / 2, rtol=0, atol=1e-15)
    np.testing.assert_allclose(w, v / 2, rtol=0, atol=1e-15)
    assert np.all((a > 0) & (a < 1))
    if n >= 2:
        a, w = A.quadrature(n, "riemann_trapezoid")
        assert abs(w.sum() - 1.0) < 1e-12
        assert a[0] == 0.0 and a[-1] == 1.0 and np.all(np.diff(a) > 0)
        assert w[0] == w[-1] == 0.5 / (n - 1)


def test_sensor_ranking_feeds_removal_indices():
    from raindrop_b200.data import removal_indices
    T, B, N = 5, 4, 6
    g = torch.Generator().manual_seed(0)
    attr = torch.zeros(T, B, 2 * N)
    attr[:, :, :N] = torch.randn(T, B, N, generator=g)
    attr[:, :, 4] = 0
    attr[:, :, 2] = 0                             # a tie: sensors 2 and 4 both score 0, index 2 ranks first
    attr[:, :, N:] = 100.0                        # the mask half takes no part
    imp = A.sensor_importance(attr, N)
    assert imp.shape == (N,)
    np.testing.assert_allclose(imp.numpy(), attr[:, :, :N].abs().sum(0).mean(0).numpy())
    names = ["HR", "O2Sat", "Temp", "SBP", "MAP", "Resp"]
    r = A.sensor_ranking(imp, names)
    assert r.shape == (N, 2) and r.dtype.kind == "U"
    idx = r[:, 0].astype(int)
    assert sorted(idx.tolist()) == list(range(N))
    assert np.all(np.diff(imp.numpy()[idx]) <= 0)
    assert idx.tolist().index(2) < idx.tolist().index(4)
    assert [names[i] for i in idx] == r[:, 1].tolist()
    np.testing.assert_array_equal(removal_indices(B, N, 0.5, level="set", density_scores=r[:, 0]), idx[:3])
    assert A.sensor_ranking(imp)[:, 1].tolist() == [str(i) for i in idx]


def _cpu_model(train=False):
    cfg = model_config("TINY", dropout=0.2)
    return build_dropin(cfg, 3, device="cpu").train(train), make_batch(cfg, 3, seed=1)


def test_argument_validation():
    model, b = _cpu_model()
    args = (b["src"], b["static"], b["times"], b["lengths"])
    with pytest.raises(ValueError, match="eval"):
        A.integrated_gradients(model.train(), *args)
    model.eval()
    with pytest.raises(ValueError):
        A.integrated_gradients(model, *args, n_steps=0)
    with pytest.raises(ValueError):
        A.integrated_gradients(model, *args, n_steps=1, method="riemann_trapezoid")
    with pytest.raises(ValueError):
        A.integrated_gradients(model, *args, method="riemann_left")
    with pytest.raises(ValueError):
        A.integrated_gradients(model, *args, target=2)
    with pytest.raises(ValueError):
        A.integrated_gradients(model, *args, target=torch.tensor([0, 1, -1]))
    with pytest.raises(ValueError):
        A.integrated_gradients(model, *args, target=torch.tensor([0, 1]))
    with pytest.raises(ValueError):
        A.integrated_gradients(model, *args, baselines=torch.zeros(1))
    with pytest.raises(ValueError):
        A.integrated_gradients(model, b["src"][:, :, :3], b["static"], b["times"], b["lengths"])
    with pytest.raises(ValueError):
        A.integrated_gradients(model, *args, internal_batch_size=0)


def test_no_cuda_raises(monkeypatch):
    from raindrop_b200.lib import RaindropB200Error
    model, b = _cpu_model()
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RaindropB200Error):
        A.integrated_gradients(model, b["src"], b["static"], b["times"], b["lengths"], target=1)


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _model(cfg, wseed, mode):
    m = build_dropin(cfg, wseed).eval()
    m._plan.obprop_mode = mode
    return m


def _loop(model, d, target, n_steps, method="gausslegendre"):
    def fwd(s, st, t, ln):
        return model.forward(s, st, t, ln)[0]
    return ig_loop(fwd, d["src"], d["static"], d["times"], d["lengths"], target, n_steps, method)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
@pytest.mark.parametrize("name", FULL + FINGERPRINT)
def test_golden_integrated_gradients(golden_dir, name, mode):
    z, spec = _fixture(golden_dir)
    method, n_steps, tmode = spec[name]
    _, meta = load_golden(golden_dir, name)
    cfg, batch = case_setup(meta)
    d = to_dev(batch)
    model = _model(cfg, meta["weight_seed"], mode)
    target = d["y"] if tmode == "labels" else None
    attr_src, attr_st, delta = A.integrated_gradients(model, d["src"], d["static"], d["times"], d["lengths"], target=target,
                                                      n_steps=n_steps, method=method, return_convergence_delta=True)
    full = name in FULL
    tol = _exact_tol(cfg) if mode == EXACT else TOL_FAST
    errs = {}
    if mode == EXACT:
        check_against_golden(z, full, name + ".attr_src", attr_src, tol, errs)
    else:
        check_against_golden(z, full, name + ".attr_src", attr_src, SRC_L2_FAST, errs, metric=rel_l2)
    if attr_st is not None:
        check_against_golden(z, full, name + ".attr_static", attr_st, tol, errs)
    else:
        assert name + ".attr_static" not in z.files and not cfg["static"]
    # endpoints and the completeness error, on the scale of F(x) - F(x')
    ends_ref = torch.from_numpy(z[name + ".endpoint_logits"])
    tgt = torch.from_numpy(z[name + ".target"])
    ends = _endpoint_logits(model, d, tgt.cuda())
    errs["endpoint_logits"] = normwise(ends, ends_ref)
    assert errs["endpoint_logits"] < tol
    f = ends_ref.gather(2, tgt.view(1, -1, 1).expand(2, -1, 1))[:, :, 0]
    scale = float((f[1] - f[0]).abs().max()) + 1e-6
    errs["delta"] = float((delta.cpu() - torch.from_numpy(z[name + ".delta"])).abs().max()) / scale
    assert errs["delta"] < tol
    print(name, mode, errs)


def _endpoint_logits(model, d, target):
    """logits at the zero baseline and at x, through the module's forward (as the call evaluates them)."""
    N = d["src"].shape[2] // 2
    with torch.no_grad():
        x0 = d["src"].clone()
        x0[:, :, :N] = 0
        st0 = None if d["static"] is None else torch.zeros_like(d["static"])
        return torch.stack([model.forward(x0, st0, d["times"], d["lengths"])[0],
                            model.forward(d["src"], d["static"], d["times"], d["lengths"])[0]])


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name,B,opts", [("P19", 6, {"zero_sensors": 10}), ("P19", 1, {}), ("P19", 7, {"first_time_zero": True}),
                                             ("TINY8", 5, {}), ("P12", 3, {}), ("PAM", 2, {})])
def test_equals_input_grad_loop(cfg_name, B, opts):
    """Exact mode: the batched device call equals the hand-written loop of n_steps input-gradient calls at the same
    nodes (shapes: B = 1, odd B, no statics, the P12 and PAM (T > 64 attention) shapes)."""
    cfg = model_config(cfg_name, dropout=0.2)
    d = to_dev(make_batch(cfg, B, seed=40 + B, **opts))
    model = _model(cfg, 9, EXACT)
    n_steps = 6
    attr_src, attr_st = A.integrated_gradients(model, d["src"], d["static"], d["times"], d["lengths"], target=d["y"],
                                               n_steps=n_steps, internal_batch_size=4 * B)
    ref_src, ref_st = _loop(model, d, d["y"], n_steps)
    e = {"attr_src": normwise(attr_src, ref_src)}
    if ref_st is not None:
        e["attr_static"] = normwise(attr_st, ref_st)
    else:
        assert attr_st is None
    print(cfg_name, B, e)
    assert max(e.values()) < 1e-5, e
    assert torch.count_nonzero(attr_src) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
def test_chunking_invariance(mode):
    """With the arithmetic mode pinned, the chunk size (one step per chunk, 3 with a ragged tail, all at once) does not
    change the result: the running sums add the same per-step values in the same order."""
    cfg = model_config("P19", dropout=0.2)
    B, n_steps = 8, 7
    d = to_dev(make_batch(cfg, B, seed=3))
    model = _model(cfg, 4, mode)
    res = [A.integrated_gradients(model, d["src"], d["static"], d["times"], d["lengths"], n_steps=n_steps,
                                  internal_batch_size=ib) for ib in (B, 3 * B, n_steps * B)]
    for attr_src, attr_st in res[1:]:
        assert normwise(attr_src, res[0][0]) < 1e-6 and normwise(attr_st, res[0][1]) < 1e-6
    print("chunkings bitwise equal:", all(torch.equal(r[0], res[0][0]) and torch.equal(r[1], res[0][1]) for r in res[1:]))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
def test_exact_zeros(mode):
    """Bitwise zeros: the mask half, unobserved entries (x = x' = 0) and padded rows."""
    cfg = model_config("P19", dropout=0.2)
    d = to_dev(make_batch(cfg, 12, seed=5, first_time_zero=True, zero_sensors=10))
    model = _model(cfg, 3, mode)
    attr_src, _ = A.integrated_gradients(model, d["src"], d["static"], d["times"], d["lengths"], n_steps=8)
    N = cfg["d_inp"]
    bits = attr_src.view(torch.int32)
    assert torch.all(bits[:, :, N:] == 0)
    assert torch.all(bits[:, :, :N][d["src"][:, :, :N] == 0] == 0)
    # padded rows: zero timestamps after the first row (the first timestamp is 0 here, so lengths = #(t > 0) counts
    # one row fewer than the data holds, and row lengths[b] is still an observed row)
    T = attr_src.shape[0]
    padded = (d["times"] == 0) & (torch.arange(T, device="cuda")[:, None] > 0)
    assert padded.any() and torch.all(bits[padded] == 0)
    assert torch.count_nonzero(attr_src) > 0


@pytest.mark.gpu
def test_targets_and_baselines():
    """target as an int, a tensor and None (argmax at x) agree; an explicit zero baseline pair equals the default; a
    nonzero baseline gives a small completeness error too."""
    cfg = model_config("P19", dropout=0.2)
    B = 5
    d = to_dev(make_batch(cfg, B, seed=8))
    model = _model(cfg, 2, EXACT)
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    a_int = A.integrated_gradients(*args, target=1, n_steps=8)
    a_vec = A.integrated_gradients(*args, target=torch.ones(B, dtype=torch.int64, device="cuda"), n_steps=8)
    assert torch.equal(a_int[0], a_vec[0]) and torch.equal(a_int[1], a_vec[1])
    a_none = A.integrated_gradients(*args, target=None, n_steps=8, return_convergence_delta=True)
    top = _endpoint_logits(model, d, None)[1].argmax(dim=1)
    a_top = A.integrated_gradients(*args, target=top, n_steps=8, return_convergence_delta=True)
    for x, y in zip(a_none, a_top):
        assert torch.equal(x, y)
    a_zero = A.integrated_gradients(*args, target=top, n_steps=8, baselines=(0.0, torch.zeros(1, cfg["d_static"])))
    assert torch.equal(a_zero[0], a_top[0]) and torch.equal(a_zero[1], a_top[1])
    N = cfg["d_inp"]
    base = torch.full((1, 1, 2 * N), 0.3, device="cuda")
    _, _, delta = A.integrated_gradients(*args, target=top, n_steps=32, baselines=(base, None),
                                         return_convergence_delta=True)
    ends = _endpoint_logits(model, d, None)
    print("delta with a 0.3 baseline:", delta.tolist())
    assert float(delta.abs().max()) < 5e-2 * float(ends.abs().max())


@pytest.mark.gpu
def test_no_side_effects():
    """Parameters, their .grad, the dropout rng state and a bound FlatAdam (moments, step count, captured slots) are
    untouched; a model in training mode raises."""
    from raindrop_b200.optim import FlatAdam
    import torch.nn.functional as F
    cfg = model_config("P19", dropout=0.2)
    B = 16
    model = build_dropin(cfg, 8).train()
    opt = FlatAdam(model, lr=1e-3)
    for it in range(3):            # eager step, then CUDA-graph capture and replay
        d = to_dev(make_batch(cfg, B, seed=60 + it))
        logits, _, _ = model.forward(d["src"], d["static"], d["times"], d["lengths"])
        F.cross_entropy(logits, d["y"]).backward()
        opt.step()
    with pytest.raises(ValueError):
        A.integrated_gradients(model, d["src"], d["static"], d["times"], d["lengths"])
    plan = model._plan
    slot = next(iter(plan._slots.values()))
    snap = {"flat_p": opt.flat_p.detach(), "flat_g": opt.flat_g, "exp_avg": opt.exp_avg, "exp_avg_sq": opt.exp_avg_sq,
            "step": opt.step_count, "rng": plan.rng_state, "slot.src": slot.src, "slot.logits": slot.logits}
    snap.update({"param." + k: p.detach() for k, p in model.named_parameters()})
    snap.update({"grad." + k: p.grad for k, p in model.named_parameters() if p.grad is not None})
    before = {k: v.clone() for k, v in snap.items()}
    model.eval()
    A.integrated_gradients(model, d["src"], d["static"], d["times"], d["lengths"], n_steps=8)
    torch.cuda.synchronize()
    for k, v in snap.items():
        assert torch.equal(v, before[k]), k
    assert slot.fwd_graph is not None and slot.bwd_graph is not None
    model.train()
    logits, _, _ = model.forward(d["src"], d["static"], d["times"], d["lengths"])      # the captured step still runs
    F.cross_entropy(logits, d["y"]).backward()
    opt.step()


@pytest.mark.gpu
def test_cuda_graph_capture():
    """A CUDA-graph capture of one call, replayed, reproduces the eager result."""
    cfg = model_config("P19", dropout=0.2)
    B = 8
    d = to_dev(make_batch(cfg, B, seed=11))
    model = _model(cfg, 5, 0)
    kw = dict(target=None, n_steps=10, internal_batch_size=4 * B, return_convergence_delta=True)
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eager = A.integrated_gradients(*args, **kw)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = A.integrated_gradients(*args, **kw)
    for t in out:
        t.zero_()
    g.replay()
    torch.cuda.synchronize()
    for x, y in zip(out, eager):
        assert torch.equal(x, y)
