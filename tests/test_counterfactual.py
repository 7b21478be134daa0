"""Counterfactual explanations of Raindrop_v2 (raindrop_b200.counterfactual, rd_raindrop_v2_counterfactual).

CPU: the exported symbols, the scratch query, the host argument checks, a numpy restatement of the restarts' start
points (Philox site 103) and the oracle's proximal step against its closed form.  GPU: identities, the invariants of the
returned points, bitwise agreement with the module forward, a float64 replay of FISTA (oracle/counterfactual_oracle.py),
the bisection against a host replay, restarts, chunking / repeat / CUDA-graph bitwise equality and side effects, and
usefulness at the defaults.  Every GPU test pins plan.obprop_mode: the auto mode picks the ob-prop arithmetic from the
row count."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from helpers import build_dropin, to_dev
from raindrop_b200 import counterfactual as CF
from raindrop_b200.synth import make_batch, model_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXACT, FAST = 2, 1
SEED = 0x2B7E151628AED2A6
# name -> (config, B, make_batch options)
CASES = {
    "tiny_b6": ("TINY", 6, {}),
    "tiny8_b5": ("TINY8", 5, {}),                       # 8 classes, no statics
    "p19_b9": ("P19", 9, {"first_time_zero": True}),    # padded rows
    "p12_b3": ("P12", 3, {}),                           # T = 215
    "pam_b2": ("PAM", 2, {}),                           # T = 600, C = 2400
}


# ---- CPU --------------------------------------------------------------------------------------------------------------
def test_symbols_exported():
    lib_path = os.path.join(ROOT, "raindrop_b200", "csrc", "librd_b200.so")
    out = subprocess.run(["nm", "-D", "--defined-only", lib_path], capture_output=True, text=True, check=True).stdout
    names = {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert {"rd_counterfactual_scratch_bytes", "rd_raindrop_v2_counterfactual"} <= names


def test_scratch_query():
    from raindrop_b200 import lib as L
    model = build_dropin(model_config("P19", dropout=0.2), 1, device="cpu")
    lib = L.load()
    dims = model._plan.dims(128, False)
    n1, n8, n8r3 = (lib.rd_counterfactual_scratch_bytes(C.byref(dims), s, r) for s, r in ((1, 1), (8, 1), (8, 3)))
    assert 0 < n1 < n8 < n8r3
    assert lib.rd_counterfactual_scratch_bytes(C.byref(dims), 0, 1) == 0
    assert lib.rd_counterfactual_scratch_bytes(C.byref(dims), 1, 0) == 0


def _cpu_model():
    cfg = model_config("TINY", dropout=0.2)
    return build_dropin(cfg, 3, device="cpu").eval(), make_batch(cfg, 3, seed=1), cfg


def test_argument_validation():
    model, b, cfg = _cpu_model()
    args = (b["src"], b["static"], b["times"], b["lengths"])
    N, ds = cfg["d_inp"], cfg["d_static"]
    with pytest.raises(ValueError, match="eval"):
        CF.counterfactual(model.train(), *args)
    model.eval()
    bad = [dict(kappa=-1.0), dict(beta=-0.1), dict(beta=float("nan")), dict(c_init=0.0), dict(step_size=0.0),
           dict(step_size=float("inf")), dict(init_scale=-1.0), dict(n_search=0), dict(n_steps=-1), dict(n_restarts=0),
           dict(weights=np.zeros(N)), dict(weights=-np.ones(N)), dict(weights=np.ones(N + 1)),
           dict(lower=np.ones(N), upper=np.zeros(N)), dict(lower=np.ones((2, N))), dict(upper=np.full(N, np.nan)),
           dict(sensors=np.ones(N + 1, bool)), dict(sensors=np.ones(N, np.int64)), dict(internal_batch_size=0),
           dict(seed=-1), dict(step=1 << 64), dict(target=cfg["n_classes"]), dict(target=torch.tensor([0, 1, 99]))]
    for kw in bad:
        with pytest.raises(ValueError):
            CF.counterfactual(model, *args, **kw)
    cfg8 = model_config("TINY8", dropout=0.2)
    m8, b8 = build_dropin(cfg8, 3, device="cpu").eval(), make_batch(cfg8, 2, seed=1)
    with pytest.raises(ValueError, match="static"):
        CF.counterfactual(m8, b8["src"], None, b8["times"], b8["lengths"], perturb_static=True)
    with pytest.raises(ValueError):                    # no statics: [d_inp + d_static] does not exist
        CF.counterfactual(m8, b8["src"], None, b8["times"], b8["lengths"], weights=np.ones(cfg8["d_inp"] + 1))
    w = CF._per_element(np.arange(1, N + ds + 1), "weights", N, ds, 1.0, positive=True)
    assert w.dtype == np.float32 and w[-1] == N + ds
    assert np.all(CF._per_element(2.0, "lower", N, ds, -np.inf) == 2.0)
    assert np.all(CF._per_element(np.zeros(N), "lower", N, ds, -np.inf)[N:] == -np.inf)


def test_no_cuda_raises(monkeypatch):
    from raindrop_b200.lib import RaindropB200Error
    model, b, _ = _cpu_model()
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RaindropB200Error):
        CF.counterfactual(model, b["src"], b["static"], b["times"], b["lengths"])


@pytest.mark.parametrize("perturb_static", [False, True])
def test_start_restatement(perturb_static):
    """The restated site-103 start: replica 0 is zero, only S_b moves, draws stay in the box and in init_scale, they look
    uniform, and the (seed, step) key changes them."""
    from oracle.counterfactual_oracle import start_deltas
    cfg = model_config("P19", dropout=0.2)
    b = make_batch(cfg, 48, seed=4)
    N, ds, s = cfg["d_inp"], cfg["d_static"], 0.5
    sensors = np.arange(N) % 3 != 0
    lower = np.full(N + ds, -0.3, np.float32)
    upper = np.full(N + ds, np.inf, np.float32)
    src, st = b["src"].numpy(), b["static"].numpy()
    d, dst = start_deltas(src, st, 3, s, SEED, 5, sensors, perturb_static, lower, upper)
    pert = (src[:, :, N:] > 0) & sensors
    assert np.all(d[0] == 0) and np.all(dst[0] == 0)
    assert np.all(d[:, ~pert] == 0) and pert.sum() > 100
    if not perturb_static:
        assert np.all(dst == 0)
    x = src[:, :, :N]
    v = d[1:][:, pert]
    xs = np.broadcast_to(x, d[1:].shape)[:, pert]
    assert np.all(np.abs(v) <= np.float32(s))
    assert np.all(xs + v >= np.minimum(-0.3, xs) - 1e-6)          # the box [min(lower, x), inf)
    free = xs > 0.3 + s                                              # cells the lower bound cannot reach
    vf = v[free]
    assert vf.size > 100 and vf.min() < -0.9 * s and vf.max() > 0.9 * s
    assert abs(float(vf.mean())) < 0.05 * s and abs(float((vf / s).var()) - 1.0 / 3.0) < 0.05
    d2, _ = start_deltas(src, st, 3, s, SEED, 6, sensors, perturb_static, lower, upper)
    assert not np.array_equal(d, d2)
    assert not np.array_equal(d[1], d[2])                           # replicas draw apart


def test_prox_step_closed_form():
    """1-D: the minimiser of (y - alpha g - z)^2 / (2 alpha) + beta w |z| over a box is the clipped soft-threshold."""
    from oracle.counterfactual_oracle import prox_step, soft_threshold
    alpha, beta, w = 0.1, 0.5, 2.0
    lam = alpha * beta * w
    z = torch.linspace(-3, 3, 60001, dtype=torch.float64)
    for y, g, lo, hi in ((0.3, -1.0, -1.0, 1.0), (0.3, 1.0, -1.0, 1.0), (0.05, 0.1, -1.0, 1.0), (2.0, -5.0, -1.0, 0.8),
                         (-0.5, 4.0, -0.6, 0.0)):
        v = y - alpha * g
        obj = (v - z) ** 2 / (2 * alpha) + beta * w * z.abs()
        obj[(z < lo) | (z > hi)] = float("inf")
        want = float(z[obj.argmin()])
        got, vv = prox_step(torch.tensor(y, dtype=torch.float64), torch.tensor(g, dtype=torch.float64), alpha, beta,
                            torch.tensor(w, dtype=torch.float64), torch.tensor(lo, dtype=torch.float64),
                            torch.tensor(hi, dtype=torch.float64))
        assert abs(float(got) - want) <= 1e-4 and float(vv) == pytest.approx(v)
        closed = min(max(np.sign(v) * max(abs(v) - lam, 0.0), lo), hi)
        assert float(got) == pytest.approx(closed, abs=1e-15)
    assert torch.equal(soft_threshold(torch.tensor([-0.1, 0.0, 0.1]), 0.1), torch.zeros(3))


def test_bisection_rule():
    from oracle.counterfactual_oracle import bisect
    c, lo, hi = 1.0, 0.0, float("inf")
    c, lo, hi = bisect(False, c, lo, hi)
    assert (c, lo, hi) == (10.0, 1.0, float("inf"))
    c, lo, hi = bisect(True, c, lo, hi)
    assert (c, lo, hi) == (5.5, 1.0, 10.0)
    c, lo, hi = bisect(False, c, lo, hi)
    assert (c, lo, hi) == (7.75, 5.5, 10.0)


# ---- GPU --------------------------------------------------------------------------------------------------------------
def _setup(name, mode=EXACT, wseed=9, dseed=3):
    cfg_name, B, opts = CASES[name]
    cfg = model_config(cfg_name, dropout=0.2)
    d = to_dev(make_batch(cfg, B, seed=dseed, **opts))
    model = build_dropin(cfg, wseed).eval()
    model._plan.obprop_mode = mode
    return cfg, d, model


def _args(d):
    return d["src"], d["static"], d["times"], d["lengths"]


def _bits(t):
    return t.view(torch.int32)


def _margin(logits, target):
    z = logits.double().clone()
    zt = z.gather(1, target[:, None])[:, 0]
    z.scatter_(1, target[:, None], -float("inf"))
    return zt - z.max(dim=1).values


# ---- 1. identity
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_identity(name):
    cfg, d, model = _setup(name)
    pred = None
    for K in (0, 3):
        r = CF.counterfactual(model, *_args(d), target=pred, n_steps=K, n_search=2, beta=0.1,
                              perturb_static=d["static"] is not None)
        pred = r.clean_logits.argmax(1) if pred is None else pred
        if K == 0:                                     # another target and no steps: invalid everywhere, x returned
            assert not r.valid.any() and torch.all(torch.isinf(r.distance))
            assert torch.equal(_bits(r.src), _bits(d["src"])) and torch.equal(r.logits, r.clean_logits)
            assert not r.round_valid.any()
            r = CF.counterfactual(model, *_args(d), target=pred, n_steps=0)
        assert r.valid.all() and torch.all(r.distance == 0), name
        assert torch.equal(_bits(r.src), _bits(d["src"])) and torch.equal(r.logits, r.clean_logits)
        assert torch.equal(r.target, pred) and r.round_valid.all()
        if d["static"] is not None:
            assert torch.equal(r.static, d["static"])
        assert torch.all(r.l0 == 0) and not r.sensors_changed.any()


# ---- 2. invariants
def _check_invariants(r, d, cfg, kappa, beta, weights, lower, upper, sensors, ps):
    N, ds = cfg["d_inp"], (cfg["d_static"] if d["static"] is not None else 0)
    x = d["src"]
    pert = x[:, :, N:] > 0
    if sensors is not None:
        pert = pert & sensors.cuda()
    assert torch.equal(_bits(r.src)[:, :, N:], _bits(x)[:, :, N:])
    assert torch.equal(_bits(r.src)[:, :, :N][~pert], _bits(x)[:, :, :N][~pert])
    w = torch.as_tensor(weights, dtype=torch.float32).cuda()
    lo = torch.as_tensor(lower, dtype=torch.float32).cuda()
    hi = torch.as_tensor(upper, dtype=torch.float32).cuda()
    v, xv = r.src[:, :, :N], x[:, :, :N]
    assert torch.all(v >= torch.minimum(lo[:N], xv)) and torch.all(v <= torch.maximum(hi[:N], xv))
    if d["static"] is not None:
        if ps:
            s, xs = r.static, d["static"]
            assert torch.all(s >= torch.minimum(lo[N:], xs)) and torch.all(s <= torch.maximum(hi[N:], xs))
        else:
            assert torch.equal(r.static, d["static"])
    m = _margin(r.logits, r.target)
    assert torch.equal(r.valid, (m > 0) & (m >= kappa))
    # distance from the returned input: delta there carries one fp32 rounding of x + delta per element
    dl = (v.double() - xv.double()) * w[:N].double()
    dist = float(beta) * dl.abs().sum(dim=(0, 2)) + (dl ** 2).sum(dim=(0, 2))
    slack = (torch.finfo(torch.float32).eps * (xv.double().abs() + (v.double() - xv.double()).abs())
             * w[:N].double()).sum(dim=(0, 2))
    if ps and d["static"] is not None:
        sl = (r.static.double() - d["static"].double()) * w[N:].double()
        dist = dist + float(beta) * sl.abs().sum(1) + (sl ** 2).sum(1)
        slack = slack + (torch.finfo(torch.float32).eps * (d["static"].double().abs() + sl.abs()) * w[N:].double()).sum(1)
    scale = 1.0 + float(beta) + 2 * (dl.abs().amax(dim=(0, 2)) if N else 0)
    ok = r.valid
    assert torch.all((dist[ok] - r.distance[ok]).abs() <= 4 * slack[ok] * scale[ok] + 1e-12), (dist, r.distance)
    inv = ~r.valid
    assert torch.all(torch.isinf(r.distance[inv]))
    assert torch.equal(_bits(r.src)[:, inv], _bits(x)[:, inv]) and torch.equal(r.logits[inv], r.clean_logits[inv])
    assert torch.allclose(r.l1[ok] * float(beta) + r.l2[ok] ** 2, r.distance[ok], rtol=1e-4, atol=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("kappa", [0.0, 0.05])
def test_invariants(name, kappa):
    cfg, d, model = _setup(name)
    N = cfg["d_inp"]
    ds = cfg["d_static"] if d["static"] is not None else 0
    ps = d["static"] is not None
    sensors = torch.arange(N) % 4 != 1
    g = np.random.default_rng(0)
    weights = g.uniform(0.5, 2.0, N + ds).astype(np.float32)
    lower = np.full(N + ds, -0.4, np.float32)
    upper = np.full(N + ds, 0.6, np.float32)
    r = CF.counterfactual(model, *_args(d), kappa=kappa, beta=0.05, step_size=0.1, c_init=100.0, n_search=2, n_steps=6,
                          n_restarts=2, init_scale=0.3, seed=SEED, step=3, sensors=sensors, perturb_static=ps,
                          weights=weights, lower=lower, upper=upper)
    _check_invariants(r, d, cfg, kappa, 0.05, weights, lower, upper, sensors, ps)
    assert torch.equal(r.sensors_changed[:, ~sensors.cuda()], torch.zeros_like(r.sensors_changed[:, ~sensors.cuda()]))


# ---- 3. module forward
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
def test_logits_are_module_forward(name, mode):
    """With one chunk of B rows, logits and clean_logits are bitwise the module's eval forward."""
    cfg, d, model = _setup(name, mode)
    B = d["src"].shape[1]
    r = CF.counterfactual(model, *_args(d), step_size=0.2, c_init=1000.0, beta=0.0, n_search=1, n_steps=4,
                          perturb_static=d["static"] is not None, internal_batch_size=B)
    with torch.no_grad():
        f = model.forward(r.src, r.static if r.static is not None else d["static"], d["times"], d["lengths"])[0]
        c = model.forward(*_args(d))[0]
    assert torch.equal(r.logits, f)
    assert torch.equal(r.clean_logits, c)


# ---- 4. oracle
def _oracle(cfg, wseed):
    from oracle.raindrop_oracle import build_oracle_model
    from raindrop_b200.synth import synth_weights
    o = build_oracle_model(cfg).eval()
    synth_weights(o, cfg, seed=wseed)
    return o.double()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("R", [1, 2])
@pytest.mark.parametrize("sparse", [False, True], ids=["beta0", "beta_box"])
def test_matches_oracle(name, R, sparse):
    from oracle import counterfactual_oracle as CO
    cfg, d, model = _setup(name, EXACT)
    N = cfg["d_inp"]
    ds = cfg["d_static"] if d["static"] is not None else 0
    ps = d["static"] is not None
    alpha, c0, K, init = 0.2, 1000.0, 4, 0.3
    beta = 0.002 if sparse else 0.0
    lower = np.full(N + ds, -6.0 if sparse else -np.inf, np.float32)      # binds on some of TINY8's cells
    upper = np.full(N + ds, 6.0 if sparse else np.inf, np.float32)
    kw = dict(kappa=0.0, beta=beta, c_init=c0, step_size=alpha, n_search=1, n_steps=K)
    r = CF.counterfactual(model, *_args(d), n_restarts=R, init_scale=init, seed=SEED, step=2, perturb_static=ps,
                          lower=lower, upper=upper, **kw)
    cpu = {k: (v.cpu() if v is not None else None) for k, v in d.items()}
    starts = CO.start_deltas(cpu["src"].numpy(), None if cpu["static"] is None else cpu["static"].numpy(), R, init, SEED,
                             2, None, ps, lower, upper)
    recs, _ = CO.search(_oracle(cfg, 9), cpu["src"], cpu["static"], cpu["times"], cpu["lengths"], r.target.cpu(),
                        n_restarts=R, starts=starts, lower=lower, upper=upper, perturb_static=ps, **kw)
    B = d["src"].shape[1]
    best = CO.best_points(recs, B)
    got = (r.src[:, :, :N].double() - d["src"][:, :, :N].double()).cpu()
    # PGD's tolerances, with the long-sequence attention path (T > 64: P12, PAM) held to 1e-2: each FISTA step moves delta
    # by alpha c = 200 times the input gradient, so that path's gradient error grows faster here than in PGD's
    # normalised steps (a float32 replay on the CPU stays within 1e-6 of the float64 one)
    tol = 1e-2 if cfg["max_len"] > 64 else 2e-3
    lam = alpha * beta
    checked = 0
    for b in range(B):
        ms = torch.stack([rec["m"][b] for rec in recs])
        if float(ms.abs().min()) < 1e-4:                         # a margin near the validity threshold
            continue
        ds_ = sorted(float(rec["d"][b]) for rec in recs if bool(rec["valid"][b]))
        if len(ds_) >= 2 and ds_[1] - ds_[0] < 1e-4 * (1 + ds_[0]):   # near-tie in the selection
            continue
        if best[b] < 0:
            assert not bool(r.valid[b]) and torch.equal(_bits(r.src[:, b]), _bits(d["src"][:, b])), b
            continue
        assert bool(r.valid[b]), b
        rec = recs[best[b]]
        ref = rec["delta"][:, b]
        assert float((got[:, b] - ref).abs().max()) <= tol * max(float(ref.abs().max()), 1e-12), (b, best[b])
        assert abs(float(r.distance[b]) - float(rec["d"][b])) <= tol * (1 + abs(float(rec["d"][b])))
        if ps:
            rs = rec["delta_static"][b]
            gs = (r.static[b].double() - d["static"][b].double()).cpu()
            assert float((gs - rs).abs().max()) <= tol * max(float(rs.abs().max()), 1e-12)
        if lam > 0:
            # the zero pattern, where the soft-threshold's inputs were farther from it than the returned delta may drift
            margin = 1e-3 * lam if cfg["max_len"] <= 64 else tol * float(ref.abs().max())
            far = rec["slack"][:, b] > margin
            assert torch.equal((got[:, b] == 0)[far], (ref == 0)[far]), b
        checked += 1
    print(name, R, sparse, "samples checked against the oracle:", checked, "of", B)
    assert checked >= 1


# ---- 5. bisection
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny_b6", "tiny8_b5", "p19_b9"])
def test_bisection_replay(name):
    from oracle.counterfactual_oracle import bisect
    cfg, d, model = _setup(name)
    c_init, S = 3.0, 5
    r = CF.counterfactual(model, *_args(d), c_init=c_init, step_size=0.2, n_search=S, n_steps=3, n_restarts=2, seed=1)
    rv = r.round_valid.cpu().numpy()
    got = r.c.cpu().numpy()
    assert rv.shape == (d["src"].shape[1], 2, S)
    for b in range(rv.shape[0]):
        for k in range(2):
            c, lo, hi = c_init, 0.0, float("inf")
            for s in range(S):
                c, lo, hi = bisect(bool(rv[b, k, s]), c, lo, hi)
            assert got[b, k] == c, (b, k, got[b, k], c)
    # a sample is valid iff some round of some replica found a valid point
    assert torch.equal(r.valid, r.round_valid.flatten(1).any(1))


# ---- 6. restarts
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_restarts(name):
    cfg, d, model = _setup(name)
    kw = dict(step_size=0.2, c_init=100.0, beta=0.05, n_search=2, n_steps=4, seed=SEED, step=1,
              perturb_static=d["static"] is not None)
    r1 = CF.counterfactual(model, *_args(d), n_restarts=1, **kw)
    r3 = CF.counterfactual(model, *_args(d), n_restarts=3, **kw)
    assert torch.all(r3.valid[r1.valid])
    assert torch.all(r3.distance[r1.valid] <= r1.distance[r1.valid])
    # replica 0 is the one-replica search
    assert torch.equal(r3.c[:, :1], r1.c) and torch.equal(r3.round_valid[:, :1], r1.round_valid)
    assert torch.equal(r3.clean_logits, r1.clean_logits) and torch.equal(r3.target, r1.target)


# ---- 7. repeatability
@pytest.mark.gpu
def test_chunking_repeat_graph_bitwise_and_no_side_effects():
    cfg, d, model = _setup("p19_b9", FAST)
    B = d["src"].shape[1]
    plan = model._prepare(torch.device("cuda"))
    snap = {"rng": plan.rng_state.clone()}
    snap.update({"param." + k: p.detach().clone() for k, p in model.named_parameters()})
    cpu_rng = torch.get_rng_state()
    cuda_rng = torch.cuda.get_rng_state()
    kw = dict(step_size=0.2, c_init=50.0, beta=0.05, n_search=2, n_steps=3, n_restarts=2, seed=5, step=2,
              perturb_static=True, lower=-2.0, upper=2.0)
    fields = ("src", "static", "logits", "clean_logits", "target", "valid", "distance", "c", "round_valid", "l1", "l2",
              "l0", "sensors_changed")
    res = [CF.counterfactual(model, *_args(d), internal_batch_size=ib, **kw) for ib in (1, 7, B, B)]
    for r in res[1:]:
        for f in fields:
            assert torch.equal(getattr(r, f), getattr(res[0], f)), f
    # a CUDA-graph capture of the call, replayed
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        CF.counterfactual(model, *_args(d), internal_batch_size=B, **kw)
    torch.cuda.current_stream().wait_stream(st)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        rg = CF.counterfactual(model, *_args(d), internal_batch_size=B, **kw)
    for t in (rg.src, rg.logits, rg.distance, rg.c):
        t.fill_(0)
    graph.replay()
    torch.cuda.synchronize()
    for f in fields:
        assert torch.equal(getattr(rg, f), getattr(res[0], f)), f
    assert torch.equal(plan.rng_state, snap["rng"])
    for k, p in model.named_parameters():
        assert torch.equal(p.detach(), snap["param." + k]) and p.grad is None, k
    assert torch.equal(torch.get_rng_state(), cpu_rng) and torch.equal(torch.cuda.get_rng_state(), cuda_rng)
    # the default target is the runner-up
    z = res[0].clean_logits.clone()
    z.scatter_(1, z.argmax(1, keepdim=True), -float("inf"))
    assert torch.equal(res[0].target, z.argmax(1))


# ---- 8. usefulness
@pytest.mark.gpu
def test_defaults_find_counterfactuals_on_p19():
    cfg = model_config("P19", dropout=0.2)
    d = to_dev(make_batch(cfg, 64, seed=11))
    model = build_dropin(cfg, 9).eval()
    model._plan.obprop_mode = FAST
    r = CF.counterfactual(model, *_args(d), n_restarts=2, seed=1)
    N, ds = cfg["d_inp"], cfg["d_static"]
    _check_invariants(r, d, cfg, 0.0, 0.1, np.ones(N + ds, np.float32), np.full(N + ds, -np.inf, np.float32),
                      np.full(N + ds, np.inf, np.float32), None, False)
    rate = float(r.valid.float().mean())
    print("P19 synthetic, defaults with 2 restarts: validity rate %.3f, median L0 %s" %
          (rate, r.l0[r.valid].median().item() if r.valid.any() else None))
    assert r.valid.any()
    # every valid result is independently valid under the module forward
    with torch.no_grad():
        f = model.forward(r.src, d["static"], d["times"], d["lengths"])[0]
    m = _margin(f, r.target)
    assert torch.all(m[r.valid] > 0)
