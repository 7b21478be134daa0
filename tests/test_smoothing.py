"""Randomized smoothing of Raindrop_v2 (raindrop_b200.smoothing, rd_raindrop_v2_smooth_counts).

CPU: the exported symbols, the scratch query, the host argument checks, a numpy restatement of the noise stream and
Cohen's PREDICT / CERTIFY statistics against hand-computed scipy values.  GPU: the noisy inputs against the restatement,
the votes against the module's argmax on exactly those inputs, sigma = 0, chunking and key algebra, CUDA-graph replay,
certify / predict against the host statistics, and SmoothingTrainStep against TrainStep.  Every GPU test pins
plan.obprop_mode: the auto mode picks the ob-prop arithmetic from the row count."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from helpers import build_dropin, to_dev
from raindrop_b200 import smoothing as SM
from raindrop_b200.synth import make_batch, model_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXACT, FAST = 2, 1
SITE_SMOOTH = 100
SEED = 0x2B7E151628AED2A6
# name -> (config, B, make_batch options): the cases of the PGD tests
CASES = {
    "tiny_b6": ("TINY", 6, {}),
    "tiny8_b5": ("TINY8", 5, {}),                       # no statics
    "p19_b9": ("P19", 9, {"first_time_zero": True}),    # padded rows
    "p12_b3": ("P12", 3, {}),                           # T = 215
    "pam_b2": ("PAM", 2, {}),                           # T = 600
}


# ---- numpy restatement of the noise ----------------------------------------------------------------------------------
def _normals(seed, step, idx):
    """Box-Muller on the Philox block's word pairs at site 100, as rd_dp_add_noise: element i takes (x, y) for
    i & 3 in {0, 1}, (z, w) for {2, 3}, and the cos branch for even i."""
    from oracle.dropout_masks import philox4x32_10
    seed, step = int(seed), int(step) & 0xFFFFFFFFFFFFFFFF
    idx = np.asarray(idx, dtype=np.uint64)
    blk = idx >> np.uint64(2)
    ctr = np.stack([blk & np.uint64(0xFFFFFFFF), blk >> np.uint64(32), np.full_like(blk, SITE_SMOOTH),
                    np.full_like(blk, step & 0xFFFFFFFF)], -1)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) ^ (step >> 32)], dtype=np.uint64)
    w = philox4x32_10(ctr, key).astype(np.uint64)
    hi = (idx & np.uint64(2)) != 0
    a = np.where(hi, w[..., 2], w[..., 0])
    b = np.where(hi, w[..., 3], w[..., 1])
    u1 = ((a >> np.uint64(8)).astype(np.float64) + 1.0) / 16777216.0
    u2 = (b >> np.uint64(8)).astype(np.float64) / 16777216.0
    r, t = np.sqrt(-2.0 * np.log(u1)), 2.0 * np.pi * u2
    return np.where((idx & np.uint64(1)) != 0, r * np.sin(t), r * np.cos(t)).astype(np.float32)


def noisy_inputs(src, static, sigma, seed, step, sensors=None, perturb_static=False):
    """The replicate at key (seed, step): (src [T, B, 2N], static [B, ds] or None) with x + sigma z on S_b, z of element
    e of sample b at index b*(T*N + ds) + e (e = t*N + n, T*N + j for statics)."""
    src = np.asarray(src, dtype=np.float32)
    T, B, N2 = src.shape
    N = N2 // 2
    ds = 0 if static is None else np.asarray(static).shape[1]
    E = T * N + ds
    pert = src[:, :, N:] > 0
    if sensors is not None:
        pert &= np.asarray(sensors, dtype=bool)[None, None, :]
    idx = (np.arange(B)[None, :, None] * E + np.arange(T)[:, None, None] * N + np.arange(N)[None, None, :]).astype(np.uint64)
    d = np.float32(sigma) * _normals(seed, step, idx)
    x = src[:, :, :N]
    out = src.copy()
    out[:, :, :N] = np.where(pert & (d != 0), x + d, x)
    st = None
    if static is not None:
        st = np.asarray(static, dtype=np.float32).copy()
        if perturb_static:
            ids = (np.arange(B)[:, None] * E + T * N + np.arange(ds)[None, :]).astype(np.uint64)
            ds_ = np.float32(sigma) * _normals(seed, step, ids)
            st = np.where(ds_ != 0, st + ds_, st)
    return out, st


# ---- CPU --------------------------------------------------------------------------------------------------------------
def test_symbols_exported():
    lib_path = os.path.join(ROOT, "raindrop_b200", "csrc", "librd_b200.so")
    out = subprocess.run(["nm", "-D", "--defined-only", lib_path], capture_output=True, text=True, check=True).stdout
    names = {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert {"rd_smooth_scratch_bytes", "rd_raindrop_v2_smooth_counts", "rd_debug_smoothing_inputs"} <= names


def test_scratch_query():
    from raindrop_b200 import lib as L
    cfg = model_config("P19", dropout=0.2)
    model = build_dropin(cfg, 1, device="cpu")
    lib = L.load()
    dims = model._plan.dims(128, False)
    n1, n8 = lib.rd_smooth_scratch_bytes(C.byref(dims), 1), lib.rd_smooth_scratch_bytes(C.byref(dims), 8)
    assert 0 < n1 < n8
    assert lib.rd_smooth_scratch_bytes(C.byref(dims), 0) == 0


def _cpu_model():
    cfg = model_config("TINY", dropout=0.2)
    return build_dropin(cfg, 3, device="cpu").eval(), make_batch(cfg, 3, seed=1), cfg


def test_argument_validation():
    model, b, cfg = _cpu_model()
    args = (b["src"], b["static"], b["times"], b["lengths"])
    with pytest.raises(ValueError, match="eval"):
        SM.smooth_counts(model.train(), *args, sigma=0.1, n_samples=10)
    model.eval()
    bad = [dict(sigma=-0.1), dict(sigma=float("nan")), dict(sigma=float("inf")), dict(sigma=0.1, n_samples=0),
           dict(sigma=0.1, sensors=np.ones(cfg["d_inp"] + 1, bool)), dict(sigma=0.1, sensors=np.ones(cfg["d_inp"], np.int64)),
           dict(sigma=0.1, internal_batch_size=0), dict(sigma=0.1, seed=-1), dict(sigma=0.1, step=1 << 64),
           dict(sigma=0.1, step=(1 << 64) - 5)]
    for kw in bad:
        kw.setdefault("n_samples", 10)
        with pytest.raises(ValueError):
            SM.smooth_counts(model, *args, **kw)
    for alpha in (0.0, 1.0, -0.5, float("nan")):
        with pytest.raises(ValueError):
            SM.predict(model, *args, sigma=0.1, alpha=alpha)
        with pytest.raises(ValueError):
            SM.certify(model, *args, sigma=0.1, alpha=alpha)
        with pytest.raises(ValueError):
            SM.predict_from_counts(np.ones((2, 3), np.int64), alpha)
    for kw in (dict(n0=0), dict(n_samples=0)):
        with pytest.raises(ValueError):
            SM.certify(model, *args, sigma=0.1, **kw)
    with pytest.raises(ValueError):
        SM.certify_from_counts(np.ones((2, 3), np.int64), np.ones((2, 3), np.int64), -1.0)
    with pytest.raises(ValueError):
        SM.certify_from_counts(np.ones((2, 3), np.int64), np.ones((2, 2), np.int64), 0.1)
    with pytest.raises(ValueError):
        SM.certify_from_counts(np.ones((2, 3), np.int64), np.full((2, 3), 5, np.int64), 0.1, n=10)   # 15 votes > n
    with pytest.raises(ValueError):
        SM.predict_from_counts(np.array([[1.5, 2.0]]))
    cfg8 = model_config("TINY8", dropout=0.2)
    m8, b8 = build_dropin(cfg8, 3, device="cpu").eval(), make_batch(cfg8, 2, seed=1)
    with pytest.raises(ValueError, match="static"):
        SM.smooth_counts(m8, b8["src"], None, b8["times"], b8["lengths"], sigma=0.1, n_samples=4, perturb_static=True)


def test_no_cuda_raises(monkeypatch):
    from raindrop_b200.lib import RaindropB200Error
    model, b, _ = _cpu_model()
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RaindropB200Error):
        SM.smooth_counts(model, b["src"], b["static"], b["times"], b["lengths"], sigma=0.1, n_samples=4)


def test_train_step_refused(monkeypatch):
    import torch.distributed as dist
    from raindrop_b200.lib import RaindropB200Error
    cfg = model_config("TINY", dropout=0.2)
    model = build_dropin(cfg, 3, device="cpu")
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    with pytest.raises(RaindropB200Error, match="one GPU"):
        SM.SmoothingTrainStep(model, 4, sigma=0.1)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 1)
    with pytest.raises(ValueError):
        SM.SmoothingTrainStep(model, 4, sigma=-1.0)
    m8 = build_dropin(model_config("TINY8", dropout=0.2), 3, device="cpu")
    with pytest.raises(ValueError, match="static"):
        SM.SmoothingTrainStep(m8, 4, sigma=0.1, perturb_static=True)


@pytest.mark.parametrize("perturb_static", [False, True])
def test_noise_restatement(perturb_static):
    """The restated stream: standard normal on S_b, zero elsewhere, disjoint replicates under step + m."""
    cfg = model_config("P19", dropout=0.2)
    b = make_batch(cfg, 64, seed=4)
    N, sigma = cfg["d_inp"], 0.5
    sensors = np.arange(N) % 3 != 0
    x, st = b["src"].numpy(), b["static"].numpy()
    y, ys = noisy_inputs(x, st, sigma, SEED, 5, sensors, perturb_static)
    pert = (x[:, :, N:] > 0) & sensors
    assert pert.sum() > 1000
    assert np.array_equal(y[:, :, N:].view(np.int32), x[:, :, N:].view(np.int32))
    assert np.array_equal(y[:, :, :N][~pert].view(np.int32), x[:, :, :N][~pert].view(np.int32))
    z = (y[:, :, :N][pert].astype(np.float64) - x[:, :, :N][pert]) / sigma
    assert abs(z.mean()) < 0.05 and abs(z.var() - 1.0) < 0.05
    if perturb_static:
        zs = (ys.astype(np.float64) - st) / sigma
        assert abs(zs.mean()) < 0.1 and abs(zs.var() - 1.0) < 0.15
    else:
        assert np.array_equal(ys, st)
    y2, _ = noisy_inputs(x, st, sigma, SEED, 6, sensors, perturb_static)
    z2 = (y2[:, :, :N][pert].astype(np.float64) - x[:, :, :N][pert]) / sigma
    assert abs(np.corrcoef(z, z2)[0, 1]) < 0.05                   # replicate m + 1 is fresh noise
    y0, _ = noisy_inputs(x, st, 0.0, SEED, 5, sensors, perturb_static)
    assert np.array_equal(y0.view(np.int32), x.view(np.int32))


def test_predict_from_counts():
    from scipy.stats import binomtest
    counts = np.array([[90, 10, 0],       # clear winner
                       [50, 50, 0],       # tie between the top two: p = 1
                       [0, 0, 0],         # every vote invalid
                       [3, 7, 60],        # winner in the last class
                       [12, 2, 0],        # p-value close to alpha
                       [5, 5, 5]], dtype=np.int64)
    alpha = 0.01
    got = SM.predict_from_counts(counts, alpha)
    p4 = binomtest(12, 14, 0.5).pvalue                # 0.0129...
    assert p4 > alpha
    assert got.tolist() == [0, -1, -1, 2, -1, -1]
    assert SM.predict_from_counts(counts, 0.02).tolist() == [0, -1, -1, 2, 0, -1]
    assert binomtest(90, 100, 0.5).pvalue <= alpha
    assert SM.predict_from_counts(torch.tensor([[0, 9]]), 0.01).tolist() == [1]     # 2^-8 < 0.01
    assert SM.predict_from_counts(torch.tensor([[0, 6]]), 0.01).tolist() == [-1]    # 2^-5 > 0.01


def test_certify_from_counts():
    from scipy.stats import beta, norm
    sigma, alpha, n = 0.25, 0.001, 1000
    c0 = np.array([[100, 0], [0, 100], [60, 40], [100, 0], [50, 50], [10, 90]], dtype=np.int64)
    c = np.array([[1000, 0],              # k = n: p_lower = alpha^(1/n)
                  [1000, 0],              # c_A = 1 but k = 0: p_lower = 0, abstain
                  [700, 300],
                  [540, 458],             # two invalid votes: n = 1000 counts them against c_A
                  [600, 400],             # tie in the selection: c_A = 0
                  [0, 1000]], dtype=np.int64)
    pred, radius, pl = SM.certify_from_counts(c0, c, sigma, alpha, n=n)
    assert pl[0] == pytest.approx(alpha ** (1.0 / n), rel=1e-12)
    assert pl[1] == 0.0 and pred[1] == -1 and radius[1] == -1.0
    assert pl[2] == pytest.approx(beta.ppf(alpha, 700, 301), rel=1e-12)
    assert pl[3] == pytest.approx(beta.ppf(alpha, 540, 461), rel=1e-12)
    assert pred.tolist() == [0, -1, 0, -1, 0, 1]
    for b in (0, 2, 4, 5):
        assert radius[b] == pytest.approx(sigma * norm.ppf(pl[b]), rel=1e-12)
    assert pl[3] < 0.5 and radius[3] == -1.0
    # without n the row sums are the draws: the two invalid votes drop out
    _, _, pl_sum = SM.certify_from_counts(c0, c, sigma, alpha)
    assert pl_sum[3] == pytest.approx(beta.ppf(alpha, 540, 459), rel=1e-12) and pl_sum[3] > pl[3]
    # p_lower straddling 1/2: the smallest k with beta.ppf(alpha, k, n - k + 1) >= 1/2 certifies radius ~0
    ks = np.arange(n + 1)
    lo = np.where(ks > 0, beta.ppf(alpha, np.maximum(ks, 1), n - ks + 1), 0.0)
    k_star = int(np.argmax(lo >= 0.5))
    cc = np.array([[k_star - 1, n - k_star + 1], [k_star, n - k_star]], dtype=np.int64)
    pred, radius, pl = SM.certify_from_counts(np.array([[1, 0], [1, 0]]), cc, sigma, alpha)
    assert pl[0] < 0.5 <= pl[1]
    assert pred.tolist() == [-1, 0] and radius[0] == -1.0 and 0.0 <= radius[1] < 0.01 * sigma


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


def _inputs(model, d, sigma, seed, step, m0, nc, sensors=None, ps=False):
    """rd_debug_smoothing_inputs: replicates m0 .. m0+nc-1 at key (seed, step), replicate-major."""
    from raindrop_b200 import lib as L
    from raindrop_b200.adversarial import _sensor_mask
    lib, dev = L.load(), torch.device("cuda", torch.cuda.current_device())
    plan = model._prepare(dev)
    T, B, N2 = d["src"].shape
    dims = plan.dims(B, False)
    key = torch.tensor(np.array([seed, step], dtype=np.uint64).view(np.int64), device=dev)
    sens = _sensor_mask(sensors, N2 // 2, dev)
    src_e = torch.empty(T, nc * B, N2, device=dev)
    st_e = torch.empty(nc * B, d["static"].shape[1], device=dev) if d["static"] is not None else None
    tm_e = torch.empty(T, nc * B, device=dev)
    ln_e = torch.empty(nc * B, dtype=torch.int64, device=dev)
    L.check(lib.rd_debug_smoothing_inputs(C.byref(dims), d["src"].data_ptr(), L.ptr(d["static"]), d["times"].data_ptr(),
                                          d["lengths"].data_ptr(), L.ptr(sens), int(ps), sigma, key.data_ptr(), m0, nc,
                                          src_e.data_ptr(), L.ptr(st_e), tm_e.data_ptr(), ln_e.data_ptr(),
                                          L.stream_ptr(dev)),
            "rd_debug_smoothing_inputs")
    return src_e, st_e, tm_e, ln_e


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_noise_matches_restatement(name):
    cfg, d, model = _setup(name)
    N, B, sigma = cfg["d_inp"], d["src"].shape[1], 0.7
    sensors = torch.arange(N) % 4 != 1
    ps = d["static"] is not None
    m0, nc = 3, 2
    src_e, st_e, tm_e, ln_e = _inputs(model, d, sigma, SEED, 10, m0, nc, sensors, ps)
    x = d["src"].cpu().numpy()
    st = None if d["static"] is None else d["static"].cpu().numpy()
    pert = (x[:, :, N:] > 0) & sensors.numpy()
    for m in range(nc):
        rows = slice(m * B, (m + 1) * B)
        want, want_st = noisy_inputs(x, st, sigma, SEED, 10 + m0 + m, sensors.numpy(), ps)
        got = src_e[:, rows].cpu().numpy()
        assert np.array_equal(got[:, :, N:].view(np.int32), x[:, :, N:].view(np.int32))
        assert np.array_equal(got[:, :, :N][~pert].view(np.int32), x[:, :, :N][~pert].view(np.int32))
        ulp = np.spacing(np.abs(want[:, :, :N]).astype(np.float32))
        assert np.all(np.abs(got[:, :, :N] - want[:, :, :N]) <= 2 * ulp)
        assert not np.array_equal(got[:, :, :N][pert], x[:, :, :N][pert])
        assert torch.equal(tm_e[:, rows], d["times"]) and torch.equal(ln_e[rows], d["lengths"])
        if ps:
            gs = st_e[rows].cpu().numpy()
            assert np.all(np.abs(gs - want_st) <= 2 * np.spacing(np.abs(want_st).astype(np.float32)))
    # padded rows (time 0 after the first step: mask 0) stay the input bit for bit
    pad = (d["times"] == 0) & (torch.arange(cfg["max_len"], device="cuda")[:, None] > 0)
    assert pad.any() or name != "p19_b9"
    for m in range(nc):
        got = src_e[:, m * B:(m + 1) * B][pad]
        assert torch.equal(got.view(torch.int32), d["src"][pad].view(torch.int32))
    # the same replicate under another chunking: key (seed, step + m0) with m0 = 0
    again = _inputs(model, d, sigma, SEED, 10 + m0, 0, nc, sensors, ps)
    assert torch.equal(again[0], src_e)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_votes_are_module_argmax(name):
    """With one chunk of B*n rows, the counts are the bincount of torch.argmax of the module's eval forward on exactly
    the exported rows."""
    cfg, d, model = _setup(name)
    B, n, sigma = d["src"].shape[1], 6, 1.0
    ps = d["static"] is not None
    counts = SM.smooth_counts(model, *_args(d), sigma=sigma, n_samples=n, seed=SEED, step=2, perturb_static=ps,
                              internal_batch_size=B * n)
    src_e, st_e, tm_e, ln_e = _inputs(model, d, sigma, SEED, 2, 0, n, None, ps)
    with torch.no_grad():
        logits = model.forward(src_e, st_e, tm_e, ln_e)[0]
    assert torch.isfinite(logits).all()
    votes = logits.argmax(1).view(n, B)
    want = torch.zeros_like(counts)
    for b in range(B):
        want[b] = torch.bincount(votes[:, b], minlength=cfg["n_classes"])
    assert torch.equal(counts, want)
    assert torch.equal(counts.sum(1), torch.full((B,), n, device="cuda"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_zero_sigma_votes_the_clean_class(name):
    cfg, d, model = _setup(name)
    n = 5
    counts = SM.smooth_counts(model, *_args(d), sigma=0.0, n_samples=n, perturb_static=d["static"] is not None)
    with torch.no_grad():
        clean = model.forward(*_args(d))[0].argmax(1)
    want = torch.zeros_like(counts)
    want[torch.arange(len(clean)), clean] = n
    assert torch.equal(counts, want)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_chunking_key_algebra_graph_and_no_side_effects(name):
    cfg, d, model = _setup(name, FAST)
    B = d["src"].shape[1]
    n, a = 12, 5
    plan = model._prepare(torch.device("cuda"))
    snap = {"rng": plan.rng_state.clone()}
    snap.update({"param." + k: p.detach().clone() for k, p in model.named_parameters()})
    kw = dict(sigma=0.8, seed=SEED, perturb_static=d["static"] is not None)
    res = [SM.smooth_counts(model, *_args(d), n_samples=n, step=4, internal_batch_size=ib, **kw)
           for ib in (B, 7 * B, n * B, n * B)]
    for r in res[1:]:
        assert torch.equal(r, res[0])
    split = (SM.smooth_counts(model, *_args(d), n_samples=a, step=4, internal_batch_size=3 * B, **kw) +
             SM.smooth_counts(model, *_args(d), n_samples=n - a, step=4 + a, internal_batch_size=2 * B, **kw))
    assert torch.equal(split, res[0])
    # CUDA graph: capture after an eager call with the same key and shapes; a later eager call does not disturb it
    gkw = dict(n_samples=n, step=4, internal_batch_size=7 * B, **kw)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eager = SM.smooth_counts(model, *_args(d), **gkw)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = SM.smooth_counts(model, *_args(d), **gkw)
    SM.smooth_counts(model, *_args(d), n_samples=3, step=9, internal_batch_size=B, **kw)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager) and torch.equal(out, res[0])
    torch.cuda.synchronize()
    assert torch.equal(plan.rng_state, snap["rng"])
    for k, p in model.named_parameters():
        assert torch.equal(p.detach(), snap["param." + k]) and p.grad is None, k


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_certify_and_predict_match_host_statistics(name):
    cfg, d, model = _setup(name)
    sigma, n0, n, alpha = 0.5, 20, 200, 0.01
    ps = d["static"] is not None
    r = SM.certify(model, *_args(d), sigma=sigma, n0=n0, n_samples=n, alpha=alpha, seed=3, step=7, perturb_static=ps)
    c0 = SM.smooth_counts(model, *_args(d), sigma=sigma, n_samples=n0, seed=3, step=7, perturb_static=ps)
    c = SM.smooth_counts(model, *_args(d), sigma=sigma, n_samples=n, seed=3, step=7 + n0, perturb_static=ps)
    assert torch.equal(r.counts0, c0) and torch.equal(r.counts, c)
    pred, radius, pl = SM.certify_from_counts(c0, c, sigma, alpha, n=n)
    assert np.array_equal(r.prediction, pred) and np.array_equal(r.radius, radius) and np.array_equal(r.p_lower, pl)
    p = SM.predict(model, *_args(d), sigma=sigma, n_samples=n, alpha=alpha, seed=3, step=7, perturb_static=ps)
    cp = SM.smooth_counts(model, *_args(d), sigma=sigma, n_samples=n, seed=3, step=7, perturb_static=ps)
    assert np.array_equal(p, SM.predict_from_counts(cp, alpha))


@pytest.mark.gpu
def test_certify_small_sigma_certifies_the_clean_prediction():
    cfg, d, model = _setup("tiny_b6")
    with torch.no_grad():
        logits = model.forward(*_args(d))[0]
    top2 = logits.topk(2, dim=1).values
    sure = (top2[:, 0] - top2[:, 1] > 1e-2).cpu().numpy()
    assert sure.any()
    sigma = 1e-4
    r = SM.certify(model, *_args(d), sigma=sigma, n0=50, n_samples=500, alpha=0.001, seed=1)
    clean = logits.argmax(1).cpu().numpy()
    assert np.array_equal(r.prediction[sure], clean[sure])
    assert np.all(r.radius[sure] > 0) and np.all(r.radius[sure] <= sigma * 4)


# ---- Gaussian-augmentation training -----------------------------------------------------------------------------------
RNG0 = (0x1234ABCD5678, 11)


def _train_model(cfg, mode=EXACT):
    model = build_dropin(cfg, 21).train()
    plan = model._prepare(torch.device("cuda"))
    plan.obprop_mode = mode
    plan.rng_state.copy_(torch.tensor(RNG0, dtype=torch.int64))
    return model


def _run(step, n):
    losses = [step.step().clone() for _ in range(n)]
    torch.cuda.synchronize()
    return (step.flat_p.clone(), step.exp_avg.clone(), step.exp_avg_sq.clone(), torch.cat(losses),
            step.plan.rng_state.clone())


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
def test_smoothing_step_at_zero_sigma_is_train_step(use_graph):
    from raindrop_b200.train import TrainStep
    cfg = model_config("P19", dropout=0.2)
    B = 37
    batch = to_dev(make_batch(cfg, B, seed=5, first_time_zero=True))
    out = []
    for smooth in (False, True):
        model = _train_model(cfg)
        s = SM.SmoothingTrainStep(model, B, sigma=0.0, perturb_static=True, noise_seed=3, use_graph=use_graph) if smooth \
            else TrainStep(model, B, use_graph=use_graph)
        s.load_batch(batch)
        out.append(_run(s, 3))
    for a, b in zip(*out):
        assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("name", ["tiny_b6", "tiny8_b5"])
def test_smoothing_step_is_train_step_on_noisy_batch(use_graph, name):
    """One step from a given state equals TrainStep on the batch exported for the step's key; the key advances by one
    per step; restoring the state and the key replays the step."""
    from raindrop_b200.train import TrainStep
    cfg_name, B, _ = CASES[name]
    cfg = model_config(cfg_name, dropout=0.2)
    batch = to_dev(make_batch(cfg, B, seed=7))
    N, sigma = cfg["d_inp"], 0.3
    sensors = torch.arange(N) % 3 != 2
    ps = batch["static"] is not None
    model = _train_model(cfg)
    s = SM.SmoothingTrainStep(model, B, sigma=sigma, sensors=sensors, perturb_static=ps, noise_seed=SEED,
                              use_graph=use_graph, lr=1e-3)
    s.set_noise_key(SEED, 4)
    s.load_batch(batch)
    s.step()                                        # moves the parameters
    torch.cuda.synchronize()
    assert s.noise_key_state() == (SEED, 5)
    state = [t.clone() for t in s._state()]
    ref_model = _train_model(cfg)
    ref = TrainStep(ref_model, B, use_graph=False, lr=1e-3)
    ref.flat_p.copy_(s.flat_p); ref.exp_avg.copy_(s.exp_avg); ref.exp_avg_sq.copy_(s.exp_avg_sq)
    ref.step_count.copy_(s.step_count); ref.plan.rng_state.copy_(s.plan.rng_state)
    src_e, st_e, _, _ = _inputs(ref_model, batch, sigma, SEED, 5, 0, 1, sensors, ps)
    ref.load_batch(dict(batch, src=src_e, static=st_e))
    got = _run(s, 1)
    want = _run(ref, 1)
    for x, y in zip(got, want):
        assert torch.equal(x, y)
    assert torch.equal(s.noisy_src, src_e)
    assert not torch.equal(s.noisy_src, batch["src"])
    assert s.noise_key_state() == (SEED, 6)
    for t, v in zip(s._state(), state):
        t.copy_(v)
    s.set_noise_key(SEED, 5)
    again = _run(s, 1)
    for x, y in zip(got, again):
        assert torch.equal(x, y)
