"""Early prediction of Raindrop_v2 (raindrop_b200.early, rd_raindrop_v2_prefix_logits).

CPU: the exported symbols, the scratch query, the host argument checks, a numpy restatement of the cutoffs (by row,
by horizon, and the training draws at Philox site 104: pinned values, bounds, uniformity), and first_alarm /
horizon_metrics against hand cases and scipy.  GPU: the cutoffs, prefix lengths and truncated rows against the
restatement, the logits against the module's eval forward on torch-truncated copies (bitwise, per chunk), the full
prefix against the plain forward, chunking, repeat calls and CUDA-graph replay without side effects, the large scratch
plans, the training draws, and PrefixTrainStep against TrainStep.  Every GPU test pins plan.obprop_mode: the auto mode
picks the ob-prop arithmetic from the row count."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch

from helpers import build_dropin, to_dev
from raindrop_b200 import early as EP
from raindrop_b200.synth import make_batch, model_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXACT, FAST = 2, 1
SITE_PREFIX = 104
SEED = 0x2B7E151628AED2A6
PINNED_DRAWS = [60, 22, 38, 60, 60, 60, 6, 60]     # slots 0 .. 7 of the P19 draws at (SEED, 7) below
CASES = {
    "tiny_b6": ("TINY", 6, {}),
    "tiny8_b5": ("TINY8", 5, {}),                       # no statics, 8 classes
    "p19_b9": ("P19", 9, {"first_time_zero": True}),    # padded rows, first time 0
    "p12_b3": ("P12", 3, {}),                           # T = 215
    "pam_b2": ("PAM", 2, {}),                           # T = 600
}


# ---- numpy restatement ------------------------------------------------------------------------------------------------
def prefix_lengths(times, lengths, r):
    """The lengths of cutoffs r [..., B] of records times [T, B], lengths [B]."""
    times, lengths, r = np.asarray(times), np.asarray(lengths, np.int64), np.asarray(r, np.int64)
    T = times.shape[0]
    seen = np.concatenate([np.zeros((1, times.shape[1]), np.int64), np.cumsum(times > 0, axis=0)])
    cnt = np.take_along_axis(seen, np.minimum(r, T).reshape(-1, times.shape[1]), axis=0).reshape(r.shape)
    return np.where(r >= T, lengths, np.minimum(lengths, cnt))


def row_cutoffs(rows, B, T):
    return np.repeat(np.clip(np.asarray(rows, np.int64), 0, T)[:, None], B, axis=1)


def horizon_cutoffs(times, horizons):
    """r[k, b] = the leading rows of sample b with times <= h_k (float32 comparisons)."""
    times = np.asarray(times, np.float32)
    T, B = times.shape
    out = np.zeros((len(horizons), B), np.int64)
    for k, h in enumerate(np.asarray(horizons, np.float32)):
        le = times <= h
        out[k] = np.where(le.all(axis=0), T, np.argmin(le, axis=0))
    return out


def _words(seed, step, b, j0, n):
    """Words j0 .. j0+n-1 (j0 % 4 == 0) of slot b's stream at key (seed, step), site 104: index (b << 32) + j, word
    index & 3 of the Philox block at counter index >> 2."""
    from oracle.dropout_masks import philox4x32_10
    seed, step = int(seed), int(step) & 0xFFFFFFFFFFFFFFFF
    blk = np.uint64((int(b) << 30) + j0 // 4) + np.arange((n + 3) // 4, dtype=np.uint64)
    ctr = np.stack([blk & np.uint64(0xFFFFFFFF), blk >> np.uint64(32), np.full_like(blk, SITE_PREFIX),
                    np.full_like(blk, step & 0xFFFFFFFF)], -1)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) ^ (step >> 32)], dtype=np.uint64)
    return [int(w) for w in philox4x32_10(ctr, key).reshape(-1)[:n]]


def drawn_cutoffs(times, seed, step, p_full, min_fraction, rows=None):
    """The training cutoffs [B] of rd_debug_prefix_inputs with rng = (seed, step)."""
    times = np.asarray(times, np.float32)
    T, B = times.shape
    out = np.empty(B, np.int64)
    for b in range(B):
        if rows is not None and rows[b] >= 0:
            out[b] = min(int(rows[b]), T)
            continue
        obs = np.flatnonzero(times[:, b] > 0)
        if obs.size == 0:
            out[b] = T
            continue
        R, f = int(obs[-1]) + 1, int(obs[0])
        words = iter(_words(seed, step, b, 0, 64))
        if next(words) < math.floor(p_full * 2.0 ** 32):
            out[b] = T
            continue
        lo = max(f + 1, math.ceil(min_fraction * R))
        r = R - lo + 1                                  # Lemire's bounded integer in [0, r)
        x = next(words) * r
        if x & 0xFFFFFFFF < r:
            t = ((1 << 32) - r) % r
            while x & 0xFFFFFFFF < t:
                x = next(words) * r
        out[b] = lo + (x >> 32)
    return out


# ---- CPU --------------------------------------------------------------------------------------------------------------
def test_symbols_exported():
    lib_path = os.path.join(ROOT, "raindrop_b200", "csrc", "librd_b200.so")
    out = subprocess.run(["nm", "-D", "--defined-only", lib_path], capture_output=True, text=True, check=True).stdout
    names = {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert {"rd_prefix_scratch_bytes", "rd_raindrop_v2_prefix_logits", "rd_debug_prefix_inputs"} <= names


def test_scratch_query():
    from raindrop_b200 import lib as L
    cfg = model_config("P19", dropout=0.2)
    model = build_dropin(cfg, 1, device="cpu")
    lib = L.load()
    dims = model._plan.dims(128, False)
    sizes = [lib.rd_prefix_scratch_bytes(C.byref(dims), k) for k in (1, 2, 5, 12, 60)]
    assert 0 < sizes[0] and all(a < b for a, b in zip(sizes, sizes[1:]))
    assert lib.rd_prefix_scratch_bytes(C.byref(dims), 0) == 0
    assert lib.rd_prefix_scratch_bytes(C.byref(dims), -3) == 0
    assert lib.rd_prefix_scratch_bytes(C.byref(dims), 1 << 30) == 0        # B * chunk > 2^30 rows


def _cpu_model():
    cfg = model_config("TINY", dropout=0.2)
    return build_dropin(cfg, 3, device="cpu").eval(), make_batch(cfg, 3, seed=1), cfg


def test_argument_validation():
    model, b, cfg = _cpu_model()
    T = cfg["max_len"]
    args = (b["src"], b["static"], b["times"], b["lengths"])
    with pytest.raises(ValueError, match="eval"):
        EP.prefix_predict(model.train(), *args)
    model.eval()
    bad = [dict(horizons=[1.0], rows=[1]), dict(horizons=[1.0, float("nan")]), dict(horizons=[]), dict(rows=[]),
           dict(rows=[0, T + 1]), dict(rows=[-1]), dict(rows=[1.5]), dict(rows=[[1, 2]]), dict(horizons=[True]),
           dict(internal_batch_size=0)]
    for kw in bad:
        with pytest.raises(ValueError):
            EP.prefix_predict(model, *args, **kw)
    assert EP._check_prefixes([float("-inf"), 0, float("inf")], None, T)[0] == "horizons"     # +-inf are allowed
    kind, v = EP._check_prefixes(None, None, T)
    assert kind == "rows" and v.tolist() == list(range(1, T + 1))
    res = EP.PrefixResult(torch.zeros(2, 3, 2), None, None)
    for cls in (2, -1, 1.0, True):
        with pytest.raises(ValueError):
            EP.first_alarm(res, 0.5, cls=cls)
    with pytest.raises(ValueError):
        EP.first_alarm(res, float("nan"))
    with pytest.raises(ValueError):
        EP.horizon_metrics(res, [1, 1])                 # no negatives
    with pytest.raises(ValueError):
        EP.horizon_metrics(res, [0, 1, 1])              # 3 labels for 2 samples


def test_no_cuda_raises(monkeypatch):
    from raindrop_b200.lib import RaindropB200Error
    model, b, _ = _cpu_model()
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RaindropB200Error):
        EP.prefix_predict(model, b["src"], b["static"], b["times"], b["lengths"], rows=[1, 2])


def test_train_step_refused(monkeypatch):
    import torch.distributed as dist
    from raindrop_b200.lib import RaindropB200Error
    cfg = model_config("TINY", dropout=0.2)
    model = build_dropin(cfg, 3, device="cpu")
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    with pytest.raises(RaindropB200Error, match="one GPU"):
        EP.PrefixTrainStep(model, 4)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 1)
    for kw in (dict(p_full=1.5), dict(p_full=float("nan")), dict(min_fraction=-0.1)):
        with pytest.raises(ValueError):
            EP.PrefixTrainStep(model, 4, **kw)


def test_cutoff_restatement_hand_case():
    #                t=0  1    2    3    4        sample 0 sorted, 1 padded after row 2, 2 starts at time 0, 3 unsorted
    times = np.array([[1., 0., 0., 5.],
                      [2., 1., 1., 1.],
                      [3., 2., 2., 2.],
                      [4., 0., 3., 9.],
                      [5., 0., 4., 3.]], np.float32)
    lengths = (times > 0).sum(0)
    hz = horizon_cutoffs(times, [-np.inf, 0.0, 2.0, 4.0, np.inf])
    assert hz.tolist() == [[0, 0, 0, 0], [0, 1, 1, 0], [2, 5, 3, 0], [4, 5, 5, 0], [5, 5, 5, 5]]
    assert prefix_lengths(times, lengths, hz).tolist() == [[0, 0, 0, 0], [0, 0, 0, 0], [2, 2, 2, 0], [4, 2, 4, 0],
                                                           [5, 2, 4, 5]]
    assert row_cutoffs([0, 3, 9], 2, 5).tolist() == [[0, 0], [3, 3], [5, 5]]


def test_drawn_cutoffs_restatement():
    """Pinned draws, lo_b <= r <= R_b, p_full at its ends, caller rows, and a chi-square test of uniformity."""
    from scipy.stats import chisquare
    cfg = model_config("P19", dropout=0.2)
    b = make_batch(cfg, 64, seed=4, first_time_zero=True)
    times = b["times"].numpy()
    T = times.shape[0]
    r = drawn_cutoffs(times, SEED, 7, 0.5, 0.25)
    assert r[:8].tolist() == PINNED_DRAWS
    full = r == T
    assert 10 < full.sum() < 54
    for bb in np.flatnonzero(~full):
        obs = np.flatnonzero(times[:, bb] > 0)
        R, f = obs[-1] + 1, obs[0]
        assert max(f + 1, math.ceil(0.25 * R)) <= r[bb] <= R
    assert prefix_lengths(times, b["lengths"].numpy(), r).min() >= 1
    assert (drawn_cutoffs(times, SEED, 7, 1.0, 0.25) == T).all()
    assert not (drawn_cutoffs(times, SEED, 7, 0.0, 0.25) == T).any()
    rows = np.where(np.arange(64) % 3 == 0, np.arange(64) % 7, -1)
    rr = drawn_cutoffs(times, SEED, 7, 0.5, 0.25, rows)
    assert np.array_equal(rr[rows >= 0], rows[rows >= 0]) and np.array_equal(rr[rows < 0], r[rows < 0])
    # one record observed on rows 2 .. 11 (R = 12, f = 2), min_fraction 0: r uniform on 3 .. 12
    tm = np.zeros((20, 1), np.float32)
    tm[2:12, 0] = np.arange(1, 11)
    draws = np.array([drawn_cutoffs(tm, SEED, s, 0.0, 0.0)[0] for s in range(3000)])
    assert draws.min() == 3 and draws.max() == 12
    assert chisquare(np.bincount(draws - 3, minlength=10)).pvalue > 1e-3



def _result(p):
    """A PrefixResult of two-class logits whose softmax P(class 1) is p [B, K]."""
    p = np.asarray(p, np.float64)
    return EP.PrefixResult(torch.from_numpy(np.stack([np.zeros_like(p), np.log(p) - np.log1p(-p)], -1)), None, None)


def test_first_alarm():
    res = _result([[0.1, 0.4, 0.6, 0.9],        # fires at k = 2
                   [0.7, 0.2, 0.1, 0.8],        # at once
                   [0.1, 0.2, 0.3, 0.4],        # never
                   [0.5, 0.5, 0.5, 0.5]])       # logit 0: exactly 1/2
    assert EP.first_alarm(res, 0.55).tolist() == [2, 0, -1, -1]
    assert EP.first_alarm(res, 0.35).tolist() == [1, 0, 3, 0]
    assert EP.first_alarm(res, 0.0).tolist() == [0, 0, 0, 0]
    assert EP.first_alarm(res, 0.95).tolist() == [-1, -1, -1, -1]
    assert EP.first_alarm(res, 0.65, cls=0).tolist() == [0, 1, 0, -1]       # P(class 0) = 1 - p


def test_horizon_metrics_against_scipy():
    from scipy.stats import mannwhitneyu
    rng = np.random.default_rng(5)
    B, K = 40, 3
    y = np.arange(B) % 2
    p = np.empty((B, K))
    p[:, 0] = 0.5                                                      # every score tied: AUROC 1/2, AUPRC = prevalence
    p[:, 1] = np.clip(0.3 + 0.3 * y + 0.2 * rng.standard_normal(B), 0.01, 0.99)
    p[:, 2] = np.where(y == 1, 0.9, 0.1)                               # separated: 1, 1
    m = EP.horizon_metrics(_result(p), torch.tensor(y))
    assert m["auroc"][0] == 0.5 and m["auprc"][0] == pytest.approx(0.5, abs=1e-15)
    assert m["auroc"][2] == 1.0 and m["auprc"][2] == 1.0
    q = torch.softmax(_result(p).logits, 2)[:, 1, 1].numpy()
    u = mannwhitneyu(q[y == 1], q[y == 0]).statistic
    assert m["auroc"][1] == pytest.approx(u / (20 * 20), rel=1e-12)
    # average precision by its definition: mean over the positives of the precision at their rank (no ties here)
    order = np.argsort(-q)
    hits = np.cumsum(y[order])
    ap = np.mean((hits / np.arange(1, B + 1))[y[order] == 1])
    assert m["auprc"][1] == pytest.approx(ap, rel=1e-12)
    # class 0 as the positives: the mirrored ranking
    m0 = EP.horizon_metrics(_result(p), y, cls=0)
    assert m0["auroc"][1] == pytest.approx(m["auroc"][1], rel=1e-12)


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


def truncated(d, r):
    """The batch cut at cutoffs r [B] in torch: (src, static, times, lengths)."""
    T = d["src"].shape[0]
    r = torch.as_tensor(r, device=d["src"].device)
    keep = torch.arange(T, device=r.device)[:, None] < r[None, :]
    src = torch.where(keep[:, :, None], d["src"], 0.0)
    times = torch.where(keep, d["times"], 0.0)
    cnt = ((d["times"] > 0) & keep).sum(0)
    lengths = torch.where(r >= T, d["lengths"], torch.minimum(d["lengths"], cnt))
    return src, d["static"], times, lengths


def _cat(parts):
    src, st, tm, ln = zip(*parts)
    return (torch.cat(src, 1), None if st[0] is None else torch.cat(st, 0), torch.cat(tm, 1), torch.cat(ln, 0))


def _prefix_table(cfg, d):
    """Rows through the record (0, 1, a middle, T - 1, T) and horizons with ties at observed times."""
    T = cfg["max_len"]
    rows = [0, 1, T // 3, T - 1, T]
    tm = d["times"][:, 0].cpu().numpy()
    obs = tm[tm > 0]
    horizons = [float("-inf"), 0.0, float(obs[0]), float(obs[len(obs) // 2]), float(obs[-1]) + 0.5, float("inf")]
    return rows, horizons


def _debug_inputs(model, d, horizons=None, rows=None, K=None, key=None, p_full=0.5, min_fraction=0.25):
    from raindrop_b200 import lib as L
    lib, dev = L.load(), d["src"].device
    plan = model._prepare(dev)
    T, B, N2 = d["src"].shape
    dims = plan.dims(B, False)
    hz = None if horizons is None else torch.tensor(horizons, dtype=torch.float32, device=dev)
    rw = None if rows is None else torch.as_tensor(rows, dtype=torch.int32).to(dev)
    K = K or len(horizons if horizons is not None else rows)
    kt = None if key is None else torch.tensor(np.array(key, dtype=np.uint64).view(np.int64), device=dev)
    cut = torch.empty(K, B, dtype=torch.int32, device=dev)
    src_e = torch.empty(T, K * B, N2, device=dev)
    st_e = torch.empty(K * B, d["static"].shape[1], device=dev) if d["static"] is not None else None
    tm_e = torch.empty(T, K * B, device=dev)
    ln_e = torch.empty(K * B, dtype=torch.int64, device=dev)
    L.check(lib.rd_debug_prefix_inputs(C.byref(dims), d["src"].data_ptr(), L.ptr(d["static"]), d["times"].data_ptr(),
                                       d["lengths"].data_ptr(), L.ptr(hz), L.ptr(rw), K, L.ptr(kt), p_full, min_fraction,
                                       cut.data_ptr(), src_e.data_ptr(), L.ptr(st_e), tm_e.data_ptr(), ln_e.data_ptr(),
                                       L.stream_ptr(dev)),
            "rd_debug_prefix_inputs")
    return cut, (src_e, st_e, tm_e, ln_e)


def _check_rows(d, cut, ex):
    """The exported prefix-major rows are the torch truncation at each row of cut, bit for bit."""
    B = d["src"].shape[1]
    for k in range(cut.shape[0]):
        want = truncated(d, cut[k].long())
        rows = slice(k * B, (k + 1) * B)
        assert torch.equal(ex[0][:, rows].view(torch.int32), want[0].view(torch.int32))
        assert torch.equal(ex[2][:, rows].view(torch.int32), want[2].view(torch.int32))
        assert torch.equal(ex[3][rows], want[3])
        if want[1] is not None:
            assert torch.equal(ex[1][rows], want[1])


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_cutoffs_match_restatement(name):
    cfg, d, model = _setup(name)
    T, B = cfg["max_len"], d["src"].shape[1]
    rows, horizons = _prefix_table(cfg, d)
    tm, ln = d["times"].cpu().numpy(), d["lengths"].cpu().numpy()
    for kw, want in ((dict(rows=rows), row_cutoffs(rows, B, T)), (dict(horizons=horizons), horizon_cutoffs(tm, horizons))):
        cut, ex = _debug_inputs(model, d, **kw)
        assert np.array_equal(cut.cpu().numpy(), want)
        assert np.array_equal(ex[3].view(-1, B).cpu().numpy(), prefix_lengths(tm, ln, want))
        _check_rows(d, cut, ex)
        res = EP.prefix_predict(model, *_args(d), **kw)
        assert np.array_equal(res.cutoffs.cpu().numpy(), want.T)
        assert np.array_equal(res.lengths.cpu().numpy(), prefix_lengths(tm, ln, want).T)
    if name == "p19_b9":          # the first time is 0: row 0 counts toward no length
        assert (d["times"][0] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_logits_are_module_forward_per_chunk(name):
    """Chunk by chunk, the logits are bitwise the module's eval forward on the concatenation of the chunk's
    torch-truncated copies: one prefix (B rows) per chunk, and three prefixes per chunk with a ragged last chunk."""
    cfg, d, model = _setup(name)
    B, T = d["src"].shape[1], cfg["max_len"]
    rows = [0, 2, T // 2, T - 1, T, 1, T // 4]
    for kc in (1, 3):
        res = EP.prefix_predict(model, *_args(d), rows=rows, internal_batch_size=kc * B)
        assert torch.isfinite(res.logits).all()
        for k0 in range(0, len(rows), kc):
            ks = range(k0, min(len(rows), k0 + kc))
            with torch.no_grad():
                want = model.forward(*_cat([truncated(d, torch.full((B,), rows[k], device="cuda")) for k in ks]))[0]
            got = torch.cat([res.logits[:, k] for k in ks], 0)
            assert torch.equal(got, want), (kc, k0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_full_prefix_is_plain_forward(name):
    cfg, d, model = _setup(name)
    with torch.no_grad():
        want = model.forward(*_args(d))[0]
    for kw in (dict(rows=[cfg["max_len"]]), dict(horizons=[float("inf")])):
        res = EP.prefix_predict(model, *_args(d), **kw)
        assert torch.equal(res.logits[:, 0], want)
        assert torch.equal(res.lengths[:, 0], d["lengths"])


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_chunking_repeat_graph_and_no_side_effects(name):
    cfg, d, model = _setup(name, FAST)
    B, T = d["src"].shape[1], cfg["max_len"]
    plan = model._prepare(torch.device("cuda"))
    snap = {"rng": plan.rng_state.clone()}
    snap.update({"param." + k: p.detach().clone() for k, p in model.named_parameters()})
    hz = torch.tensor([0.5, 2.0, 8.0, float("inf"), -1.0], device="cuda")
    res = [EP.prefix_predict(model, *_args(d), horizons=hz, internal_batch_size=ib) for ib in (B, 2 * B, 5 * B, None)]
    res.append(EP.prefix_predict(model, *_args(d), horizons=hz))
    for r in res[1:]:
        assert torch.equal(r.logits, res[0].logits) and torch.equal(r.cutoffs, res[0].cutoffs)
        assert torch.equal(r.lengths, res[0].lengths)
    every = EP.prefix_predict(model, *_args(d), internal_batch_size=7 * B)          # every row count 1 .. T
    assert every.logits.shape == (B, T, cfg["n_classes"])
    assert torch.equal(every.cutoffs, torch.arange(1, T + 1, device="cuda", dtype=torch.int32).expand(B, T))
    # CUDA graph: capture after an eager call with the same prefixes and shapes; a later eager call does not disturb it
    gkw = dict(horizons=hz, internal_batch_size=2 * B)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        EP.prefix_predict(model, *_args(d), **gkw)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = EP.prefix_predict(model, *_args(d), **gkw)
    EP.prefix_predict(model, *_args(d), rows=[1, 2, 3], internal_batch_size=B)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out.logits, res[0].logits) and torch.equal(out.cutoffs, res[0].cutoffs)
        assert torch.equal(out.lengths, res[0].lengths)
    assert torch.equal(plan.rng_state, snap["rng"])
    for k, p in model.named_parameters():
        assert torch.equal(p.detach(), snap["param." + k]) and p.grad is None, k


@pytest.mark.gpu
def test_no_side_effects_on_a_trained_model():
    """Parameters, their .grad, the dropout rng state and a bound FlatAdam (moments, step count, captured slots) are
    untouched by prefix_predict."""
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
    plan = model._plan
    slot = next(iter(plan._slots.values()))
    snap = {"flat_p": opt.flat_p.detach(), "flat_g": opt.flat_g, "exp_avg": opt.exp_avg, "exp_avg_sq": opt.exp_avg_sq,
            "step": opt.step_count, "rng": plan.rng_state, "slot.src": slot.src, "slot.logits": slot.logits}
    snap.update({"param." + k: p.detach() for k, p in model.named_parameters()})
    snap.update({"grad." + k: p.grad for k, p in model.named_parameters() if p.grad is not None})
    before = {k: v.clone() for k, v in snap.items()}
    model.eval()
    EP.prefix_predict(model, d["src"], d["static"], d["times"], d["lengths"], horizons=[1.0, 5.0, float("inf")])
    EP.prefix_predict(model, d["src"], d["static"], d["times"], d["lengths"], internal_batch_size=3 * B)
    torch.cuda.synchronize()
    for k, v in snap.items():
        assert torch.equal(v, before[k]), k
    model.train()
    logits, _, _ = model.forward(d["src"], d["static"], d["times"], d["lengths"])      # the captured step still runs
    F.cross_entropy(logits, d["y"]).backward()
    opt.step()


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name,B,K", [("P19", 3880, 12), ("PAM", 64, 50)])
def test_large_calls_fit_the_scratch_plan(cfg_name, B, K):
    from raindrop_b200 import lib as L
    cfg = model_config(cfg_name, dropout=0.2)
    d = to_dev(make_batch(cfg, B, seed=11))
    model = build_dropin(cfg, 9).eval()
    model._plan.obprop_mode = FAST
    rows = np.linspace(1, cfg["max_len"], K).round().astype(np.int32)
    res = EP.prefix_predict(model, *_args(d), rows=rows)
    assert res.logits.shape == (B, K, cfg["n_classes"]) and torch.isfinite(res.logits).all()
    # the plan: the largest chunk whose scratch fits in 1 GiB, or one prefix per chunk when even that does not
    key, scratch = model._plan.__dict__["_prefix_scratch"]
    kc = key[1]
    dims = model._plan.dims(B, False)
    nbytes = lambda c: L.load().rd_prefix_scratch_bytes(C.byref(dims), c)       # noqa: E731
    assert scratch.numel() * 4 >= nbytes(kc) > 0
    assert kc == 1 or nbytes(kc) <= 1 << 30
    assert kc == K or nbytes(kc + 1) > 1 << 30
    last = EP.prefix_predict(model, *_args(d), rows=rows[-1:])
    assert torch.equal(last.logits[:, 0], res.logits[:, -1])


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_drawn_cutoffs_match_restatement(name):
    cfg, d, model = _setup(name)
    B = d["src"].shape[1]
    tm = d["times"].cpu().numpy()
    for step, p_full, mf, rows in ((3, 0.5, 0.25, None), (4, 0.0, 0.0, None), (5, 0.3, 0.6, None),
                                   (6, 0.5, 0.25, np.where(np.arange(B) % 2 == 0, np.arange(B) * 3, -1))):
        cut, ex = _debug_inputs(model, d, rows=rows, K=1, key=(SEED, step), p_full=p_full, min_fraction=mf)
        want = drawn_cutoffs(tm, SEED, step, p_full, mf, rows)
        assert np.array_equal(cut[0].cpu().numpy(), want)
        _check_rows(d, cut, ex)
    cut, ex = _debug_inputs(model, d, K=1, key=(SEED, 9), p_full=1.0)
    assert (cut == cfg["max_len"]).all()
    assert torch.equal(ex[0], d["src"]) and torch.equal(ex[2], d["times"]) and torch.equal(ex[3], d["lengths"])


# ---- training on truncated records ------------------------------------------------------------------------------------
RNG0 = (0x1234ABCD5678, 11)


def _train_model(cfg, mode=EXACT):
    model = build_dropin(cfg, 21).train()
    plan = model._prepare(torch.device("cuda"))
    plan.obprop_mode = mode
    plan.rng_state.copy_(torch.tensor(RNG0, dtype=torch.int64))
    return model


def _run(step, n):
    losses, logits = [], []
    for _ in range(n):
        losses.append(step.step().clone())
        logits.append(step.logits.clone())
    torch.cuda.synchronize()
    return (step.flat_p.clone(), step.exp_avg.clone(), step.exp_avg_sq.clone(), torch.cat(losses), torch.cat(logits),
            step.plan.rng_state.clone())


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
def test_full_records_step_is_train_step(use_graph):
    from raindrop_b200.train import TrainStep
    cfg = model_config("P19", dropout=0.2)
    B = 37
    batch = to_dev(make_batch(cfg, B, seed=5, first_time_zero=True))
    out = []
    for prefix in (False, True):
        model = _train_model(cfg)
        s = EP.PrefixTrainStep(model, B, p_full=1.0, noise_seed=3, use_graph=use_graph) if prefix \
            else TrainStep(model, B, use_graph=use_graph)
        s.load_batch(batch)
        out.append(_run(s, 3))
    for a, b in zip(*out):
        assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("name", ["tiny_b6", "tiny8_b5", "p19_b9"])
def test_given_rows_step_is_train_step_on_truncated_batch(use_graph, name):
    from raindrop_b200.train import TrainStep
    cfg_name, B, opts = CASES[name]
    cfg = model_config(cfg_name, dropout=0.2)
    T = cfg["max_len"]
    batch = to_dev(make_batch(cfg, B, seed=7, **opts))
    rows = torch.tensor([(3 * b + 1) % (T + 1) for b in range(B)])
    s = EP.PrefixTrainStep(_train_model(cfg), B, noise_seed=SEED, use_graph=use_graph, lr=1e-3)
    s.load_batch(dict(batch, rows=rows))
    ref = TrainStep(_train_model(cfg), B, use_graph=use_graph, lr=1e-3)
    src, st, tm, ln = truncated(batch, rows.cuda())
    ref.load_batch(dict(batch, src=src, static=st, times=tm, lengths=ln))
    got, want = _run(s, 3), _run(ref, 3)
    for x, y in zip(got, want):
        assert torch.equal(x, y)
    assert torch.equal(s.cutoffs[0].cpu(), rows.int())


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny_b6", "p19_b9"])
def test_drawn_step_and_key_restore(name):
    """One step equals TrainStep on the batch exported for the step's key; the key advances by one per step; restoring
    the state and the key replays the step."""
    from raindrop_b200.train import TrainStep
    cfg_name, B, opts = CASES[name]
    cfg = model_config(cfg_name, dropout=0.2)
    batch = to_dev(make_batch(cfg, B, seed=7, **opts))
    model = _train_model(cfg)
    s = EP.PrefixTrainStep(model, B, p_full=0.2, min_fraction=0.1, noise_seed=SEED, lr=1e-3)
    s.set_noise_key(SEED, 4)
    s.load_batch(batch)
    s.step()
    torch.cuda.synchronize()
    assert s.noise_key_state() == (SEED, 5)
    state = [t.clone() for t in s._state()]
    ref_model = _train_model(cfg)
    ref = TrainStep(ref_model, B, use_graph=False, lr=1e-3)
    ref.flat_p.copy_(s.flat_p); ref.exp_avg.copy_(s.exp_avg); ref.exp_avg_sq.copy_(s.exp_avg_sq)
    ref.step_count.copy_(s.step_count); ref.plan.rng_state.copy_(s.plan.rng_state)
    cut, ex = _debug_inputs(ref_model, batch, K=1, key=(SEED, 5), p_full=0.2, min_fraction=0.1)
    assert np.array_equal(cut[0].cpu().numpy(), drawn_cutoffs(batch["times"].cpu().numpy(), SEED, 5, 0.2, 0.1))
    assert (cut < cfg["max_len"]).any()
    ref.load_batch(dict(batch, src=ex[0], static=ex[1], times=ex[2], lengths=ex[3]))
    got = _run(s, 1)
    want = _run(ref, 1)
    for x, y in zip(got, want):
        assert torch.equal(x, y)
    assert torch.equal(s.cutoffs, cut)
    assert s.noise_key_state() == (SEED, 6)
    for t, v in zip(s._state(), state):
        t.copy_(v)
    s.set_noise_key(SEED, 5)
    again = _run(s, 1)
    for x, y in zip(got, again):
        assert torch.equal(x, y)
