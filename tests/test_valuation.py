"""KNN-Shapley data valuation for Raindrop_v2 (raindrop_b200.valuation: rd_knn_shapley, rd_debug_knn_rank).

CPU: the float64 oracle's recursion and suffix form against brute-force enumeration of every coalition (N <= 10, K from
1 to N + 2, two and three classes, tied similarities, with and without the query's own record), efficiency, the exported
symbols, the scratch queries, the refusals of the C entry before any launch, the host refusals and the calls without
CUDA.  GPU: the device similarities against numpy float64 dots and its ranking against np.lexsort where the gaps are
clear; per_query, values and utility against the oracle on the device's own features at TINY / TINY8 / P19 / P12 / PAM on
both layers, k = 1, 10, n, n + 5, small and tail-sized training sets, both modes; bitwise ties of duplicated records;
efficiency; bitwise invariance under chunking, split accumulating calls, repeat runs and CUDA-graph replay; no side
effects on the model; the full-size P19 case and the scratch plan at PAM and LARGE widths.  Every GPU test on a model
pins plan.obprop_mode: the auto mode picks the ob-prop arithmetic from the row count."""
import os
import subprocess

import numpy as np
import pytest
import torch

from helpers import build_dropin, to_dev
from oracle import valuation_oracle as VO
from raindrop_b200 import lib as L
from raindrop_b200 import valuation as VA
from raindrop_b200.synth import make_batch, model_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXACT, FAST = 2, 1
TOL = 1e-12
NEW_SYMBOLS = ("rd_knn_shapley_scratch_bytes", "rd_knn_shapley", "rd_debug_knn_rank")


# ---- CPU --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 2, 3, 5, 8, 10])
@pytest.mark.parametrize("C", [2, 3])
def test_oracle_recursion_equals_enumeration(N, C):
    rng = np.random.default_rng(10 * N + C)
    for exclude in (None, 0, N // 2):
        n = N + (exclude is not None)
        if exclude is not None and exclude >= n:
            continue
        sim = np.round(rng.uniform(-1, 1, n), 1)                 # ties at one decimal
        sim[: n // 2] = sim[n // 2: 2 * (n // 2)]                 # and some exact duplicates
        y = rng.integers(0, C, n)
        yq = int(rng.integers(0, C))
        order = VO.rank(sim, exclude=exclude)
        assert len(order) == N
        m = y[order] == yq
        for K in range(1, N + 3):
            brute = VO.brute_force(sim, y, yq, K, exclude=exclude)
            rec = np.zeros(n)
            rec[order] = VO.recursion(m, K)
            suf = np.zeros(n)
            suf[order] = VO.suffix_form(m, K)
            assert np.abs(rec - brute).max() <= 1e-12, (K, exclude)
            assert np.abs(suf - brute).max() <= 1e-12, (K, exclude)
            assert abs(rec.sum() - VO.utility(m, K)) <= 1e-12          # efficiency
            if exclude is not None:
                assert brute[exclude] == 0.0


def test_oracle_forms_agree_at_larger_n():
    rng = np.random.default_rng(3)
    for N, K in [(39, 44), (39, 5), (200, 1), (200, 10), (500, 500)]:
        m = rng.integers(0, 2, N).astype(bool)
        assert np.abs(VO.recursion(m, K) - VO.suffix_form(m, K)).max() <= 1e-12
        assert abs(VO.recursion(m, K).sum() - VO.utility(m, K)) <= 1e-12


def test_oracle_rank_ties_go_to_the_lower_index():
    sim = np.array([0.5, 0.9, 0.5, 0.9, -0.1])
    assert VO.rank(sim).tolist() == [1, 3, 0, 2, 4]
    assert VO.rank(sim, exclude=3).tolist() == [1, 0, 2, 4]


def test_symbols_and_scratch_queries():
    lib_path = os.path.join(ROOT, "raindrop_b200", "csrc", "librd_b200.so")
    out = subprocess.run(["nm", "-D", "--defined-only", lib_path], capture_output=True, text=True, check=True).stdout
    names = {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert set(NEW_SYMBOLS) <= names
    header = open(os.path.join(ROOT, "include", "raindrop_b200.h")).read()
    for name in NEW_SYMBOLS:
        assert name in L.SIGNATURES and name + "(" in header
    lib = L.load()
    q = lib.rd_knn_shapley_scratch_bytes
    assert 0 < q(100, 4, 1) < q(100, 4, 7) < q(1000, 4, 7)
    assert q(1, 4, 1) > 0 and q((1 << 31) - 1, 4, 1) > 0
    for bad in [(0, 4, 1), (1 << 31, 4, 1), (100, 0, 1), (100, 6, 1), (100, 4, 0), (100, 4, -1)]:
        assert q(*bad) == 0, bad


def test_kernel_refusals_before_any_launch():
    lib = L.load()
    P = 256                                                       # aligned fake pointers: never dereferenced

    def call(bank=P, n=10, ld=4, yt=P, qs=P, nq=3, yq=P, k=2, self_offset=-1, qc=4, scratch=P, values=P):
        return lib.rd_knn_shapley(bank, n, ld, yt, qs, nq, yq, k, self_offset, qc, 0, scratch, values, None, None, None)

    for kw in (dict(k=0), dict(n=0), dict(n=1 << 31), dict(ld=6), dict(qc=0), dict(nq=-1), dict(bank=None),
               dict(yt=None), dict(qs=None), dict(yq=None), dict(scratch=None), dict(values=None),
               dict(self_offset=-2), dict(self_offset=8), dict(n=1, nq=1, self_offset=0), dict(bank=P + 4),
               dict(scratch=P + 16)):
        assert call(**kw) == -2, kw
    assert b"rd_knn_shapley" in lib.rd_last_error_string()
    assert lib.rd_debug_knn_rank(P, 10, 4, P, 0, -1, P, P, P, None) == -2
    assert lib.rd_debug_knn_rank(P, 10, 4, P, 3, 8, P, P, P, None) == -2
    assert lib.rd_debug_knn_rank(None, 10, 4, P, 3, -1, P, P, P, None) == -2


def test_host_refusals():
    f, y = torch.zeros(6, 5), torch.zeros(6, dtype=torch.int64)
    for kw in (dict(k=0), dict(k=1.5), dict(k=True), dict(internal_batch_size=0)):
        with pytest.raises(ValueError):
            VA.knn_shapley_from_features(f, y, **kw)
    bad = [(torch.zeros(6), y), (torch.zeros(0, 5), y[:0]), (f, y[:5]), (f, y.float()), (f, y.bool()),
           (f[:1], y[:1])]                                                        # leave-one-out needs 2 records
    for args in bad:
        with pytest.raises(ValueError):
            VA.knn_shapley_from_features(*args)
    for q, yq in ((torch.zeros(3, 4), y[:3]), (torch.zeros(3, 5), None), (torch.zeros(3, 5), y[:2])):
        with pytest.raises(ValueError):
            VA.knn_shapley_from_features(f, y, q, yq)
    with pytest.raises(ValueError):
        VA.knn_shapley_from_features(f, y, None, y)
    cfg = model_config("TINY", dropout=0.2)
    m = build_dropin(cfg, 3, device="cpu").eval()
    b = make_batch(cfg, 4, seed=1)
    data = dict(src=b["src"], static=b["static"], times=b["times"], lengths=b["lengths"], y=b["y"])
    with pytest.raises(ValueError, match="layer"):
        VA.knn_shapley(m, data, layer="logits")
    with pytest.raises(ValueError, match="label"):
        VA.knn_shapley(m, dict(data, y=None))
    with pytest.raises(ValueError, match="k must"):
        VA.knn_shapley(m, data, k=0)
    with pytest.raises(ValueError):
        VA.knn_shapley(m, data, query=dict(data, times=b["times"][:, :2]))
    m.train()
    with pytest.raises(ValueError, match="eval"):
        VA.knn_shapley(m, data)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the behaviour without CUDA")
def test_calls_without_cuda_raise():
    f, y = torch.rand(6, 5), torch.zeros(6, dtype=torch.int64)
    with pytest.raises(L.RaindropB200Error):
        VA.knn_shapley_from_features(f, y)
    with pytest.raises(L.RaindropB200Error):
        VA.knn_shapley_from_features(f, y, f[:2], y[:2])
    cfg = model_config("TINY", dropout=0.2)
    m = build_dropin(cfg, 3, device="cpu").eval()
    b = make_batch(cfg, 4, seed=1)
    with pytest.raises(L.RaindropB200Error):
        VA.knn_shapley(m, dict(src=b["src"], static=b["static"], times=b["times"], lengths=b["lengths"], y=b["y"]))


# ---- GPU --------------------------------------------------------------------------------------------------------------
def _bank(f):
    lib = L.load()
    n, F = f.shape
    Fp = (F + 3) // 4 * 4
    return VA._bank(lib, f.float().contiguous(), n, F, Fp), Fp


def _device_rank(bank, n, Fp, queries, nq, self_offset=-1):
    """(sim [nq, n] fp64, order [nq, n]) of rd_debug_knn_rank."""
    lib = L.load()
    nb = lib.rd_knn_shapley_scratch_bytes(n, Fp, nq)
    scratch = torch.empty((nb + 255) // 256 * 32, dtype=torch.float64, device="cuda")
    sim = torch.empty(nq, n, dtype=torch.float64, device="cuda")
    order = torch.empty(nq, n, dtype=torch.int64, device="cuda")
    L.check(lib.rd_debug_knn_rank(bank.data_ptr(), n, Fp, queries.data_ptr(), nq, self_offset, scratch.data_ptr(),
                                  sim.data_ptr(), order.data_ptr(), L.stream_ptr()), "rd_debug_knn_rank")
    return sim.cpu().numpy(), order.cpu().numpy()


def _oracle(ft, yt, fq=None, yq=None, k=10):
    """The oracle on the device's own normalised rows, ranked by the device's similarities (checked against numpy
    float64 dots to 1e-13 here as well)."""
    n = ft.shape[0]
    bank, Fp = _bank(ft)
    loo = fq is None
    queries, nq = (bank, n) if loo else (_bank(fq)[0], fq.shape[0])
    sim, _ = _device_rank(bank, n, Fp, queries, nq, 0 if loo else -1)
    b64 = bank[:n].double().cpu().numpy()
    q64 = queries[:nq].double().cpu().numpy()
    ref = q64 @ b64.T
    if loo:
        np.fill_diagonal(ref, np.nan)
    assert np.nanmax(np.abs(sim - ref)) <= 1e-13
    yt = yt.cpu().numpy()
    yq = yt if loo else yq.cpu().numpy()
    return VO.knn_shapley(np.where(np.isnan(sim), 0.0, sim), yt, yq, k, self_offset=0 if loo else None)


def _check(res, ref, n_query):
    per, values, util = ref
    assert np.abs(res.utility.cpu().numpy() - util).max() <= TOL
    assert np.abs(res.values.cpu().numpy() - values).max() <= TOL
    if res.per_query is not None:
        pq = res.per_query.cpu().numpy()
        assert np.abs(pq - per).max() <= TOL
        assert np.abs(pq.sum(1) - res.utility.cpu().numpy()).max() <= TOL            # efficiency per query
    assert abs(res.values.sum().item() - res.utility.mean().item()) <= TOL
    assert res.values.dtype == torch.float64 and res.values.shape[0] == per.shape[1] and len(util) == n_query


@pytest.mark.gpu
@pytest.mark.parametrize("F,n,nq,self_mode", [(37, 300, 70, False), (100, 129, 64, True), (132, 65, 1, False),
                                               (4, 1000, 130, True)])
def test_similarities_and_ranking_against_numpy(F, n, nq, self_mode):
    rng = np.random.default_rng(F + n)
    ft = torch.from_numpy(rng.normal(size=(n, F)).astype(np.float32)).cuda()
    bank, Fp = _bank(ft)
    if self_mode:
        queries, off = bank, 0
        nq = n
    else:
        queries, off = _bank(torch.from_numpy(rng.normal(size=(nq, F)).astype(np.float32)).cuda())[0], -1
    sim, order = _device_rank(bank, n, Fp, queries, nq, off)
    ref = queries[:nq].double().cpu().numpy() @ bank[:n].double().cpu().numpy().T
    for q in range(nq):
        ex = q if self_mode else None
        want = VO.rank(ref[q], exclude=ex)
        s = np.sort(ref[q][want])[::-1]
        assert np.all(-np.diff(s) > 1e-12), "the oracle's consecutive gaps are clear"
        got = order[q][:-1] if self_mode else order[q]
        assert np.array_equal(got, want), q
        if self_mode:
            assert order[q][-1] == q and np.isnan(sim[q, q])
            sim[q, q] = ref[q, q]
    assert np.abs(sim - ref).max() <= 1e-13


@pytest.mark.gpu
def test_duplicated_records_tie_bitwise_and_rank_by_index():
    rng = np.random.default_rng(1)
    base = rng.normal(size=(40, 23)).astype(np.float32)
    ft = np.concatenate([base, base[[3, 3, 17]], base[:5]])              # exact copies at the end
    t = torch.from_numpy(ft).cuda()
    bank, Fp = _bank(t)
    n = ft.shape[0]
    q = _bank(torch.from_numpy(rng.normal(size=(9, 23)).astype(np.float32)).cuda())[0]
    sim, order = _device_rank(bank, n, Fp, q, 9)
    for a, b in [(3, 40), (3, 41), (17, 42), (0, 43), (4, 47)]:
        assert np.array_equal(sim[:, a], sim[:, b])                     # bitwise
        pos = np.argsort(order, axis=1)
        assert np.all(pos[:, a] < pos[:, b])
    y = torch.from_numpy(rng.integers(0, 2, n)).cuda()
    yq = torch.from_numpy(rng.integers(0, 2, 9)).cuda()
    res = VA.knn_shapley_from_features(t, y, torch.from_numpy(rng.normal(size=(9, 23)).astype(np.float32)).cuda(), yq,
                                       k=3, per_query=True)
    assert torch.isfinite(res.values).all()


MODEL_CASES = {
    "tiny": ("TINY", 7, 5),
    "tiny8": ("TINY8", 9, 4),                       # 8 classes, no statics
    "p19": ("P19", 130, 33),                        # tile tails of 64
    "p12": ("P12", 23, 6),
    "pam": ("PAM", 67, 5),                          # 8 classes
}


def _model_data(name, n, seed):
    cfg = model_config(MODEL_CASES[name][0], dropout=0.2)
    model = build_dropin(cfg, 11).eval()
    model._plan.obprop_mode = EXACT
    b = to_dev(make_batch(cfg, n, seed=seed))
    if cfg["n_classes"] > 2:
        b["y"] = torch.arange(n, device="cuda") % cfg["n_classes"]
    return cfg, model, dict(src=b["src"], static=b["static"], times=b["times"], lengths=b["lengths"], y=b["y"])


def _slice(d, i0, i1):
    return dict(src=d["src"][:, i0:i1], static=None if d["static"] is None else d["static"][i0:i1],
                times=d["times"][:, i0:i1], lengths=d["lengths"][i0:i1], y=d["y"][i0:i1])


@pytest.mark.gpu
@pytest.mark.parametrize("layer", ["hidden", "pooled"])
@pytest.mark.parametrize("name", list(MODEL_CASES))
def test_matches_the_oracle_on_model_features(name, layer):
    from raindrop_b200.ood import features
    _, n, nq = MODEL_CASES[name]
    cfg, model, d = _model_data(name, n + nq, seed=3)
    train, query = _slice(d, 0, n), _slice(d, n, n + nq)
    ft, _ = features(model, train["src"], train["static"], train["times"], train["lengths"], layer)
    fq, _ = features(model, query["src"], query["static"], query["times"], query["lengths"], layer)
    for k in (1, 10, n, n + 5):
        res = VA.knn_shapley(model, train, query, k=k, layer=layer, per_query=True)
        assert res.layer == layer and res.k == k and not res.leave_one_out
        _check(res, _oracle(ft, train["y"], fq, query["y"], k), nq)
        loo = VA.knn_shapley(model, train, k=k, layer=layer, per_query=True)
        assert loo.leave_one_out and torch.all(loo.per_query.diagonal() == 0)
        _check(loo, _oracle(ft, train["y"], k=k), n)


@pytest.mark.gpu
@pytest.mark.parametrize("n,nq,F,C", [(1, 5, 9, 2), (2, 3, 8, 2), (3, 70, 5, 8), (63, 64, 12, 2), (65, 129, 13, 8),
                                      (130, 2, 40, 3)])
def test_small_and_tail_sized_sets(n, nq, F, C):
    rng = np.random.default_rng(n * 7 + nq)
    ft = torch.from_numpy(np.maximum(rng.normal(size=(n, F)), 0).astype(np.float32)).cuda()
    fq = torch.from_numpy(np.maximum(rng.normal(size=(nq, F)), 0).astype(np.float32)).cuda()
    yt = torch.from_numpy(rng.integers(0, C, n)).cuda()
    yq = torch.from_numpy(rng.integers(0, C, nq)).cuda()
    for k in sorted({1, 10, n, n + 5}):
        _check(VA.knn_shapley_from_features(ft, yt, fq, yq, k=k, per_query=True), _oracle(ft, yt, fq, yq, k), nq)
        if n >= 2:
            _check(VA.knn_shapley_from_features(ft, yt, k=k, per_query=True), _oracle(ft, yt, k=k), n)


@pytest.mark.gpu
def test_bitwise_chunking_split_calls_runs_and_graph_replay():
    rng = np.random.default_rng(8)
    n, nq, F = 517, 203, 44
    ft = torch.from_numpy(rng.normal(size=(n, F)).astype(np.float32)).cuda()
    fq = torch.from_numpy(rng.normal(size=(nq, F)).astype(np.float32)).cuda()
    yt = torch.from_numpy(rng.integers(0, 3, n)).cuda()
    yq = torch.from_numpy(rng.integers(0, 3, nq)).cuda()
    for q, y in ((fq, yq), (None, None)):
        runs = [VA.knn_shapley_from_features(ft, yt, q, y, k=7, per_query=True, internal_batch_size=b)
                for b in (None, 1, 5, 64, 203, 10_000, None)]
        for r in runs[1:]:
            for f in ("values", "utility", "per_query"):
                assert torch.equal(getattr(r, f), getattr(runs[0], f)), f
    # a query set split over accumulating calls gives the sums bitwise
    lib = L.load()
    bank, Fp = _bank(ft)
    qb, _ = _bank(fq)
    ytd, yqd = yt.contiguous(), yq.contiguous()
    nb = lib.rd_knn_shapley_scratch_bytes(n, Fp, 64)
    scratch = torch.empty((nb + 255) // 256 * 32, dtype=torch.float64, device="cuda")
    values = torch.empty(n, dtype=torch.float64, device="cuda")
    for i, (a, b) in enumerate([(0, 50), (50, 51), (51, 203)]):
        L.check(lib.rd_knn_shapley(bank.data_ptr(), n, Fp, ytd.data_ptr(), qb[a:].data_ptr(), b - a, yqd[a:].data_ptr(), 7,
                                   -1, 64, int(i > 0), scratch.data_ptr(), values.data_ptr(), None, None, L.stream_ptr()),
                "rd_knn_shapley")
    whole = VA.knn_shapley_from_features(ft, yt, fq, yq, k=7)
    assert torch.equal(values / nq, whole.values)
    # CUDA-graph replay after an eager call with the same shapes
    eager = VA.knn_shapley_from_features(ft, yt, fq, yq, k=7, per_query=True, internal_batch_size=64)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        VA.knn_shapley_from_features(ft, yt, fq, yq, k=7, per_query=True, internal_batch_size=64)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cap = VA.knn_shapley_from_features(ft, yt, fq, yq, k=7, per_query=True, internal_batch_size=64)
    for t in (cap.values, cap.utility, cap.per_query):
        t.fill_(0)
    g.replay()
    torch.cuda.synchronize()
    for f in ("values", "utility", "per_query"):
        assert torch.equal(getattr(cap, f), getattr(eager, f)), f


@pytest.mark.gpu
def test_no_side_effects_and_sources():
    from raindrop_b200.data import DeviceDataset
    cfg, model, d = _model_data("tiny", 30, seed=4)
    ds = DeviceDataset(d["src"], d["static"], d["times"], d["y"])
    plan = model._prepare(d["src"].device)
    params = [p.detach().clone() for p in model.parameters()]
    rng = plan.rng_state.clone()
    sel = torch.tensor([5, 0, 29, 7, 11, 3, 18, 21, 1, 9, 14, 2])
    a = VA.knn_shapley(model, (ds, sel[:8]), (ds, sel[8:]), k=3, per_query=True)
    b = VA.knn_shapley(model, _pick(d, sel[:8]), _pick(d, sel[8:]), k=3, per_query=True, internal_batch_size=3)
    for f in ("values", "utility", "per_query"):
        assert torch.equal(getattr(a, f), getattr(b, f)), f
    VA.knn_shapley(model, ds, k=4)
    assert torch.equal(plan.rng_state, rng) and not model.training
    assert all(torch.equal(p, q) for p, q in zip(model.parameters(), params))
    assert all(p.grad is None for p in model.parameters())


def _pick(d, sel):
    ix = sel.cuda()
    return dict(src=d["src"][:, ix], static=d["static"][ix], times=d["times"][:, ix], lengths=d["lengths"][ix],
                y=d["y"][ix])


@pytest.mark.gpu
def test_non_finite_features_refused():
    f = torch.rand(10, 6, device="cuda")
    y = torch.zeros(10, dtype=torch.int64, device="cuda")
    f[3, 2] = float("nan")
    with pytest.raises(ValueError, match="finite"):
        VA.knn_shapley_from_features(f, y)
    with pytest.raises(ValueError, match="finite"):
        VA.knn_shapley_from_features(torch.rand(10, 6, device="cuda"), y, f, y)


@pytest.mark.gpu
def test_full_size_p19():
    """P19 synthetic weights: 31,000 training and 3,880 query records, and leave-one-out over the training set."""
    import time
    cfg = model_config("P19", dropout=0.2)
    model = build_dropin(cfg, 5).eval()
    model._plan.obprop_mode = FAST
    n, nq = 31_000, 3_880
    b = to_dev(make_batch(cfg, n + nq, seed=19))
    d = dict(src=b["src"], static=b["static"], times=b["times"], lengths=b["lengths"], y=b["y"])
    train, query = _slice(d, 0, n), _slice(d, n, n + nq)
    from raindrop_b200.ood import features
    ft, _ = features(model, train["src"], train["static"], train["times"], train["lengths"])
    fq, _ = features(model, query["src"], query["static"], query["times"], query["lengths"])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = VA.knn_shapley_from_features(ft, train["y"], fq, query["y"], k=10)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    loo = VA.knn_shapley_from_features(ft, train["y"], k=10)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    for r, m in ((res, nq), (loo, n)):
        assert abs(r.values.sum().item() - r.utility.mean().item()) <= TOL
        assert r.utility.shape[0] == m and torch.isfinite(r.values).all()
    assert torch.equal(res.values, VA.knn_shapley(model, train, query, k=10).values)
    # 16 random queries of each mode against the oracle on the device's features
    pick = np.sort(np.random.default_rng(0).choice(nq, 16, replace=False))
    sub = VA.knn_shapley_from_features(ft, train["y"], fq[pick], query["y"][pick], k=10, per_query=True)
    per, _, util = _oracle(ft, train["y"], fq[pick], query["y"][pick], 10)
    assert np.abs(sub.per_query.cpu().numpy() - per).max() <= TOL
    assert np.abs(sub.utility.cpu().numpy() - util).max() <= TOL
    assert np.abs(res.utility[pick].cpu().numpy() - util).max() <= TOL
    lib = L.load()
    bank, Fp = _bank(ft)
    pick = np.sort(np.random.default_rng(1).choice(n, 16, replace=False))
    sim_all = []
    for i in pick:
        sim, _ = _device_rank(bank, n, Fp, bank[i:], 1, i)
        sim_all.append(sim[0])
    yt = train["y"].cpu().numpy()
    nb = lib.rd_knn_shapley_scratch_bytes(n, Fp, 1)
    scratch = torch.empty((nb + 255) // 256 * 32, dtype=torch.float64, device="cuda")
    ytd = train["y"].contiguous()
    for i, sim in zip(pick, sim_all):
        row = torch.empty(1, n, dtype=torch.float64, device="cuda")
        util1 = torch.empty(1, dtype=torch.float64, device="cuda")
        v = torch.empty(n, dtype=torch.float64, device="cuda")
        L.check(lib.rd_knn_shapley(bank.data_ptr(), n, Fp, ytd.data_ptr(), bank[i:].data_ptr(), 1, ytd[i:].data_ptr(), 10,
                                   int(i), 1, 0, scratch.data_ptr(), v.data_ptr(), row.data_ptr(), util1.data_ptr(),
                                   L.stream_ptr()), "rd_knn_shapley")
        sim[i] = 0.0
        per, _, util = VO.knn_shapley(sim[None], yt, yt[i:i + 1], 10, self_offset=i)
        assert np.abs(row.cpu().numpy() - per).max() <= TOL
        assert abs(util1.item() - util[0]) <= TOL and abs(util1.item() - loo.utility[i].item()) == 0
    print("knn_shapley P19 n=%d: %d queries %.3f s, leave-one-out %.3f s" % (n, nq, t1 - t0, t2 - t1))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["PAM", "LARGE"])
def test_scratch_plan_at_wide_features(name):
    cfg = model_config(name)
    d_ob = cfg["d_model"] // cfg["d_inp"]
    F = cfg["d_inp"] * d_ob + 16 + (cfg["d_inp"] if cfg["static"] else 0)
    n, nq = 12_000, 5_000
    lib = L.load()
    Fp = (F + 3) // 4 * 4
    qc = VA._chunk(lib, n, Fp, nq, None)
    assert lib.rd_knn_shapley_scratch_bytes(n, Fp, qc) <= VA.DEFAULT_SCRATCH_BYTES and 1 < qc < nq
    g = torch.Generator(device="cuda").manual_seed(2)
    ft = torch.relu(torch.randn(n, F, device="cuda", generator=g))
    fq = torch.relu(torch.randn(nq, F, device="cuda", generator=g))
    yt = torch.randint(0, cfg["n_classes"], (n,), device="cuda", generator=g)
    yq = torch.randint(0, cfg["n_classes"], (nq,), device="cuda", generator=g)
    res = VA.knn_shapley_from_features(ft, yt, fq, yq, k=10)
    one = VA.knn_shapley_from_features(ft, yt, fq, yq, k=10, internal_batch_size=nq)
    assert torch.equal(res.values, one.values)
    assert abs(res.values.sum().item() - res.utility.mean().item()) <= TOL
