"""Batch active learning for Raindrop_v2 (raindrop_b200.active: rd_batch_bald, rd_badge).

CPU: the exported symbols and scratch queries, the host refusals, the calls without CUDA, and the float64 oracle itself:
its exact BatchBALD against a direct sum over the full joint table, the sampled estimator's mean against the exact
value, the (configuration, pick) -> Philox counter mapping, and the factorised BADGE distance against the materialised
one.  GPU: batch_bald and badge against the oracle on the same draws (exact mode, sampled mode, the switch; C = 2 and
8), scores[0] against mc_dropout's mutual information, k = 200 picks of confident replicates, bitwise invariance under
internal_batch_size, CUDA-graph replay, no side effects on the model, pool_logits against the wrapped calls, and one
full-size P19 pool."""
import os
import subprocess
import time

import numpy as np
import pytest
import torch

from helpers import build_dropin, to_dev
from oracle import active_oracle as AO
from oracle.dropout_masks import philox4x32_10
from raindrop_b200 import active as AC
from raindrop_b200 import lib as L
from raindrop_b200.synth import make_batch, model_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXACT = 2
SCORE_RTOL = 1e-5
NEW_SYMBOLS = ("rd_batch_bald_scratch_bytes", "rd_batch_bald", "rd_badge_scratch_bytes", "rd_badge")


def _logits(M, N, C, seed, scale=2.0):
    """Replicates that disagree: a per-point centre plus per-replicate noise."""
    rng = np.random.default_rng(seed)
    centre = rng.normal(size=(1, N, C)) * scale
    return (centre + rng.normal(size=(M, N, C)) * scale).astype(np.float32)


# ---- CPU --------------------------------------------------------------------------------------------------------------
def test_symbols_exported():
    lib_path = os.path.join(ROOT, "raindrop_b200", "csrc", "librd_b200.so")
    out = subprocess.run(["nm", "-D", "--defined-only", lib_path], capture_output=True, text=True, check=True).stdout
    names = {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert set(NEW_SYMBOLS) <= names
    header = open(os.path.join(ROOT, "include", "raindrop_b200.h")).read()
    for name in NEW_SYMBOLS:
        assert name in L.SIGNATURES and name + "(" in header
    assert "#define RD_ACTIVE_MAX_CLASSES %d" % L.ACTIVE_MAX_CLASSES in header
    assert "#define RD_ACTIVE_MAX_REPLICATES %d" % L.ACTIVE_MAX_REPLICATES in header
    assert "#define RD_ACTIVE_MAX_CONFIGS %d" % L.ACTIVE_MAX_CONFIGS in header


def test_scratch_queries_and_kernel_refusals():
    lib = L.load()
    q = lib.rd_batch_bald_scratch_bytes
    assert 0 < q(100, 20, 2, 64, 10) < q(100, 20, 2, 64, 100) < q(100, 20, 2, 4096, 100)
    for bad in [(0, 20, 2, 64, 10), (100, 0, 2, 64, 10), (100, 1025, 2, 64, 10), (100, 20, 1, 64, 10),
                (100, 20, 9, 64, 10), (100, 20, 2, 0, 10), (100, 20, 2, 65537, 10), (100, 20, 2, 64, 0)]:
        assert q(*bad) == 0, bad
    assert q(100, 1024, 8, 65536, 100) > 0
    assert lib.rd_badge_scratch_bytes(100, 16, 2) > 0
    for bad in [(0, 16, 2), (100, 0, 2), (100, 16, 1), (100, 16, 9)]:
        assert lib.rd_badge_scratch_bytes(*bad) == 0, bad
    # refused before any launch: bad sizes, k > N, NULL pointers
    assert lib.rd_batch_bald(256, 100, 20, 2, 101, 64, 0, 0, 10, 256, 256, 256, 256, 256, None) == -2
    assert lib.rd_batch_bald(256, 100, 20, 9, 3, 64, 0, 0, 10, 256, 256, 256, 256, 256, None) == -2
    assert lib.rd_batch_bald(None, 100, 20, 2, 3, 64, 0, 0, 10, 256, 256, 256, 256, 256, None) == -2
    assert b"rd_batch_bald" in lib.rd_last_error_string()
    assert lib.rd_badge(256, 256, 100, 16, 2, 0, 0, 0, 256, 256, 256, None) == -2
    assert lib.rd_badge(256, 256, 100, 16, 9, 3, 0, 0, 256, 256, 256, None) == -2


def test_argument_errors_raise_on_the_host():
    z = torch.zeros(4, 10, 2)
    for kw in (dict(k=0), dict(k=11), dict(k=2.0), dict(k=True), dict(k=2, n_configs=0), dict(k=2, n_configs=65537),
               dict(k=2, seed=-1), dict(k=2, step=1 << 64), dict(k=2, internal_batch_size=0)):
        with pytest.raises(ValueError):
            AC.batch_bald(z, **kw)
    for shape in ((4, 10, 1), (4, 10, 9), (1025, 3, 2), (4, 0, 2), (10, 2)):
        with pytest.raises(ValueError):
            AC.batch_bald(torch.zeros(shape), k=1)
    h, lg = torch.zeros(10, 5), torch.zeros(10, 3)
    for args in ((h, lg, 0), (h, lg, 11), (h, torch.zeros(9, 3), 2), (h, torch.zeros(10, 9), 2), (h, torch.zeros(10, 1), 2),
                 (torch.zeros(10, 0), lg, 2), (h[None], lg, 2)):
        with pytest.raises(ValueError):
            AC.badge_from_features(*args)
    with pytest.raises(ValueError):
        AC.badge_from_features(h, lg, 2, seed=-1)
    cfg = model_config("TINY", dropout=0.2)
    m = build_dropin(cfg, 3, device="cpu").eval()
    b = make_batch(cfg, 4, seed=1)
    pool = dict(src=b["src"], static=b["static"], times=b["times"], lengths=b["lengths"])
    with pytest.raises(ValueError):
        AC.pool_logits(m, pool, batch_size=0)
    with pytest.raises(ValueError):
        AC.pool_logits(m, pool, n_samples=0)
    with pytest.raises(TypeError):
        AC.pool_logits(m, pool, posterior=object())
    with pytest.raises(ValueError):
        AC.pool_logits(m, dict(pool, times=b["times"][:, :2]))
    with pytest.raises(ValueError):
        AC.badge(m, pool, 5)                                        # k > N
    m.train()
    with pytest.raises(ValueError):
        AC.badge(m, pool, 2)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the behaviour without CUDA")
def test_calls_without_cuda_raise():
    with pytest.raises(L.RaindropB200Error):
        AC.batch_bald(torch.zeros(4, 10, 2), k=2)
    with pytest.raises(L.RaindropB200Error):
        AC.badge_from_features(torch.zeros(10, 5), torch.zeros(10, 3), 2)
    cfg = model_config("TINY", dropout=0.2)
    m = build_dropin(cfg, 3, device="cpu").eval()
    b = make_batch(cfg, 4, seed=1)
    pool = dict(src=b["src"], static=b["static"], times=b["times"], lengths=b["lengths"])
    with pytest.raises(L.RaindropB200Error):
        AC.pool_logits(m, pool, n_samples=2)
    with pytest.raises(L.RaindropB200Error):
        AC.badge(m, pool, 2)


@pytest.mark.parametrize("C,N,k", [(2, 6, 3), (3, 5, 3), (2, 4, 2)])
def test_oracle_exact_equals_the_full_joint_table(C, N, k):
    x = _logits(7, N, C, seed=10 + C + N)
    idx, scores = AO.batch_bald_bruteforce(x, k)
    res = AO.batch_bald(x, k, n_configs=C ** k)
    assert np.array_equal(res["indices"], idx) and res["exact"].all()
    for i in range(k):
        direct = AO.joint_table_mi(x, list(idx[: i + 1]))
        assert abs(scores[i] - direct) <= 1e-12 * max(1.0, abs(direct))
        assert abs(res["scores"][i] - direct) <= 1e-12 * max(1.0, abs(direct))
    assert np.allclose(res["bald"], [AO.joint_table_mi(x, [n]) for n in range(N)], rtol=0, atol=1e-12)


def test_oracle_sampled_estimate_is_unbiased_within_four_standard_errors():
    x = _logits(8, 6, 2, seed=3)
    exact = AO.batch_bald(x, 4, n_configs=16)
    assert exact["exact"].all()
    runs = np.array([AO.batch_bald(x, 4, n_configs=4, seed=s, follow=exact["indices"])["scores"] for s in range(300)])
    sampled = AO.batch_bald(x, 4, n_configs=4)["exact"]
    assert sampled.tolist() == [True, True, True, False]
    mean, se = runs[:, 3].mean(), runs[:, 3].std(ddof=1) / np.sqrt(len(runs))
    assert se > 0 and abs(mean - exact["scores"][3]) < 4 * se, (mean, se, exact["scores"][3])


def test_active_learning_draws_map_to_philox_counters():
    seed, step = 0x0123456789ABCDEF, (1 << 32) + 5
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) ^ (step >> 32)], dtype=np.uint64)
    for s, j in [(0, 0), (1, 0), (7, 3), (65535, 199)]:
        ctr = np.array([s, j, AO.SITE_BATCHBALD, step & 0xFFFFFFFF], dtype=np.uint64)
        assert np.array_equal(AO.active_words(seed, step, AO.SITE_BATCHBALD, s, j), philox4x32_10(ctr, key))
    w = philox4x32_10(np.array([5, 0, AO.SITE_BADGE, step & 0xFFFFFFFF], dtype=np.uint64), key)
    assert AO.badge_uniform(seed, step, 5) == ((int(w[0]) >> 5) * 2.0 ** 26 + (int(w[1]) >> 6)) * 2.0 ** -53
    # replicate m_s = floor(word M / 2^32) and labels from the fp32 inverse CDF
    ms = AO.sample_replicates(10, 4, seed, step)
    words = AO.active_words(seed, step, AO.SITE_BATCHBALD, np.arange(4), 0)[:, 0]
    assert ms.tolist() == [(int(v) * 10) >> 32 for v in words]
    p32 = np.array([[[0.25, 0.75]]], dtype=np.float32).repeat(10, 0)
    u = (AO.active_words(seed, step, AO.SITE_BATCHBALD, np.arange(4), 3)[:, 0] >> 8) * 2.0 ** -24
    assert AO.draw_labels(p32, ms, 0, 2, seed, step).tolist() == [int(v >= 0.25) for v in u]
    # the sites are past every dropout and sampling site of the library
    assert AO.SITE_BATCHBALD > 104 and AO.SITE_BADGE > 104 and AO.SITE_BATCHBALD != AO.SITE_BADGE


def test_factorised_badge_distance_equals_the_materialised_one():
    rng = np.random.default_rng(5)
    for C in (2, 3, 8):
        h = np.maximum(rng.normal(size=(12, 17)), 0).astype(np.float32)
        z = (rng.normal(size=(12, C)) * 3).astype(np.float32)
        g = AO.badge_embeddings(h, z)
        for i in range(12):
            for c in range(12):
                ref = ((g[i] - g[c]) ** 2).sum()
                got = AO.badge_factorised_d2(h, z, i, c)
                assert abs(got - ref) <= 1e-12 * max(ref, 1e-300) or (i == c and got < 1e-12), (C, i, c, got, ref)


# ---- GPU --------------------------------------------------------------------------------------------------------------
def _assert_clear_gaps(res, tol=SCORE_RTOL):
    """The oracle's best and second-best candidates differ by more than the score tolerance at every step."""
    for i, sc in enumerate(res["all_scores"]):
        top = np.sort(sc[np.isfinite(sc)])[::-1]
        if len(top) > 1:
            assert top[0] - top[1] > tol * abs(top[0]), (i, top[:2])


def _check_against_oracle(x, k, n_configs, seed=7, step=3):
    got = AC.batch_bald(torch.from_numpy(x).cuda(), k, n_configs=n_configs, seed=seed, step=step)
    ref = AO.batch_bald(x, k, n_configs=n_configs, seed=seed, step=step)
    _assert_clear_gaps(ref)
    assert np.array_equal(got.indices.cpu().numpy(), ref["indices"])
    assert got.exact.cpu().numpy().tolist() == ref["exact"].tolist()
    s = got.scores.cpu().numpy()
    assert np.all(np.abs(s - ref["scores"]) <= SCORE_RTOL * np.abs(ref["scores"])), (s, ref["scores"])
    b = got.bald.cpu().numpy()
    assert np.all(np.abs(b - ref["bald"]) <= SCORE_RTOL * np.abs(ref["bald"]).max())
    assert s[0] == b[got.indices[0].item()]
    return got, ref


@pytest.mark.gpu
@pytest.mark.parametrize("C,M,N,k,n_configs", [
    (2, 20, 150, 5, 64),        # exact only
    (2, 20, 150, 10, 64),       # exact, the switch at pick 7, sampled
    (2, 33, 300, 8, 2),         # sampled from pick 2 on, M not a multiple of 32
    (8, 12, 60, 6, 512),        # exact to pick 3, then sampled
    (8, 40, 70, 4, 700),        # C^|A| = 512 <= 700 < 4096
    (3, 100, 500, 6, 10_000),   # P19-like replicate count
])
def test_batch_bald_matches_the_oracle(C, M, N, k, n_configs):
    x = _logits(M, N, C, seed=100 * C + M + N + k)
    got, ref = _check_against_oracle(x, k, n_configs)
    assert ref["exact"].any()


@pytest.mark.gpu
def test_first_score_is_mc_dropout_mutual_information():
    from raindrop_b200.uncertainty import mc_dropout
    cfg = model_config("TINY", dropout=0.3)
    model = build_dropin(cfg, 21).eval()
    model._plan.obprop_mode = EXACT
    d = to_dev(make_batch(cfg, 40, seed=4))
    res = mc_dropout(model, d["src"], d["static"], d["times"], d["lengths"], n_samples=30, seed=11, step=5,
                     return_samples=True)
    bb = AC.batch_bald(res.samples, 3)
    i0 = bb.indices[0].item()
    mi = res.mutual_information.double()
    assert i0 == int(torch.argmax(bb.bald).item())
    assert abs(bb.scores[0].item() - mi[i0].item()) <= SCORE_RTOL * abs(mi[i0].item())
    assert torch.allclose(bb.bald, mi, rtol=0, atol=SCORE_RTOL * mi.abs().max().item())


@pytest.mark.gpu
def test_confident_replicates_do_not_underflow():
    rng = np.random.default_rng(17)
    M, N, C, k = 16, 300, 2, 200
    x = (np.sign(rng.normal(size=(M, N, C))) * 9 + rng.normal(size=(M, N, C))).astype(np.float32)
    got = AC.batch_bald(torch.from_numpy(x).cuda(), k, n_configs=256, seed=3)
    s = got.scores.cpu().numpy()
    assert np.isfinite(s).all() and np.isfinite(got.bald.cpu().numpy()).all()
    idx = got.indices.cpu().numpy()
    assert len(set(idx.tolist())) == k
    ref = AO.batch_bald(x, k, n_configs=256, seed=3, follow=idx)
    assert np.all(np.abs(s - ref["scores"]) <= SCORE_RTOL * np.abs(ref["scores"])), np.max(np.abs(s / ref["scores"] - 1))
    # the case needs the scaled rows: unscaled, some configuration's product of the picks' probabilities under some
    # replicate is below the smallest fp32 denormal (2^-149)
    p, p32 = AO.softmax(x)
    ms = AO.sample_replicates(M, 256, 3, 0)
    logprod = np.zeros((256, M))
    for j, a in enumerate(idx):
        if not ref["exact"][j]:
            logprod += np.log(p[:, a, :].T[AO.draw_labels(p32, ms, a, j, 3, 0)])
    assert logprod.min() < -149 * np.log(2.0)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [2, 3, 8])
def test_badge_matches_the_oracle(C):
    rng = np.random.default_rng(40 + C)
    N, F, k = 500, 40, 30
    h = np.maximum(rng.normal(size=(N, F)), 0).astype(np.float32)
    z = (rng.normal(size=(N, C)) * 2).astype(np.float32)
    got = AC.badge_from_features(torch.from_numpy(h).cuda(), torch.from_numpy(z).cuda(), k, seed=9, step=2)
    ref = AO.badge(h, z, k, seed=9, step=2)
    assert np.all(ref["margins"][1:] > 1e-9)
    assert np.array_equal(got.indices.cpu().numpy(), ref["indices"])
    d2 = got.d2.cpu().numpy()
    assert np.isinf(d2[0])
    assert np.all(np.abs(d2[1:] - ref["d2"][1:]) <= 1e-10 * ref["d2"][1:])


@pytest.mark.gpu
def test_badge_all_zero_distances_take_the_lowest_unchosen_index():
    h = torch.ones(6, 4, device="cuda")
    z = torch.tensor([[1.0, 0.0]] * 6, device="cuda")              # six identical embeddings
    got = AC.badge_from_features(h, z, 4)
    assert got.indices.tolist() == [0, 1, 2, 3]
    assert got.d2[1:].tolist() == [0.0, 0.0, 0.0]


@pytest.mark.gpu
def test_bitwise_invariant_to_internal_batch_size_and_graph_replay():
    x = torch.from_numpy(_logits(24, 333, 2, seed=8)).cuda()
    runs = [AC.batch_bald(x, 9, n_configs=32, seed=1, internal_batch_size=b) for b in (None, 1, 7, 64, 1000)]
    for r in runs[1:]:
        for f in ("indices", "scores", "exact", "bald"):
            assert torch.equal(getattr(r, f), getattr(runs[0], f)), f
    h = torch.from_numpy(np.maximum(np.random.default_rng(2).normal(size=(333, 24)), 0).astype(np.float32)).cuda()
    z = x[0].contiguous()
    eager_b = AC.badge_from_features(h, z, 12, seed=4)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        AC.batch_bald(x, 9, n_configs=32, seed=1, internal_batch_size=7)
        AC.badge_from_features(h, z, 12, seed=4)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cap = AC.batch_bald(x, 9, n_configs=32, seed=1, internal_batch_size=7)
        cap_b = AC.badge_from_features(h, z, 12, seed=4)
    for t in (cap.indices, cap.scores, cap_b.indices, cap_b.d2):
        t.fill_(0)
    g.replay()
    torch.cuda.synchronize()
    for f in ("indices", "scores", "exact", "bald"):
        assert torch.equal(getattr(cap, f), getattr(runs[0], f)), f
    assert torch.equal(cap_b.indices, eager_b.indices) and torch.equal(cap_b.d2, eager_b.d2)


@pytest.mark.gpu
def test_pool_logits_and_badge_over_an_unlabelled_pool():
    from raindrop_b200 import laplace as LA
    from raindrop_b200 import swag as SW
    from raindrop_b200.data import DeviceDataset
    from raindrop_b200.ood import features
    from raindrop_b200.uncertainty import mc_dropout
    cfg = model_config("TINY", dropout=0.2)
    model = build_dropin(cfg, 21).eval()
    model._plan.obprop_mode = EXACT
    d = to_dev(make_batch(cfg, 23, seed=6))
    ds = DeviceDataset(d["src"], d["static"], d["times"], None)
    sel = torch.tensor([3, 0, 22, 5, 9, 14, 1, 7, 18, 11])
    plan = model._prepare(d["src"].device)
    params = [p.detach().clone() for p in model.parameters()]
    rng = plan.rng_state.clone()

    def part(lo, hi):
        ix = sel[lo:hi].cuda()
        return d["src"][:, ix], d["static"][ix], d["times"][:, ix], d["lengths"][ix]

    got = AC.pool_logits(model, (ds, sel), n_samples=5, seed=3, step=2, batch_size=4)
    want = torch.cat([mc_dropout(model, *part(i, i + 4), n_samples=5, seed=3, step=2, return_samples=True).samples
                      for i in (0, 4, 8)], dim=1)
    assert got.shape == (5, 10, cfg["n_classes"]) and torch.equal(got, want)
    post = SW.SWAG(model, rank=2)
    post.collect(model)
    got = AC.pool_logits(model, (ds, sel), posterior=[post, post], n_samples=3, seed=1, batch_size=6)
    want = torch.cat([SW.swag_predictive(model, [post, post], *part(i, i + 6), n_samples=3, seed=1,
                                         return_samples=True).samples for i in (0, 6)], dim=1)
    assert got.shape[0] == 6 and torch.equal(got, want)
    la = LA.laplace_fit(model, dict(src=d["src"], static=d["static"], times=d["times"], lengths=d["lengths"], y=d["y"]))
    got = AC.pool_logits(model, ds, posterior=la, n_samples=4, seed=2, batch_size=100)
    want = LA.laplace_predictive(model, la, d["src"], d["static"], d["times"], d["lengths"], link="mc", n_samples=4,
                                 seed=2, return_samples=True).samples
    assert torch.equal(got, want)
    res = AC.badge(model, (ds, sel), 4, seed=5)
    h, z = features(model, *part(0, 10))
    ref = AC.badge_from_features(h, z, 4, seed=5)
    assert torch.equal(res.indices, ref.indices) and torch.equal(res.d2, ref.d2)
    assert torch.equal(AC.badge(model, (ds, sel), 4, seed=5, internal_batch_size=3).indices, ref.indices)
    assert torch.equal(plan.rng_state, rng) and not model.training
    assert all(torch.equal(p, q) for p, q in zip(model.parameters(), params))
    assert all(p.grad is None for p in model.parameters())


@pytest.mark.gpu
def test_full_size_p19_pool():
    M, N, C, k = 100, 31_000, 2, 100
    x = torch.from_numpy(_logits(M, N, C, seed=19, scale=1.5)).cuda()
    AC.batch_bald(x, 2)                                              # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = AC.batch_bald(x, k)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    idx = res.indices.cpu().numpy()
    s = res.scores.cpu().numpy()
    assert len(set(idx.tolist())) == k and np.isfinite(s).all()
    assert res.exact.cpu().numpy().tolist() == [C ** i <= 10_000 for i in range(k)]
    assert idx[0] == int(torch.argmax(res.bald).item()) and s[0] == res.bald.max().item()
    assert np.all(np.diff(s[:14]) > 0)                              # exact joint MI grows with the batch
    h = torch.relu(torch.randn(N, 64, device="cuda"))
    bg = AC.badge_from_features(h, x[0].contiguous(), k, seed=1)
    assert len(set(bg.indices.tolist())) == k and torch.isfinite(bg.d2[1:]).all()
    print("batch_bald P19 N=%d M=%d k=%d: %.3f s" % (N, M, k, dt))
