"""Randomized ablation of Raindrop_v2 (raindrop_b200.ablation, rd_raindrop_v2_ablation_counts).

CPU: the exported symbols, the scratch query, the host argument checks, a numpy restatement of the subset streams
(Philox words, Lemire's bounded integer, partial Fisher-Yates, lexicographic unranking) and both certificates against
brute-force exact evaluations.  GPU: the keep tables and ablated rows against the restatement, the votes against the
module's argmax on exactly those rows, keep = P, chunking and key algebra, CUDA-graph replay, certify / predict against
the host statistics, the soundness of the exact certificate under real changes of the certified number of players, a
LARGE call with P = 129, and AblationTrainStep against TrainStep.  Every GPU test pins plan.obprop_mode."""
import ctypes as C
import itertools
import math
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest
import torch

from helpers import build_dropin, to_dev
from raindrop_b200 import ablation as AB
from raindrop_b200.synth import make_batch, model_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXACT, FAST = 2, 1
SITE_ABLATE = 101
SEED = 0x2B7E151628AED2A6
CASES = {
    "tiny_b6": ("TINY", 6, {}),
    "tiny8_b5": ("TINY8", 5, {}),                       # no statics
    "p19_b9": ("P19", 9, {"first_time_zero": True}),    # padded rows
    "p12_b3": ("P12", 3, {}),                           # T = 215
    "pam_b2": ("PAM", 2, {}),                           # T = 600
}


# ---- numpy restatement ------------------------------------------------------------------------------------------------
def _words(seed, step, b, j0, n):
    """Words j0 .. j0+n-1 (j0 % 4 == 0) of sample b's stream at key (seed, step): index (b << 32) + j, word index & 3
    of the Philox block at counter index >> 2, site 101."""
    from oracle.dropout_masks import philox4x32_10
    seed, step = int(seed), int(step) & 0xFFFFFFFFFFFFFFFF
    blk = np.uint64((int(b) << 30) + j0 // 4) + np.arange((n + 3) // 4, dtype=np.uint64)
    ctr = np.stack([blk & np.uint64(0xFFFFFFFF), blk >> np.uint64(32), np.full_like(blk, SITE_ABLATE),
                    np.full_like(blk, step & 0xFFFFFFFF)], -1)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) ^ (step >> 32)], dtype=np.uint64)
    return [int(w) for w in philox4x32_10(ctr, key).reshape(-1)[:n]]


class _Stream:
    def __init__(self, seed, step, b, words=None):
        self.seed, self.step, self.b = seed, step, b
        self.buf = list(words) if words is not None else []
        self.j = 0

    def next(self):
        if self.j == len(self.buf):
            self.buf += _words(self.seed, self.step, self.b, len(self.buf), 16)
        self.j += 1
        return self.buf[self.j - 1]


def lemire(stream, r):
    """Lemire's unbiased integer in [0, r) with rejection, as the keep kernel draws it."""
    x = stream.next() * r
    if x & 0xFFFFFFFF < r:
        t = ((1 << 32) - r) % r
        while x & 0xFFFFFFFF < t:
            x = stream.next() * r
    return x >> 32


def sampled_keep(seed, step, b, P, k):
    s = _Stream(seed, step, b)
    perm = list(range(P))
    for i in range(k):
        j = i + lemire(s, P - i)
        perm[i], perm[j] = perm[j], perm[i]
    keep = np.zeros(P, np.uint8)
    keep[perm[:k]] = 1
    return keep


def unrank(rank, P, k):
    """The k-subset of lexicographic rank `rank` of range(P) (itertools.combinations order); none for rank >= C(P, k)."""
    keep = np.zeros(P, np.uint8)
    if rank >= math.comb(P, k):
        return keep
    x = 0
    for i in range(k):
        while rank >= math.comb(P - x - 1, k - i - 1):
            rank -= math.comb(P - x - 1, k - i - 1)
            x += 1
        keep[x] = 1
        x += 1
    return keep


def keep_table(B, P, k, m_range, seed, step, exhaustive):
    """[len(m_range) * B, P] uint8, row (m - m0)*B + b."""
    rows = [unrank(step + m, P, k) if exhaustive else sampled_keep(seed, step + m, b, P, k)
            for m in m_range for b in range(B)]
    return np.stack(rows)


def ablated_inputs(src, static, keep, sensors, ablate_static, ablate_mask):
    """The rows of keep [B, P] applied to one copy of the batch (src [T, B, 2N], static [B, ds] or None)."""
    src = np.asarray(src, dtype=np.float32).copy()
    N = src.shape[2] // 2
    players = np.arange(N) if sensors is None else np.flatnonzero(np.asarray(sensors))
    for p, n in enumerate(players):
        gone = keep[:, p] == 0
        src[:, gone, n] = 0.0
        if ablate_mask:
            src[:, gone, N + n] = 0.0
    st = None if static is None else np.asarray(static, dtype=np.float32).copy()
    if ablate_static:
        st[keep[:, -1] == 0] = 0.0
    return src, st


# ---- CPU --------------------------------------------------------------------------------------------------------------
def test_symbols_exported():
    lib_path = os.path.join(ROOT, "raindrop_b200", "csrc", "librd_b200.so")
    out = subprocess.run(["nm", "-D", "--defined-only", lib_path], capture_output=True, text=True, check=True).stdout
    names = {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert {"rd_ablation_scratch_bytes", "rd_raindrop_v2_ablation_counts", "rd_debug_ablation_inputs"} <= names


def test_scratch_query():
    """The smoothing layout (chunk_layout) plus the keep table [cc*B, P] bytes, in 64-float pieces; 0 when invalid."""
    from raindrop_b200 import lib as L
    lib = L.load()
    for name in ("TINY", "TINY8", "P19", "P12", "PAM"):
        cfg = model_config(name, dropout=0.2)
        model = build_dropin(cfg, 1, device="cpu")
        for B in (1, 5, 128):
            dims = model._plan.dims(B, False)
            for cc in (1, 7, 64):
                base = lib.rd_smooth_scratch_bytes(C.byref(dims), cc)
                for P in (1, 5, 37, 129):
                    table = -(-cc * B * P // 4)
                    want = base + -(-table // 64) * 64 * 4
                    assert lib.rd_ablation_scratch_bytes(C.byref(dims), P, cc) == want, (name, B, cc, P)
            for P, cc in ((0, 1), (-1, 1), (L.ABLATION_MAX_PLAYERS + 1, 1), (5, 0)):
                assert lib.rd_ablation_scratch_bytes(C.byref(dims), P, cc) == 0


def _cpu_model(name="TINY"):
    cfg = model_config(name, dropout=0.2)
    return build_dropin(cfg, 3, device="cpu").eval(), make_batch(cfg, 3, seed=1), cfg


def test_argument_validation():
    model, b, cfg = _cpu_model()
    args = (b["src"], b["static"], b["times"], b["lengths"])
    N = cfg["d_inp"]
    with pytest.raises(ValueError, match="eval"):
        AB.ablation_counts(model.train(), *args, keep=2, n_samples=10)
    model.eval()
    bad = [dict(keep=0), dict(keep=N + 1), dict(keep=N + 2, ablate_static=True), dict(keep=3, sensors=np.arange(N) < 2),
           dict(keep=1, sensors=np.ones(N + 1, bool)), dict(keep=1, sensors=np.ones(N, np.int64)),
           dict(keep=1, sensors=np.zeros(N, bool)), dict(keep=2, n_samples=0), dict(keep=2, n_samples=None),
           dict(keep=2, internal_batch_size=0), dict(keep=2, seed=-1), dict(keep=2, step=(1 << 64) - 5),
           dict(keep=2, exhaustive=True, n_samples=math.comb(N, 2) + 1),
           dict(keep=2, exhaustive=True, step=3, n_samples=math.comb(N, 2) - 2),
           dict(keep=2, exhaustive=True, step=math.comb(N, 2))]
    for kw in bad:
        kw.setdefault("n_samples", 10)
        with pytest.raises(ValueError):
            AB.ablation_counts(model, *args, **kw)
    with pytest.raises(ValueError, match="2\\^31"):
        AB._check_subsets(129, 64)
    assert AB._check_subsets(34, 5) == math.comb(34, 5)
    for alpha in (0.0, 1.0, float("nan")):
        with pytest.raises(ValueError):
            AB.certify(model, *args, keep=2, alpha=alpha)
        with pytest.raises(ValueError):
            AB.predict(model, *args, keep=2, alpha=alpha)
    for kw in (dict(n0=0), dict(n_samples=0), dict(keep=7)):
        kw.setdefault("keep", 2)
        with pytest.raises(ValueError):
            AB.certify(model, *args, **kw)
    with pytest.raises(ValueError):
        AB.certify_from_counts(np.ones((2, 3), np.int64), np.ones((2, 3), np.int64), 5, 6)
    with pytest.raises(ValueError):
        AB.certify_exact_from_counts(np.full((1, 2), 6, np.int64), 4, 2)     # 12 votes > C(4, 2)
    m8, b8, _ = _cpu_model("TINY8")
    with pytest.raises(ValueError, match="static"):
        AB.ablation_counts(m8, b8["src"], None, b8["times"], b8["lengths"], keep=2, n_samples=4, ablate_static=True)


def test_no_cuda_raises(monkeypatch):
    from raindrop_b200.lib import RaindropB200Error
    model, b, _ = _cpu_model()
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RaindropB200Error):
        AB.ablation_counts(model, b["src"], b["static"], b["times"], b["lengths"], keep=2, n_samples=4)


def test_train_step_refused(monkeypatch):
    import torch.distributed as dist
    from raindrop_b200.lib import RaindropB200Error
    cfg = model_config("TINY", dropout=0.2)
    model = build_dropin(cfg, 3, device="cpu")
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    with pytest.raises(RaindropB200Error, match="one GPU"):
        AB.AblationTrainStep(model, 4, keep=2)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 1)
    for kw in (dict(keep=0), dict(keep=6), dict(keep=2, sensors=np.zeros(5, bool))):
        with pytest.raises(ValueError):
            AB.AblationTrainStep(model, 4, **kw)
    m8 = build_dropin(model_config("TINY8", dropout=0.2), 3, device="cpu")
    with pytest.raises(ValueError, match="static"):
        AB.AblationTrainStep(m8, 4, keep=2, ablate_static=True)


def test_fisher_yates_is_uniform():
    """All 15 subsets of C(6, 2) from the restated stream: a chi-square test at 8,000 rows over (b, step)."""
    from scipy.stats import chisquare
    P, k = 6, 2
    index = {c: i for i, c in enumerate(itertools.combinations(range(P), k))}
    hits = np.zeros(len(index), np.int64)
    for step in range(40):
        for b in range(200):
            hits[index[tuple(np.flatnonzero(sampled_keep(SEED, step, b, P, k)))]] += 1
    assert hits.sum() == 8000 and hits.min() > 0
    assert chisquare(hits).pvalue > 1e-3
    # rows differ across samples and steps: the stream is indexed by (b, step)
    assert not np.array_equal(sampled_keep(SEED, 0, 0, 19, 5), sampled_keep(SEED, 0, 1, 19, 5)) or \
        not np.array_equal(sampled_keep(SEED, 0, 0, 19, 5), sampled_keep(SEED, 1, 0, 19, 5))


def test_lemire_rejection_branch():
    """P = 19 and P - i for every i are not powers of two: a low word below 2^32 mod r is rejected and the next word
    drawn; otherwise the high word of x * r is the draw."""
    for r in (3, 19, 18, 129, 1000003):
        t = ((1 << 32) - r) % r
        assert t > 0
        w_acc = 0xDEADBEEF
        s = _Stream(0, 0, 0, [0, w_acc])          # word 0: x = 0, low word 0 < t -> rejected
        assert lemire(s, r) == (w_acc * r) >> 32 and s.j == 2
        s = _Stream(0, 0, 0, [w_acc])
        assert lemire(s, r) == (w_acc * r) >> 32 and s.j == 1
    assert lemire(_Stream(0, 0, 0, [0]), 1) == 0           # r = 1 consumes one word and returns 0
    # the bounded integer is uniform on [0, r) for a non-power of two
    s = _Stream(SEED, 3, 7)
    draws = np.array([lemire(s, 19) for _ in range(19 * 400)])
    assert draws.min() == 0 and draws.max() == 18
    from scipy.stats import chisquare
    assert chisquare(np.bincount(draws, minlength=19)).pvalue > 1e-3


@pytest.mark.parametrize("P,k", [(1, 1), (5, 1), (5, 5), (6, 2), (7, 3), (10, 4), (12, 6)])
def test_unrank_is_itertools_order(P, k):
    combos = list(itertools.combinations(range(P), k))
    for rank, c in enumerate(combos):
        assert tuple(np.flatnonzero(unrank(rank, P, k))) == c
    assert not unrank(len(combos), P, k).any()


def _brute_sampled(p_lower, P, k):
    """Largest rho with ceil(p_lower J)/J - Delta(rho) > 1/2, Delta(rho) = 1 - C(P - rho, k)/C(P, k), in Fractions."""
    J = math.comb(P, k)
    p = Fraction(math.ceil(Fraction(float(p_lower)) * J), J)
    best = -1
    for rho in range(P - k + 1):
        if p - (1 - Fraction(math.comb(P - rho, k), J)) > Fraction(1, 2):
            best = rho
    return best


def test_sampled_certificate_against_brute_force():
    from scipy.stats import beta
    alpha, n = 0.001, 1000
    rng = np.random.default_rng(0)
    for P, k in ((6, 2), (12, 1), (19, 5), (34, 5), (7, 7)):
        ks = np.concatenate([[0, n], rng.integers(400, n, size=40)])
        c = np.stack([ks, n - ks], 1).astype(np.int64)
        c0 = np.tile(np.array([[3, 1]], np.int64), (len(ks), 1))
        pred, radius, pl = AB.certify_from_counts(c0, c, P, k, alpha, n=n)
        for i in range(len(ks)):
            want = _brute_sampled(pl[i], P, k)
            assert radius[i] == want and pred[i] == (0 if want >= 0 else -1), (P, k, ks[i])
            if ks[i] > 0:
                assert pl[i] == pytest.approx(beta.ppf(alpha, ks[i], n - ks[i] + 1), rel=1e-12)
        assert pred[0] == -1 and radius[0] == -1                 # n_A = 0: p_lower = 0
        if k == P:
            assert radius.max() <= 0                             # keep = P certifies rho = 0 at most
    # ties in the selection: c_A = the lowest index
    pred, _, _ = AB.certify_from_counts(np.array([[5, 5]]), np.array([[990, 10]]), 6, 2, alpha)
    assert pred[0] == 0
    pred, _, _ = AB.certify_from_counts(np.array([[5, 5]]), np.array([[10, 990]]), 6, 2, alpha)
    assert pred[0] == -1


def test_sampled_certificate_boundary_and_rounding(monkeypatch):
    """2j = J + 2 Delta_n exactly does not certify; one more j does.  Rounding p_lower up to a multiple of 1/J
    certifies radii that the unrounded bound does not."""
    P, k = 6, 2
    J = math.comb(P, k)                                          # 15
    for rho in range(P - k + 1):
        dn = J - math.comb(P - rho, k)
        if (J + 2 * dn) % 2:
            continue
        j = (J + 2 * dn) // 2
        for jj, want in ((j, rho - 1), (j + 1, rho)):
            if jj > J:
                continue
            monkeypatch.setattr(AB, "selection_lower_bound",
                                lambda c0, c, a, n=None, jj=jj: (np.array([0]), np.array([(jj - 0.5) / J])))
            _, radius, _ = AB.certify_from_counts(np.array([[1, 0]]), np.array([[1, 0]]), P, k)
            assert radius[0] == max(want, -1), (rho, jj)
    monkeypatch.undo()
    # rounding: a count whose p_lower lies strictly between two multiples of 1/J certifies as the upper one
    found = False
    n, alpha = 500, 0.001
    for kA in range(300, n + 1):
        _, radius, pl = AB.certify_from_counts(np.array([[1, 0]]), np.array([[kA, n - kA]]), P, k, alpha)
        unrounded = -1
        for rho in range(P - k + 1):
            if Fraction(float(pl[0])) - (1 - Fraction(math.comb(P - rho, k), J)) > Fraction(1, 2):
                unrounded = rho
        assert radius[0] >= unrounded
        found |= radius[0] > unrounded
    assert found


def _brute_exact(counts, P, k):
    """For every set R of rho players, the subsets meeting R (enumerated) can each move one vote from c_A to any c."""
    subsets = list(itertools.combinations(range(P), k))
    J = len(subsets)
    out = []
    for row in counts:
        ca = int(np.argmax(row))
        if row[ca] == 0:
            out.append((-1, -1))
            continue
        best = -1
        for rho in range(P - k + 1):
            ok = True
            for R in itertools.combinations(range(P), rho):
                dn = sum(1 for s in subsets if set(s) & set(R))
                assert dn == J - math.comb(P - rho, k)
                for c in range(len(row)):
                    if c != ca:
                        a, o = int(row[ca]) - dn, int(row[c]) + dn
                        ok &= a > o or (a == o and ca < c)
                break                                            # every R of the same size meets as many subsets
            if not ok:
                break
            best = rho
        out.append((ca, best))
    return out


def test_exact_certificate_against_brute_force():
    P, k = 6, 2                                                  # J = 15, Delta_n(rho) = 0, 5, 9, 12, 14
    counts = np.array([[15, 0, 0],        # unanimous
                       [0, 0, 0],         # every vote invalid: abstain
                       [10, 5, 0],        # n_A - n_c = 5
                       [5, 5, 5],         # three-way tie: c_A = 0 wins ties, rho = 0
                       [5, 10, 0],        # c_A = 1
                       [8, 7, 0],
                       [12, 2, 1],
                       [3, 3, 9],         # tie in the runners-up
                       [14, 0, 0]], dtype=np.int64)      # one invalid vote
    pred, radius = AB.certify_exact_from_counts(counts, P, k)
    assert list(zip(pred.tolist(), radius.tolist())) == _brute_exact(counts, P, k)
    assert radius[0] == 1 and pred[1] == -1 and radius[3] == 0     # rho = 2 meets 9 of the 15 subsets
    # equality n_A - dn == n_c + dn certifies only when c_A < c
    J = 15
    dn1 = J - math.comb(P - 1, k)                                # 5
    pred, radius = AB.certify_exact_from_counts(np.array([[2 * dn1, 0], [0, 2 * dn1]]), P, k)
    assert radius.tolist() == [1, 0]
    pred, radius = AB.certify_exact_from_counts(np.array([[2 * dn1 + 1, 1], [1, 2 * dn1 + 1]]), P, k)
    assert radius.tolist() == [1, 0]
    pred, radius = AB.certify_exact_from_counts(np.array([[2 * dn1 + 2, 1], [1, 2 * dn1 + 2]]), P, k)
    assert radius.tolist() == [1, 1]
    pred, radius = AB.certify_exact_from_counts(np.array([[2 * dn1 - 1, 0]]), P, k)
    assert radius.tolist() == [0]
    pred, radius = AB.certify_exact_from_counts(np.array([[1, 0]]), 4, 4)     # keep = P: rho = 0 at most
    assert radius.tolist() == [0]


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


def _players(N, sensors, ast):
    return (N if sensors is None else int(np.asarray(sensors).sum())) + int(ast)


def _inputs(model, d, keep, seed, step, m0, nc, sensors=None, ast=False, amask=True, exhaustive=False):
    """rd_debug_ablation_inputs: the keep table and rows of replicates m0 .. m0+nc-1 at key (seed, step)."""
    from raindrop_b200 import lib as L
    from raindrop_b200.adversarial import _sensor_mask
    lib, dev = L.load(), torch.device("cuda", torch.cuda.current_device())
    plan = model._prepare(dev)
    T, B, N2 = d["src"].shape
    P = _players(N2 // 2, None if sensors is None else sensors.cpu(), ast)
    dims = plan.dims(B, False)
    key = torch.tensor(np.array([seed, step], dtype=np.uint64).view(np.int64), device=dev)
    sens = _sensor_mask(sensors, N2 // 2, dev)
    table = torch.empty(nc * B, P, dtype=torch.uint8, device=dev)
    src_e = torch.empty(T, nc * B, N2, device=dev)
    st_e = torch.empty(nc * B, d["static"].shape[1], device=dev) if d["static"] is not None else None
    tm_e = torch.empty(T, nc * B, device=dev)
    ln_e = torch.empty(nc * B, dtype=torch.int64, device=dev)
    L.check(lib.rd_debug_ablation_inputs(C.byref(dims), d["src"].data_ptr(), L.ptr(d["static"]), d["times"].data_ptr(),
                                         d["lengths"].data_ptr(), L.ptr(sens), P, int(ast), int(amask), keep,
                                         int(exhaustive), key.data_ptr(), m0, nc, table.data_ptr(), src_e.data_ptr(),
                                         L.ptr(st_e), tm_e.data_ptr(), ln_e.data_ptr(), L.stream_ptr(dev)),
            "rd_debug_ablation_inputs")
    return table, src_e, st_e, tm_e, ln_e


@pytest.mark.gpu
@pytest.mark.parametrize("amask", [True, False], ids=["mask", "values"])
@pytest.mark.parametrize("exhaustive", [False, True], ids=["sampled", "exhaustive"])
@pytest.mark.parametrize("name", list(CASES))
def test_inputs_match_restatement(name, exhaustive, amask):
    cfg, d, model = _setup(name)
    N, B = cfg["d_inp"], d["src"].shape[1]
    ast = d["static"] is not None
    for sensors in (torch.arange(N) % 3 != 1, None):
        P = _players(N, sensors, ast)
        k = max(1, P // 3)
        m0, nc, step = (1, 2, 0) if exhaustive else (3, 2, 5)
        table, src_e, st_e, tm_e, ln_e = _inputs(model, d, k, SEED, step, m0, nc, sensors, ast, amask, exhaustive)
        want_keep = keep_table(B, P, k, range(m0, m0 + nc), SEED, step, exhaustive)
        assert np.array_equal(table.cpu().numpy(), want_keep)
        assert (want_keep.sum(1) == k).all()
        x = d["src"].cpu().numpy()
        st = None if d["static"] is None else d["static"].cpu().numpy()
        for m in range(nc):
            rows = slice(m * B, (m + 1) * B)
            want, want_st = ablated_inputs(x, st, want_keep[rows], None if sensors is None else sensors.numpy(), ast,
                                           amask)
            assert np.array_equal(src_e[:, rows].cpu().numpy().view(np.int32), want.view(np.int32))
            assert torch.equal(tm_e[:, rows], d["times"]) and torch.equal(ln_e[rows], d["lengths"])
            if st is not None:
                assert np.array_equal(st_e[rows].cpu().numpy().view(np.int32), want_st.view(np.int32))
        # the same replicates under another chunking: key (seed, step + m0) with m0 = 0
        again = _inputs(model, d, k, SEED, step + m0, 0, nc, sensors, ast, amask, exhaustive)
        assert torch.equal(again[0], table) and torch.equal(again[1], src_e)
    # exhaustive: a rank >= J keeps no player
    if exhaustive:
        P = _players(N, None, False)
        table = _inputs(model, d, 1, SEED, P - 1, 0, 2, None, False, amask, True)[0]
        assert table[:B].sum() == B and table[B:].sum() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("exhaustive", [False, True], ids=["sampled", "exhaustive"])
@pytest.mark.parametrize("name", list(CASES))
def test_votes_are_module_argmax(name, exhaustive):
    cfg, d, model = _setup(name)
    B, N = d["src"].shape[1], cfg["d_inp"]
    ast = d["static"] is not None
    P = N + int(ast)
    k, n = 2, 6
    counts = AB.ablation_counts(model, *_args(d), keep=k, n_samples=n, seed=SEED, step=2, exhaustive=exhaustive,
                                ablate_static=ast, internal_batch_size=B * n)
    _, src_e, st_e, tm_e, ln_e = _inputs(model, d, k, SEED, 2, 0, n, None, ast, True, exhaustive)
    with torch.no_grad():
        logits = model.forward(src_e, st_e, tm_e, ln_e)[0]
    assert torch.isfinite(logits).all()
    votes = logits.argmax(1).view(n, B)
    want = torch.zeros_like(counts)
    for b in range(B):
        want[b] = torch.bincount(votes[:, b], minlength=cfg["n_classes"])
    assert torch.equal(counts, want) and P >= k


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_keep_all_votes_the_clean_class(name):
    cfg, d, model = _setup(name)
    ast = d["static"] is not None
    P = cfg["d_inp"] + int(ast)
    with torch.no_grad():
        clean = model.forward(*_args(d))[0].argmax(1)
    for exhaustive, n in ((False, 5), (True, None)):
        counts = AB.ablation_counts(model, *_args(d), keep=P, n_samples=n, exhaustive=exhaustive, ablate_static=ast)
        want = torch.zeros_like(counts)
        want[torch.arange(len(clean)), clean] = 5 if n else 1
        assert torch.equal(counts, want)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_chunking_key_algebra_graph_and_no_side_effects(name):
    cfg, d, model = _setup(name, FAST)
    B, N = d["src"].shape[1], cfg["d_inp"]
    n, a = 12, 5
    plan = model._prepare(torch.device("cuda"))
    snap = {"rng": plan.rng_state.clone()}
    snap.update({"param." + k: p.detach().clone() for k, p in model.named_parameters()})
    kw = dict(keep=2, seed=SEED, ablate_static=d["static"] is not None, sensors=torch.arange(N) != 1)
    res = [AB.ablation_counts(model, *_args(d), n_samples=n, step=4, internal_batch_size=ib, **kw)
           for ib in (B, 7 * B, n * B, n * B)]
    for r in res[1:]:
        assert torch.equal(r, res[0])
    split = (AB.ablation_counts(model, *_args(d), n_samples=a, step=4, internal_batch_size=3 * B, **kw) +
             AB.ablation_counts(model, *_args(d), n_samples=n - a, step=4 + a, internal_batch_size=2 * B, **kw))
    assert torch.equal(split, res[0])
    # exhaustive: the whole enumeration equals two calls that split it, and every sample has J votes
    ekw = dict(kw, exhaustive=True)
    full = AB.ablation_counts(model, *_args(d), internal_batch_size=5 * B, **ekw)
    J = math.comb(N - 1 + int(kw["ablate_static"]), 2)
    assert torch.equal(full.sum(1), torch.full((B,), J, device="cuda"))
    half = J // 2
    two = (AB.ablation_counts(model, *_args(d), n_samples=half, internal_batch_size=2 * B, **ekw) +
           AB.ablation_counts(model, *_args(d), step=half, internal_batch_size=3 * B, **ekw))
    assert torch.equal(two, full)
    # CUDA graph: capture after an eager call with the same key and shapes; a later eager call does not disturb it
    gkw = dict(n_samples=n, step=4, internal_batch_size=7 * B, **kw)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eager = AB.ablation_counts(model, *_args(d), **gkw)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = AB.ablation_counts(model, *_args(d), **gkw)
    AB.ablation_counts(model, *_args(d), n_samples=3, step=9, internal_batch_size=B, **kw)
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
    N = cfg["d_inp"]
    ast = d["static"] is not None
    P, k, n0, n, alpha = N + int(ast), 2, 20, 200, 0.01
    kw = dict(keep=k, ablate_static=ast)
    r = AB.certify(model, *_args(d), n0=n0, n_samples=n, alpha=alpha, seed=3, step=7, **kw)
    c0 = AB.ablation_counts(model, *_args(d), n_samples=n0, seed=3, step=7, **kw)
    c = AB.ablation_counts(model, *_args(d), n_samples=n, seed=3, step=7 + n0, **kw)
    assert torch.equal(r.counts0, c0) and torch.equal(r.counts, c)
    pred, radius, pl = AB.certify_from_counts(c0, c, P, k, alpha, n=n)
    assert np.array_equal(r.prediction, pred) and np.array_equal(r.radius, radius) and np.array_equal(r.p_lower, pl)
    assert r.n_players == P and r.keep == k
    p = AB.predict(model, *_args(d), n_samples=n, alpha=alpha, seed=3, step=7, **kw)
    assert np.array_equal(p, AB.predict_from_counts(AB.ablation_counts(model, *_args(d), n_samples=n, seed=3, step=7,
                                                                       **kw), alpha))
    e = AB.certify(model, *_args(d), exhaustive=True, **kw)
    ce = AB.ablation_counts(model, *_args(d), exhaustive=True, **kw)
    assert torch.equal(e.counts, ce) and np.isnan(e.p_lower).all()
    pe, re = AB.certify_exact_from_counts(ce, P, k)
    assert np.array_equal(e.prediction, pe) and np.array_equal(e.radius, re)


@pytest.mark.gpu
@pytest.mark.parametrize("amask", [True, False], ids=["mask", "values"])
@pytest.mark.parametrize("name", ["tiny_b6", "p19_b9"])
def test_exact_certificate_is_sound(name, amask):
    """For every sample certified at rho >= 1, overwrite the data of rho players (several random choices of players,
    values and masks), enumerate again: the prediction does not change."""
    cfg, d, model = _setup(name)
    N, B = cfg["d_inp"], d["src"].shape[1]
    ast = d["static"] is not None
    sensors = torch.arange(N) < min(N, 12)
    players = np.flatnonzero(sensors.numpy())
    P, keep = len(players) + int(ast), 1
    kw = dict(keep=keep, exhaustive=True, sensors=sensors, ablate_static=ast, ablate_mask=amask)
    r = AB.certify(model, *_args(d), **kw)
    assert (r.radius >= 1).any()
    gen = np.random.default_rng(5)
    T = d["src"].shape[0]
    checked = 0
    for b in np.flatnonzero(r.radius >= 1):
        rho = int(r.radius[b])
        for _ in range(3):
            src, st = d["src"].clone(), None if d["static"] is None else d["static"].clone()
            for p in gen.choice(P, size=rho, replace=False):
                if p == P - 1 and ast:
                    st[b] = torch.from_numpy(gen.normal(0, 3, st.shape[1]).astype(np.float32)).cuda()
                    continue
                n = players[p]
                src[:, b, n] = torch.from_numpy(gen.normal(0, 3, T).astype(np.float32)).cuda()
                if amask:
                    src[:, b, N + n] = torch.from_numpy((gen.random(T) < 0.5).astype(np.float32)).cuda()
            r2 = AB.certify(model, src, st, d["times"], d["lengths"], **kw)
            assert r2.prediction[b] == r.prediction[b], (b, rho)
            checked += 1
    assert checked > 0


@pytest.mark.gpu
def test_large_shape_129_players():
    cfg = model_config("LARGE", dropout=0.2)
    B = 2
    d = to_dev(make_batch(cfg, B, seed=3))
    model = build_dropin(cfg, 9).eval()
    model._plan.obprop_mode = FAST
    P, k, n = cfg["d_inp"] + 1, 64, 6
    assert P == 129
    counts = AB.ablation_counts(model, *_args(d), keep=k, n_samples=n, seed=SEED, step=1, ablate_static=True)
    assert torch.equal(counts.sum(1), torch.full((B,), n, device="cuda"))
    table, src_e, st_e, _, _ = _inputs(model, d, k, SEED, 1, 0, 2, None, True)
    want = keep_table(B, P, k, range(2), SEED, 1, False)
    assert np.array_equal(table.cpu().numpy(), want)
    x, st = d["src"].cpu().numpy(), d["static"].cpu().numpy()
    w, ws = ablated_inputs(x, st, want[:B], None, True, True)
    assert np.array_equal(src_e[:, :B].cpu().numpy().view(np.int32), w.view(np.int32))
    assert np.array_equal(st_e[:B].cpu().numpy().view(np.int32), ws.view(np.int32))


# ---- ablation training ------------------------------------------------------------------------------------------------
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
def test_ablation_step_keeping_every_player_is_train_step(use_graph):
    from raindrop_b200.train import TrainStep
    cfg = model_config("P19", dropout=0.2)
    B = 37
    batch = to_dev(make_batch(cfg, B, seed=5, first_time_zero=True))
    out = []
    for ablate in (False, True):
        model = _train_model(cfg)
        s = AB.AblationTrainStep(model, B, keep=cfg["d_inp"] + 1, ablate_static=True, noise_seed=3,
                                 use_graph=use_graph) if ablate else TrainStep(model, B, use_graph=use_graph)
        s.load_batch(batch)
        out.append(_run(s, 3))
    for a, b in zip(*out):
        assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("name", ["tiny_b6", "tiny8_b5"])
def test_ablation_step_is_train_step_on_ablated_batch(use_graph, name):
    """One step from a given state equals TrainStep on the batch exported for the step's key; the key advances by one
    per step; restoring the state and the key replays the step."""
    from raindrop_b200.train import TrainStep
    cfg_name, B, _ = CASES[name]
    cfg = model_config(cfg_name, dropout=0.2)
    batch = to_dev(make_batch(cfg, B, seed=7))
    N = cfg["d_inp"]
    sensors = torch.arange(N) % 3 != 2
    ast = batch["static"] is not None
    keep = 2
    model = _train_model(cfg)
    s = AB.AblationTrainStep(model, B, keep=keep, sensors=sensors, ablate_static=ast, noise_seed=SEED,
                             use_graph=use_graph, lr=1e-3)
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
    table, src_e, st_e, _, _ = _inputs(ref_model, batch, keep, SEED, 5, 0, 1, sensors, ast)
    ref.load_batch(dict(batch, src=src_e, static=st_e))
    got = _run(s, 1)
    want = _run(ref, 1)
    for x, y in zip(got, want):
        assert torch.equal(x, y)
    assert torch.equal(s.noisy_src, src_e) and torch.equal(s.keep_table, table)
    assert not torch.equal(s.noisy_src, batch["src"])
    assert s.noise_key_state() == (SEED, 6)
    for t, v in zip(s._state(), state):
        t.copy_(v)
    s.set_noise_key(SEED, 5)
    again = _run(s, 1)
    for x, y in zip(got, again):
        assert torch.equal(x, y)
