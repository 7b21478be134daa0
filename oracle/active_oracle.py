"""TEST INFRASTRUCTURE ONLY -- numpy float64 restatement of raindrop_b200.active (rd_batch_bald, rd_badge).

BatchBALD (Kirsch, van Amersfoort & Gal 2019):
  batch_bald_bruteforce   greedy picks with the joint entropy summed over the full table of all C^|A u {n}| label
                          configurations (exact; for tiny pools).
  batch_bald              the device's algorithm in float64: exact while C^|A| <= n_configs (mixed-radix rows, row j*C + c
                          of A u {n} = row j of A times p[:, n, c]), then Kirsch's importance-weighted estimate over
                          configurations drawn from the same Philox words as the kernels, with the same fp32 inverse CDF,
                          so the configurations are the device's.  Rows are kept scaled to max 1 with an fp64 log-scale,
                          as on the device, so that k = 200 picks stay finite.
BADGE (Ash et al. 2020):
  badge                   k-means++ seeding with the embeddings (p - e_yhat) (x) [h; 1] materialised.

Random words (raindrop_b200/csrc/rd_active.cu): Philox4x32-10 with key (seed lo, seed hi ^ step hi) and counter
(c0, c1, site, step lo); BatchBALD site 105 with (c0, c1) = (configuration, 0) for the replicate draw and
(configuration, j + 1) for the label of the pick of step j; BADGE site 106 with (c0, c1) = (pick, 0).
"""
import numpy as np

from .dropout_masks import philox4x32_10

SITE_BATCHBALD, SITE_BADGE = 105, 106


def active_words(seed, step, site, c0, c1):
    """Philox blocks [..., 4] (uint32) at counters (c0, c1, site, step lo) under key (seed, step); c0, c1 broadcast."""
    seed, step = int(seed) & 0xFFFFFFFFFFFFFFFF, int(step) & 0xFFFFFFFFFFFFFFFF
    c0, c1 = np.broadcast_arrays(np.asarray(c0, dtype=np.uint64), np.asarray(c1, dtype=np.uint64))
    ctr = np.empty(c0.shape + (4,), dtype=np.uint64)
    ctr[..., 0], ctr[..., 1], ctr[..., 2], ctr[..., 3] = c0, c1, site, step & 0xFFFFFFFF
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) ^ (step >> 32)], dtype=np.uint64)
    return philox4x32_10(ctr, key)


def config_counter(s, j):
    """The Philox counter words (c0, c1) of configuration s at draw slot j (0: its replicate; j + 1: its label for the
    pick of step j)."""
    return int(s), int(j)


def softmax(logits):
    """(p float64, p rounded to fp32 as the kernels store it) of logits [..., C]."""
    x = np.asarray(logits, dtype=np.float32).astype(np.float64)
    mx = x.max(axis=-1, keepdims=True)
    lp = (x - mx) - np.log(np.exp(x - mx).sum(axis=-1, keepdims=True))
    p = np.exp(lp)
    return p, p.astype(np.float32)


def expected_entropy(logits):
    """E_m H(y_n | theta_m) [N] of logits [M, N, C]."""
    x = np.asarray(logits, dtype=np.float32).astype(np.float64)
    mx = x.max(axis=-1, keepdims=True)
    lp = (x - mx) - np.log(np.exp(x - mx).sum(axis=-1, keepdims=True))
    return (-(np.exp(lp) * lp).sum(axis=-1)).mean(axis=0)


def _xlogx(q):
    return np.where(q > 0, q * np.log(np.where(q > 0, q, 1.0)), 0.0)


def batch_bald_bruteforce(logits, k):
    """Greedy exact BatchBALD by enumeration of the full joint table: (indices, scores) with scores[i] the joint mutual
    information I(y_A; theta) after pick i.  Ties to the lowest index."""
    p, _ = softmax(logits)
    M, N, C = p.shape
    ce = expected_entropy(logits)
    chosen, scores = [], []
    for _ in range(k):
        best, bv = -1, -np.inf
        for n in range(N):
            if n in chosen:
                continue
            S = chosen + [n]
            joint = np.ones((M,) + (C,) * len(S))
            for d, a in enumerate(S):
                shape = [M] + [1] * len(S)
                shape[1 + d] = C
                joint = joint * p[:, a, :].reshape(shape)
            P = joint.mean(axis=0)
            v = -_xlogx(P).sum() - ce[S].sum()
            if v > bv:
                best, bv = n, v
        chosen.append(best)
        scores.append(bv)
    return np.array(chosen, dtype=np.int64), np.array(scores)


def joint_table_mi(logits, subset):
    """I(y_subset; theta) from the full joint table over ALL N points, marginalised onto `subset` (N <= 6)."""
    p, _ = softmax(logits)
    M, N, C = p.shape
    joint = np.ones((M,) + (C,) * N)
    for a in range(N):
        shape = [M] + [1] * N
        shape[1 + a] = C
        joint = joint * p[:, a, :].reshape(shape)
    P = joint.mean(axis=0)
    other = tuple(a for a in range(N) if a not in subset)
    Ps = P.sum(axis=other) if other else P
    return -_xlogx(Ps).sum() - expected_entropy(logits)[list(subset)].sum()


def sample_replicates(M, n_configs, seed, step):
    """m_s [S]: each configuration's replicate, floor(word M / 2^32)."""
    w0 = active_words(seed, step, SITE_BATCHBALD, np.arange(int(n_configs)), 0)[:, 0].astype(np.uint64)
    return ((w0 * np.uint64(M)) >> np.uint64(32)).astype(np.int64)


def draw_labels(p32, ms, a, j, seed, step):
    """labels [S] of the configurations for the pick `a` of step j: min{c : u < fp32 cumsum_c p[m_s, a, c]}, else the
    largest class with p > 0; u = (word >> 8) 2^-24."""
    S = len(ms)
    w = active_words(seed, step, SITE_BATCHBALD, np.arange(S), j + 1)[:, 0]
    u = (w >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    col = p32[ms, a, :]                                          # [S, C] fp32
    cum = np.cumsum(col, axis=1, dtype=np.float32)               # sequential, in fp32
    hit = u[:, None] < cum
    C = col.shape[1]
    last = C - 1 - np.argmax((col > 0)[:, ::-1], axis=1)
    return np.where(hit.any(axis=1), np.argmax(hit, axis=1), last)


def _scaled(rows, ls):
    mx = rows.max(axis=1)
    ok = mx > 0
    out = np.where(ok[:, None], rows / np.where(ok, mx, 1.0)[:, None], 0.0)
    return out, np.where(ok, ls + np.log(np.where(ok, mx, 1.0)), -np.inf)


def batch_bald(logits, k, n_configs=10_000, seed=0, step=0, follow=None):
    """The device's BatchBALD in float64.  Returns dict(indices, scores, exact, bald, all_scores [k, N] (each step's
    candidate scores, chosen points -inf)).  follow: take these picks instead of the argmax (to compare step by step
    with a run that chose differently)."""
    p, p32 = softmax(logits)
    M, N, C = p.shape
    ce = expected_entropy(logits)
    logM = np.log(M)
    rows, ls, R, exact = np.ones((1, M)), np.zeros(1), 1, True
    w = np.full(1, 1.0 / M)
    chosen = np.zeros(N, dtype=bool)
    condA = 0.0
    idx, scores, exs, all_scores, bald = [], [], [], [], None
    ms = None
    for i in range(k):
        Q = np.einsum("rm,mnc->rnc", rows, p)                       # [R, N, C]
        L = (ls - logM)[:, None, None]
        v = np.where(Q > 0, Q * (L + np.log(np.where(Q > 0, Q, 1.0))), 0.0).sum(axis=2)
        H = -(w[:, None] * v).sum(axis=0)
        sc = H - condA - ce
        if i == 0:
            bald = sc.copy()
        sc = np.where(chosen, -np.inf, sc)
        best = int(np.argmax(sc)) if follow is None else int(follow[i])
        idx.append(best)
        scores.append(sc[best])
        exs.append(exact)
        all_scores.append(sc)
        chosen[best] = True
        condA += ce[best]
        if i + 1 == k:
            break
        if exact and R * C <= n_configs:
            new = (rows[:, None, :] * p[:, best, :].T[None, :, :]).reshape(R * C, M)
            rows, ls = _scaled(new, np.repeat(ls, C))
            w = np.where(np.isfinite(ls), np.exp(ls) / M, 0.0)
            R *= C
            continue
        if exact:                                                   # the switch: replay every pick so far
            exact = False
            R = int(n_configs)
            ms = sample_replicates(M, n_configs, seed, step)
            rows, ls = np.ones((R, M)), np.zeros(R)
            todo = list(enumerate(idx))
        else:
            todo = [(i, best)]
        for j, a in todo:
            rows, ls = _scaled(rows * p[:, a, :].T[draw_labels(p32, ms, a, j, seed, step)], ls)
        rs = rows.sum(axis=1)
        w = np.where(rs > 0, 1.0 / (R * np.where(rs > 0, rs, 1.0)), 0.0)
    return dict(indices=np.array(idx, dtype=np.int64), scores=np.array(scores), exact=np.array(exs), bald=bald,
                all_scores=np.array(all_scores))


def badge_uniform(seed, step, pick):
    w = active_words(seed, step, SITE_BADGE, pick, 0)
    return float((int(w[0] >> 5) << 26 | int(w[1] >> 6)) * 2.0 ** -53)


def badge_embeddings(hidden, logits):
    """g [N, C * (F + 1)] = (p - e_yhat) (x) [h; 1], materialised in float64."""
    h = np.asarray(hidden, dtype=np.float32).astype(np.float64)
    z = np.asarray(logits, dtype=np.float32)
    p, _ = softmax(z)
    a = p.copy()
    a[np.arange(len(z)), z.argmax(axis=1)] -= 1.0
    ht = np.concatenate([h, np.ones((len(h), 1))], axis=1)
    return (a[:, :, None] * ht[:, None, :]).reshape(len(h), -1)


def badge_factorised_d2(hidden, logits, i, c):
    """|g_i - g_c|^2 in the factorised form the kernels use, in float64."""
    h = np.asarray(hidden, dtype=np.float32).astype(np.float64)
    z = np.asarray(logits, dtype=np.float32)
    p, _ = softmax(z)
    a = p.copy()
    a[np.arange(len(z)), z.argmax(axis=1)] -= 1.0
    nh = (h * h).sum(axis=1) + 1.0
    na = (a * a).sum(axis=1)
    return max(0.0, na[i] * nh[i] + na[c] * nh[c] - 2.0 * (a[i] @ a[c]) * (h[i] @ h[c] + 1.0))


def badge(hidden, logits, k, seed=0, step=0):
    """dict(indices, d2, margins): BADGE with the embeddings materialised; margins[i] = the distance of pick i's
    uniform target from the nearest CDF boundary, relative to the total (inf for the first pick)."""
    g = badge_embeddings(hidden, logits)
    N = len(g)
    norms = (g * g).sum(axis=1)
    first = int(np.argmax(norms))
    idx, d2s, margins = [first], [np.inf], [np.inf]
    D2 = np.full(N, np.inf)
    chosen = np.zeros(N, dtype=bool)
    chosen[first] = True
    for i in range(1, k):
        c = idx[-1]
        D2 = np.minimum(D2, ((g - g[c]) ** 2).sum(axis=1))
        D2[chosen] = 0.0
        total = D2.sum()
        if total > 0:
            cum = np.cumsum(D2)
            target = badge_uniform(seed, step, i) * total
            j = int(np.searchsorted(cum, target, side="right"))
            j = min(j, N - 1)
            bounds = cum[D2 > 0]
            margins.append(float(np.min(np.abs(bounds - target)) / total))
        else:
            j = int(np.flatnonzero(~chosen)[0])
            margins.append(np.inf)
        idx.append(j)
        d2s.append(D2[j])
        chosen[j] = True
    return dict(indices=np.array(idx, dtype=np.int64), d2=np.array(d2s), margins=np.array(margins))
