"""TEST INFRASTRUCTURE ONLY -- numpy float64 restatement of raindrop_b200.valuation (rd_knn_shapley), and a brute-force
Shapley value by enumeration of every coalition of the kNN utility it is the exact value of.

Utility of a coalition S for a query with label y_q (Jia et al., VLDB 2019):
    U(S) = (1/K) #{the min(K, |S|) records of S nearest to q that carry label y_q},  U({}) = 0
Nearest: similarity descending, ties to the lower training index (np.lexsort((index, -sim))).
"""
import itertools
import math

import numpy as np


def rank(sim, exclude=None):
    """The candidate indices in ranked order: similarity descending, ties to the lower index; `exclude` left out."""
    sim = np.asarray(sim, dtype=np.float64)
    idx = np.arange(sim.size)
    order = np.lexsort((idx, -sim))
    return order if exclude is None else order[order != exclude]


def recursion(match, K):
    """Shapley values in rank order of a ranked match vector m_1 .. m_N (Theorem 1, base case generalised to K > N):
    s_N = m_N c_N, s_r = s_{r+1} + (m_r - m_{r+1}) c_r, c_r = min(K, r) / (r K)."""
    m = np.asarray(match, dtype=np.float64)
    N = m.size
    s = np.zeros(N)
    c = lambda r: min(K, r) / (r * K)
    s[N - 1] = m[N - 1] * c(N)
    for r in range(N - 1, 0, -1):
        s[r - 1] = s[r] + (m[r - 1] - m[r]) * c(r)
    return s


def suffix_form(match, K):
    """The same values as s_r = m_r c_r - sum_{j = max(r, K) + 1}^{N} m_j / (j (j - 1))."""
    m = np.asarray(match, dtype=np.float64)
    N = m.size
    t = np.array([m[j - 1] / (j * (j - 1)) if j > K else 0.0 for j in range(1, N + 1)])
    tail = np.concatenate([np.cumsum(t[::-1])[::-1][1:], [0.0]])     # sum_{j > r} t_j
    return np.array([m[r - 1] * min(K, r) / (r * K) for r in range(1, N + 1)]) - tail


def utility(match, K):
    """U of the whole ranked set: matches among the min(K, N) nearest, over K."""
    m = np.asarray(match, dtype=np.float64)
    return float(m[:min(K, m.size)].sum() / K)


def brute_force(sim, y_train, y_q, K, exclude=None):
    """Shapley values [n] of every training record by enumeration of all coalitions of the candidates (at most 12);
    an excluded record gets 0."""
    sim = np.asarray(sim, dtype=np.float64)
    n = sim.size
    players = [i for i in range(n) if i != exclude]
    N = len(players)
    assert N <= 12, "enumeration is for N <= 12"
    order = rank(sim)
    pos = np.empty(n, dtype=np.int64)
    pos[order] = np.arange(n)
    match = np.asarray(y_train) == y_q

    def U(S):
        if not S:
            return 0.0
        near = sorted(S, key=lambda i: pos[i])[:K]
        return sum(match[i] for i in near) / K

    phi = np.zeros(n)
    for i in players:
        others = [j for j in players if j != i]
        for size in range(N):
            w = math.factorial(size) * math.factorial(N - size - 1) / math.factorial(N)
            for S in itertools.combinations(others, size):
                phi[i] += w * (U(list(S) + [i]) - U(list(S)))
    return phi


def knn_shapley(sim, y_train, y_query, K, self_offset=None):
    """(per_query [nq, n], values [n] = the means over queries, utility [nq]) from similarities sim [nq, n]: per query
    the ranking above, the recursion, scattered to record order.  self_offset: query q is record self_offset + q,
    excluded from its own ranking (value 0 there)."""
    sim = np.asarray(sim, dtype=np.float64)
    nq, n = sim.shape
    y_train = np.asarray(y_train)
    per = np.zeros((nq, n))
    util = np.zeros(nq)
    for q in range(nq):
        ex = None if self_offset is None else self_offset + q
        order = rank(sim[q], exclude=ex)
        m = y_train[order] == y_query[q]
        per[q, order] = recursion(m, K)
        util[q] = utility(m, K)
    return per, per.mean(axis=0), util


def normalise(f):
    """rd_ood_prepare_bank's rows: the fp64 norm rounded once to fp32, the fp32 division F.normalize does."""
    f = np.asarray(f, dtype=np.float32)
    nrm = np.maximum(np.sqrt((f.astype(np.float64) ** 2).sum(axis=1)).astype(np.float32), np.float32(1e-12))
    return (f / nrm[:, None]).astype(np.float32)


def similarities(q_rows, bank_rows):
    """The fp64 dots of normalised fp32 rows."""
    return np.asarray(q_rows, dtype=np.float64) @ np.asarray(bank_rows, dtype=np.float64).T
