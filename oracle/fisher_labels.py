"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the sampled labels of the true Fisher (rd_fisher_labels, EK-FAC).

U(seed, i) for global sample index i (raindrop_b200/csrc/rd_ekfac.cu, `fisher_uniform`; include/raindrop_b200.h):

  key     = (seed lo, seed hi)
  counter = (i lo, i hi, 97, 0)                       site 97, past the dropout sites 1-96
  U       = ((w0 >> 5) * 2^26 + (w1 >> 6)) / 2^53     53 bits in [0, 1)

label = the first class c with U * sum_c' p_c' < sum_{c'' <= c} p_c'', p_c = exp(logit_c - max logit) in float64, classes
summed in order (the last class if none).
"""
import numpy as np

from .dropout_masks import philox4x32_10

_LO = np.uint64(0xFFFFFFFF)


def fisher_uniforms(n, seed, index0=0):
    """float64 [n]: U(seed, index0 + i) for i < n."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    i = np.arange(int(index0), int(index0) + int(n), dtype=np.uint64)
    ctr = np.empty((len(i), 4), dtype=np.uint64)
    ctr[:, 0], ctr[:, 1], ctr[:, 2], ctr[:, 3] = i & _LO, i >> np.uint64(32), 97, 0
    key = np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint64)
    w = philox4x32_10(ctr, key).astype(np.uint64)                                 # [n, 4]
    return ((w[:, 0] >> np.uint64(5)).astype(np.float64) * 67108864.0 +
            (w[:, 1] >> np.uint64(6)).astype(np.float64)) * (1.0 / 9007199254740992.0)


def fisher_labels(logits, seed, index0=0):
    """int64 [B]: the labels rd_fisher_labels draws from float32 logits [B, n_classes]."""
    lg = np.asarray(logits, dtype=np.float32).astype(np.float64)
    B, ncls = lg.shape
    u = fisher_uniforms(B, seed, index0)
    out = np.empty(B, dtype=np.int64)
    for b in range(B):
        m = lg[b, 0]
        for c in range(1, ncls):
            m = max(m, lg[b, c])
        p = [np.exp(lg[b, c] - m) for c in range(ncls)]
        total = 0.0
        for v in p:
            total += v
        target = u[b] * total
        cum, label = 0.0, ncls - 1
        for c in range(ncls):
            cum += p[c]
            if target < cum:
                label = c
                break
        out[b] = label
    return out
