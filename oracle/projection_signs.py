"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the random projection of rd_grad_projection (TracIn-RP).

Omega(seed, j, m) = +-1 for absolute bucket column j and projection dimension m (raindrop_b200/csrc/rd_projection.cu,
`proj_block` / `proj_sign`; include/raindrop_b200.h):

  key     = (seed lo, seed hi)
  counter = (j >> 7 lo, j >> 7 hi, m, 0)              one Philox block serves 128 consecutive columns of one dimension
  word    = block[(j >> 5) & 3]
  Omega   = -1 if bit (j & 31) of word is set, else +1
"""
import numpy as np

from .dropout_masks import philox4x32_10

_LO = np.uint64(0xFFFFFFFF)


def projection_matrix(n_cols, dim, seed, col0=0):
    """float64 [n_cols, dim]: Omega(seed, col0 + c, m) for c < n_cols, m < dim (the unscaled +-1 signs)."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    j = np.arange(int(col0), int(col0) + int(n_cols), dtype=np.uint64)
    m = np.arange(int(dim), dtype=np.uint64)
    jb = (j >> np.uint64(7))[:, None]
    ctr = np.empty((len(j), len(m), 4), dtype=np.uint64)
    ctr[..., 0], ctr[..., 1] = jb & _LO, jb >> np.uint64(32)
    ctr[..., 2], ctr[..., 3] = m[None, :], 0
    key = np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint64)
    words = philox4x32_10(ctr, key)                                               # [n_cols, dim, 4] uint32
    q = ((j >> np.uint64(5)) & np.uint64(3)).astype(np.int64)
    w = np.take_along_axis(words, np.broadcast_to(q[:, None, None], (len(j), len(m), 1)), -1)[..., 0]
    bit = (w >> (j & np.uint64(31)).astype(np.uint32)[:, None]) & np.uint32(1)
    return np.where(bit == 1, -1.0, 1.0)


def project_rows(G, dim, seed, seg_off=None, seg_len=None):
    """float64 [rows, dim]: (G restricted to the segments' columns) Omega / sqrt(dim), the restatement of
    rd_grad_projection; no segments: every column of G."""
    G = np.asarray(G, dtype=np.float64)
    if seg_off is None:
        seg_off, seg_len = [0], [G.shape[1]]
    out = np.zeros((G.shape[0], int(dim)))
    for o, n in zip(seg_off, seg_len):
        out += G[:, int(o):int(o) + int(n)] @ projection_matrix(int(n), dim, seed, col0=int(o))
    return out / np.sqrt(int(dim))
