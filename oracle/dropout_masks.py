"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the CUDA path's dropout stream.

The kernels draw every dropout decision from Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as
1, 2, 3", SC'11), counter based, so the masks of any forward can be rebuilt from its captured (seed, step) without
touching the device (raindrop_b200/csrc/rd_common.cuh, `dropout_block` / `keep_scale`):

  key     = (seed lo, seed hi ^ step hi)
  counter = (idx >> 2 lo, idx >> 2 hi, site, step lo)     one block serves four consecutive element indices
  word    = block[idx & 3]
  keep    = (word >> 8) / 2^24 >= p,  scale = 1/(1-p) in fp32, else 0

Sites and their element index spaces (rd_common.cuh `DropSite`):
  lift      1         [T, B, N*d_ob]   relu(src * R_u) before the observation propagation
  attention 16 + l    [B, H, T, T]     attention probabilities, row = query, column = key
  dropout1  32 + l    [T*B, D]         out_proj output
  FFN       48 + l    [T*B, nhid]      relu(linear1)
  dropout2  64 + l    [T*B, D]         linear2 output
"""
import numpy as np

SITE_LIFT, SITE_ATTN, SITE_RESID1, SITE_FFN, SITE_RESID2 = 1, 16, 32, 48, 64

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)


def philox4x32_10(ctr, key):
    """Philox4x32 with 10 rounds.  ctr [..., 4] and key [..., 2] (broadcast against each other), any integer
    type holding uint32 values; returns uint32 [..., 4]."""
    ctr = np.asarray(ctr, dtype=np.uint64)
    key = np.asarray(key, dtype=np.uint64)
    c0, c1, c2, c3 = (ctr[..., i] for i in range(4))
    k0, k1 = key[..., 0], key[..., 1]
    for _ in range(10):
        p0, p1 = _M0 * c0, _M1 * c2                  # 32 x 32 -> 64 bit, exact in uint64
        c0, c1, c2, c3 = (p1 >> _S32) ^ c1 ^ k0, p1 & _LO, (p0 >> _S32) ^ c3 ^ k1, p0 & _LO
        k0, k1 = (k0 + _W0) & _LO, (k1 + _W1) & _LO
    return np.stack([c0, c1, c2, c3], -1).astype(np.uint32)


def dropout_words(seed, step, site, n):
    """The 32-bit Philox word of element indices 0 .. n-1 of `site` under (seed, step)."""
    seed, step = int(seed) & 0xFFFFFFFFFFFFFFFF, int(step) & 0xFFFFFFFFFFFFFFFF
    blk = np.arange((int(n) + 3) // 4, dtype=np.uint64)
    ctr = np.empty(blk.shape + (4,), dtype=np.uint64)
    ctr[:, 0], ctr[:, 1] = blk & _LO, blk >> _S32
    ctr[:, 2], ctr[:, 3] = site, step & 0xFFFFFFFF
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) ^ (step >> 32)], dtype=np.uint64)
    return philox4x32_10(ctr, key).reshape(-1)[: int(n)]


def dropout_words_at(seed, step, site, idx):
    """The 32-bit Philox word of the given element indices (any integer array) of `site` under (seed, step): the same
    values as dropout_words(...)[idx], without generating the indices below them."""
    seed, step = int(seed) & 0xFFFFFFFFFFFFFFFF, int(step) & 0xFFFFFFFFFFFFFFFF
    idx = np.asarray(idx, dtype=np.uint64)
    blk = idx >> np.uint64(2)
    ctr = np.empty(idx.shape + (4,), dtype=np.uint64)
    ctr[..., 0], ctr[..., 1] = blk & _LO, blk >> _S32
    ctr[..., 2], ctr[..., 3] = site, step & 0xFFFFFFFF
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) ^ (step >> 32)], dtype=np.uint64)
    words = philox4x32_10(ctr, key)
    return np.take_along_axis(words, (idx & np.uint64(3)).astype(np.int64)[..., None], -1)[..., 0]


def _keep_scale(words, p):
    p32 = np.float32(p)
    inv_keep = np.float32(1.0) / (np.float32(1.0) - p32)
    u = (words >> np.uint32(8)).astype(np.float64) * 2.0 ** -24   # exact
    return np.where(u >= np.float64(p32), inv_keep, np.float32(0.0)).astype(np.float32)


def dropout_mask(seed, step, site, n, p):
    """float32 [n]: 1/(1-p) where element idx is kept, 0 where it is dropped (bitwise what the kernels multiply by)."""
    return _keep_scale(dropout_words(seed, step, site, n), p)


def dropout_mask_at(seed, step, site, idx, p):
    """dropout_mask(seed, step, site, max(idx) + 1, p)[idx], evaluated at the given element indices only."""
    return _keep_scale(dropout_words_at(seed, step, site, idx), p)


def lift_mask(rng, p, T, B, width):
    """[T, B, N*d_ob], the layout of the lifted input `h` of RaindropV2Oracle._lift."""
    return dropout_mask(rng[0], rng[1], SITE_LIFT, T * B * width, p).reshape(T, B, width)


def attention_mask(rng, p, layer, B, H, T):
    """[B, H, T, T]: [b, h, query, key]."""
    return dropout_mask(rng[0], rng[1], SITE_ATTN + layer, B * H * T * T, p).reshape(B, H, T, T)


def resid1_mask(rng, p, layer, rows, D):
    """[T*B, D], token-major rows t*B + b."""
    return dropout_mask(rng[0], rng[1], SITE_RESID1 + layer, rows * D, p).reshape(rows, D)


def ffn_mask(rng, p, layer, rows, nhid):
    return dropout_mask(rng[0], rng[1], SITE_FFN + layer, rows * nhid, p).reshape(rows, nhid)


def resid2_mask(rng, p, layer, rows, D):
    return dropout_mask(rng[0], rng[1], SITE_RESID2 + layer, rows * D, p).reshape(rows, D)


def model_masks(rng, p, cfg, B):
    """Every mask one Raindrop_v2 training forward draws, keyed as RaindropV2Oracle.forward_dense(masks=...) takes them:
    {"lift": [T, B, N*d_ob], "layers": [{"attn", "resid1", "ffn", "resid2"}] * nlayers}, numpy float32."""
    T, N, d_ob = cfg["max_len"], cfg["d_inp"], cfg["d_ob"]
    D = N * d_ob + 16
    H, nhid, rows = cfg["nhead"], cfg["nhid"], T * B
    layers = [dict(attn=attention_mask(rng, p, l, B, H, T), resid1=resid1_mask(rng, p, l, rows, D),
                   ffn=ffn_mask(rng, p, l, rows, nhid), resid2=resid2_mask(rng, p, l, rows, D))
              for l in range(cfg["nlayers"])]
    return dict(lift=lift_mask(rng, p, T, B, N * d_ob), layers=layers)


def slice_masks(masks, sl, T, B):
    """The masks of samples `sl` (a slice) of a batch of B, in the model_masks layout; numpy arrays or tensors.  A mask
    that is None or absent stays so (no dropout there)."""
    def cut(key, m):
        if key == "attn":                # [B, H, T, T]
            return m[sl]
        return m.reshape(T, B, -1)[:, sl].reshape(-1, m.shape[-1])     # token-major [T*B, width] -> [T*Bc, width]
    lift = masks.get("lift")
    return dict(lift=None if lift is None else lift[:, sl],
                layers=[{k: cut(k, m) for k, m in l.items() if m is not None} for l in masks["layers"]])


def ones_masks(cfg, B):
    """The all-keep masks (p = 0) in the layout of model_masks."""
    return model_masks((0, 0), 0.0, cfg, B)
