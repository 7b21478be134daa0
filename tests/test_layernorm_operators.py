"""The encoder's LayerNorm kernels on their own, element by element against float64.

Every encoder layer runs two LayerNorms forward and backward, and DP-SGD, TracIn, TracIn-RP, EK-FAC and the Laplace
approximation read their per-sample gradients.  The kernels (rd_kernels.cu, rd_dp.cu):
  * forward: layernorm_fwd_vec_kernel<1 | 2 | 5> (the row in registers, ITERS float4 per lane: D % 4 == 0, D <= 128
    ITERS, x, y, gamma, beta 16-byte aligned), else the generic layernorm_fwd_kernel (lane-strided);
  * backward: layernorm_bwd_fused_kernel<1, 1, 8>, <2, 1, 8>, <5, 1, 32> (one pass: dx, dx_drop and per-CTA partial
    rows of the dgamma / dbeta column sums; D % 4 == 0, D <= 640, x, dy, gamma, dx, dx_drop aligned), else the split
    pair layernorm_bwd_dx_kernel (a 128-bit path when D % 4 == 0 and the pointers it reads and writes are aligned, else
    scalar) + layernorm_bwd_param_kernel (256 rows per chunk);
  * the partial rows [chunks][2][D] are summed by two column-sum items of one tc_wgrad_group launch;
  * per sample: dp_ln_sqnorm_kernel (squared norms) and psg_ln_kernel (gradient rows, times scale).
They run here through rd_debug_layernorm (one layernorm_fwd and / or one layernorm_bwd call and the grouped column
sums, exactly as the training step and its gradient consumer issue them; the classes, chunks and keep-mask source
written back) and rd_debug_per_sample_layernorm.

Bounds, u = 2^-24, gamma_k = k u / (1 - k u).  Build: IEEE sqrtf and division, no fast-math, FMA contraction on, so
every operation rounds at most once (an fmaf rounds once for two).  A sum whose every term passes through at most k
roundings on its way (its own product roundings included) errs by at most gamma_k sum |terms|.  "fp64 terms" (k 2^-53
times the matching magnitudes) cover the float64 reference's own rounding.  Per row, with the exact mean mu, Q =
sum (x - mu)^2, W = Q / D + eps (eps as fp32), r = W^-1/2:
Forward.  The sum of x: generic, each lane adds columns lane, lane + 32, ... (ceil(D/32) terms), then the 5-level
  butterfly warp_sum: kS = ceil(D/32) + 5; vector, each lane adds (x0 + x1) + (x2 + x3) per float4 (2 roundings + 1
  into the lane sum per iteration): kS = ceil(D/128) + 7.  The mean m^ = s^ / D:
      |m^ - mu| <= e_m = gamma_kS sum|x| / D (1 + u) + u |mu|.
  The squares of d^ = fl(x - m^) (one rounding) add the same ways (kQ = kS + 1, the product), and sum (x - m^)^2 = Q +
  D (mu - m^)^2, so q^ lies in [Q (1-u)^2 (1 - gamma_kQ), (Q + D e_m^2)(1+u)^2 (1 + gamma_kQ)]; v = q^ / D, v + eps,
  sqrtf and 1 / . round once each, so rstd^ lies in [(1 - 2u) W_hi^-1/2, (1 + 2u) W_lo^-1/2] with W_hi / lo = (q_hi / lo
  / D (1 +- u) + eps)(1 +- u): |rstd^ - r| <= e_r, the larger distance.  This is no linearisation: on a near-constant
  row (Q / D <= eps) r approaches eps^-1/2 and the mean's rounding, times rstd, dominates everything.
  y = fma(fl(fl(x - m^) rstd^), gamma, beta): with e_t1 = e_m + u (|x - mu| + e_m) and e_t2 = e_t1 r_hi + |x - mu| e_r
  + u (|x - mu| + e_t1) r_hi,
      |y^ - y| <= |gamma| e_t2 (1 + u) + u |gamma| (|x - mu| r + e_t2)(1 + u) + u |y|.
Backward, on the stats {m, r} it is given (the forward's, or the exact ones rounded to fp32; the reference uses the
  same fp32 values): x^ = (x - m) r, the kernel's x^ errs by gamma_2 |x^|.  s1 = mean(dy gamma), s2 = mean(dy gamma x^):
  fused, per float4 a chain of 4 products into one value, then into the lane sum (5 roundings; 1 more per later
  iteration), then warp_sum: k1 = ceil(D/128) + 9; split 128-bit, 4 sequential adds per float4: k1 = 4 ceil(D/128) + 6;
  split scalar, lane-strided: k1 = ceil(D/32) + 6.  s2 has 2 more (x^) and 1 more (dy gamma rounded first): k2 = k1 +
  3.  Each mean: e_s = gamma_(k+1) sum |terms| / D (the division).  dx = rstd (dy gamma - s1 - x^ s2) takes at most 4
  roundings in the bracket and 1 for the product:
      |dx^ - dx| <= r E_B (1 + u) + u |dx|,  E_B = e_s1 + |x^| e_s2 + e_h (|s2| + e_s2)
                                                 + gamma_4 (|dy gamma| + |s1| + e_s1 + (|x^| + e_h)(|s2| + e_s2)).
  dx_drop = fl(dx^ m), m in {0, 1/(1-p)}: |dx_drop^ - dx m| <= m |dx^ - dx| + u m |dx^|, exactly 0 where dropped.
Column sums dgamma = sum_rows dy x^, dbeta = sum_rows dy.  Fused: each warp chains its rows of the CTA (ROWS / 8 = 1
  or 4) per column, then the CTA adds the 8 warps' rows in order through shared memory (7 roundings): kP = ROWS/8 + 9
  (x^: 2).  Split: 32-row chains per row group, 8 groups added in order: kP = 32 + 10.  The chunk sum in the grouped
  launch (test_wgrad_operators.py): (ceil(chunks/32) + 5) u sum |partial|, so
      |dgamma^ - dgamma| <= gamma_kP S + (ceil(chunks/32) + 5) u S (1 + gamma_kP),  S = sum_rows |dy x^| (dbeta: |dy|).
Per sample (rows t*B + b): each term fl(dy fl(fl(x - m) r)) (3 roundings) summed in fp64: delta = gamma_3 sum_t
  |dy x^| + fp64 terms (beta: fp64 terms only).  Squared norms: sum_d (2 |g| delta + delta^2) + fp64 terms; rows:
  |G - scale g| <= |scale| delta + u |scale| (|g| + delta).

CPU: float32 numpy emulations of every kernel's order (lanes, float4 pairs, butterflies, the 8-warp CTA sum, the
chunk sum) stay inside these bounds on six operand families, and each mutation breaks them on at least one case:
vec<2> at D = 260 (a lost column tail), the keep bit read one position off, the Philox index with a padded D, mean
and rstd swapped in stats, one warp's partial row left out of the CTA sum, s2 from dy gamma instead of dy gamma x^,
the last chunk left out of the column sum, and psg_ln without scale.  A restatement of the dispatch (the forward's
predicate over {x, y, gamma, beta}, the backward's over {x, dy, gamma, dx, dx_drop}) reproduces the plan table, and
the entries' refusals are checked.
GPU: every class and tail (17 widths x 11 row counts), each class confirmed from the written-back plan; one pointer
misaligned at a time (beta, dx_drop, gamma); the keep masks against rd_debug_dropout_mask at sites 32 + l and 64 + l
(Philox, stored bits equal to it, arbitrary bits, bits the split path ignores); seven operand families at three eps;
the P19, P12, PAM and LARGE shapes; NaN rows past `rows`, NaN-filled outputs and scratch, NaN-payload guards around
every output; the per-sample kernels at T in {1, 60, 215, 600} x B in {1, 3, 33, 128} with two cross-checks; and the
same bits across runs.  The worst err / bound of each (quantity, path, family) is printed.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from raindrop_b200 import lib as L
from test_gemm_operators import FAKE, U, refused
from test_wgrad_operators import colsum_coef

GEN, V1, V2, V5, SVEC, SSCAL = L.RD_LN_GENERIC, L.RD_LN_VEC1, L.RD_LN_VEC2, L.RD_LN_VEC5, L.RD_LN_SPLIT_VEC, \
    L.RD_LN_SPLIT_SCALAR
FUSED = (V1, V2, V5)
CLASS_NAME = {GEN: "generic", V1: "vec1", V2: "vec2", V5: "vec5", SVEC: "split-vec", SSCAL: "split-scalar"}
FAMILIES = ["normal", "offset", "flat", "outliers", "pow2", "gamma0", "zero-dy"]
WORST = {}


def lib():
    return L.load()


def gam(k):
    return k * U / (1 - k * U)


def f64(k):
    return k * 2.0 ** -53 * 1.01


def cdiv(a, b):
    return -(-a // b)


# ---- the dispatch, restated ------------------------------------------------------------------------------------------
def fwd_class(D, aligned=True):
    """layernorm_fwd: aligned = x, y, gamma and beta all 16-byte aligned"""
    if D % 4 or D > 640 or not aligned:
        return GEN
    return V1 if D <= 128 else V2 if D <= 256 else V5


def bwd_class(D, fused_aligned=True, split_aligned=True):
    """layernorm_bwd: fused_aligned = x, dy, gamma, dx, dx_drop aligned; split_aligned = the same with dx_drop only
    when the split kernel writes it (drop_p > 0)"""
    if D % 4 == 0 and D <= 640 and fused_aligned:
        return V1 if D <= 128 else V2 if D <= 256 else V5
    return SVEC if D % 4 == 0 and split_aligned else SSCAL


def bwd_rows_per_cta(D, cls):
    return 256 if cls in (SVEC, SSCAL) else (8 if D <= 256 else 32)


def scratch_floats(rows, D):
    return max(cdiv(rows, 256), cdiv(rows, 8 if D <= 256 else 32)) * 2 * D


def production_widths():
    from raindrop_b200.synth import model_config
    out = {}
    for name in ("P19", "P12", "PAM", "LARGE"):
        c = model_config(name)
        out[name] = (c["d_model"] + 16, c["max_len"] * c["batch"])
    return out


# (width, rows, misaligned pointer, drop) -> (forward class, backward class)
PLAN_TABLE = {
    ("P19", None): (V2, V2), ("P12", None): (V2, V2), ("PAM", None): (V1, V1), ("LARGE", None): (V5, V5),
    ("P19", "beta"): (GEN, V2), ("PAM", "dx_drop"): (V1, SSCAL), ("LARGE", "gamma"): (GEN, SSCAL),
    ("LARGE", "dx_drop_p0"): (V5, SVEC), (644, None): (GEN, SVEC), (1024, "y"): (GEN, SVEC), (130, None): (GEN, SSCAL),
    (641, None): (GEN, SSCAL), (640, "dx"): (V5, SSCAL), (4, None): (V1, V1),
}


def plan_of(key):
    width, mis = key
    D = production_widths()[width][0] if isinstance(width, str) else width
    fa = mis not in ("x", "y", "gamma", "beta")
    fused_ok = mis not in ("x", "dy", "gamma", "dx", "dx_drop", "dx_drop_p0")
    split_ok = mis not in ("x", "dy", "gamma", "dx", "dx_drop")          # dx_drop_p0: drop_p = 0, not written
    return fwd_class(D, fa), bwd_class(D, fused_ok, split_ok)


def test_production_widths():
    assert production_widths() == {"P19": (152, 7680), "P12": (160, 6880), "PAM": (84, 153600), "LARGE": (528, 131072)}


@pytest.mark.parametrize("key", sorted(PLAN_TABLE, key=str))
def test_dispatch_matches_plan_table(key):
    assert plan_of(key) == PLAN_TABLE[key]


def test_scratch_query_is_the_restated_size():
    for rows in (1, 7, 8, 9, 255, 256, 257, 4097, 153600):
        for D in (1, 84, 152, 256, 257, 528, 1024):
            assert lib().rd_debug_layernorm_scratch_floats(rows, D) == scratch_floats(rows, D), (rows, D)


# ---- float64 references and bounds (torch, any device) --------------------------------------------------------------
def fwd_depths(D, cls):
    if cls == GEN:
        return cdiv(D, 32) + 5, cdiv(D, 32) + 6
    return cdiv(D, 128) + 7, cdiv(D, 128) + 8


def bwd_depth(D, cls):
    if cls in FUSED:
        return cdiv(D, 128) + 9
    if cls == SVEC:
        return 4 * cdiv(D, 128) + 6
    return cdiv(D, 32) + 6


def part_depth(D, cls):
    return 42 if cls in (SVEC, SSCAL) else bwd_rows_per_cta(D, cls) // 8 + 9


def ref_forward(x, g, b, eps, cls):
    """x [rows, D], g, b [D] float64 (the fp32 operands); eps the fp32 value.  Returns y, mean, rstd, their bounds."""
    D = x.shape[1]
    kS, kQ = fwd_depths(D, cls)
    mu = x.mean(1, keepdim=True)
    xc = x - mu
    Q = (xc * xc).sum(1, keepdim=True)
    r = 1.0 / torch.sqrt(Q / D + eps)
    Sx = x.abs().sum(1, keepdim=True) / D
    e_m = gam(kS) * Sx * (1 + U) + U * mu.abs() + f64(D + 8) * Sx
    q_hi = (Q + D * e_m * e_m) * (1 + U) ** 2 * (1 + gam(kQ)) * (1 + f64(D + 8))
    q_lo = (Q * (1 - U) ** 2 * (1 - gam(kQ)) * (1 - f64(D + 8))).clamp_min(0.0)
    w_hi = (q_hi / D * (1 + U) + eps) * (1 + U)
    w_lo = (q_lo / D * (1 - U) + eps) * (1 - U)
    r_hi, r_lo = (1 + 2.01 * U) / torch.sqrt(w_lo), (1 - 2.01 * U) / torch.sqrt(w_hi)
    e_r = torch.maximum(r_hi - r, r - r_lo) + f64(8) * r
    axc = xc.abs()
    e_t1 = e_m + U * (axc + e_m)
    e_t2 = e_t1 * r_hi + axc * e_r + U * (axc + e_t1) * r_hi
    y = xc * r * g + b
    ag = g.abs()
    e_y = ag * e_t2 * (1 + U) + U * ag * (axc * r + e_t2) * (1 + U) + U * y.abs() + f64(16) * (ag * axc * r + b.abs())
    return dict(y=y, e_y=e_y, mean=mu[:, 0], e_mean=e_m[:, 0], rstd=r[:, 0], e_rstd=e_r[:, 0])


def ref_backward(x, stats, g, dy, cls, chunks, mask=None):
    """on the given stats [rows, 2] (fp32 values, float64 here): dx, dx_drop (mask [rows, D] of 0 / 1/(1-p)), dgamma,
    dbeta and their bounds"""
    D = x.shape[1]
    m, r = stats[:, :1], stats[:, 1:]
    xh = (x - m) * r
    gd = dy * g
    k1 = bwd_depth(D, cls)
    k2 = k1 + 3
    s1, s2 = gd.mean(1, keepdim=True), (gd * xh).mean(1, keepdim=True)
    e_s1 = gam(k1 + 1) * gd.abs().mean(1, keepdim=True) + f64(D + 8) * gd.abs().mean(1, keepdim=True)
    e_s2 = gam(k2 + 1) * (gd * xh).abs().mean(1, keepdim=True) + f64(D + 8) * (gd * xh).abs().mean(1, keepdim=True)
    e_h = gam(2) * xh.abs()
    dx = r * (gd - s1 - xh * s2)
    E_B = (e_s1 + xh.abs() * e_s2 + e_h * (s2.abs() + e_s2) +
           gam(4) * (gd.abs() + s1.abs() + e_s1 + (xh.abs() + e_h) * (s2.abs() + e_s2)))
    e_dx = r * E_B * (1 + U) + U * dx.abs() + f64(8) * r * (gd.abs() + s1.abs() + xh.abs() * s2.abs())
    out = dict(dx=dx, e_dx=e_dx)
    if mask is not None:
        out["dx_drop"] = dx * mask
        out["e_dx_drop"] = mask * e_dx + U * mask * (dx.abs() + e_dx)
    kP = part_depth(D, cls)
    cc = colsum_coef(chunks)
    for name, t in (("dgamma", dy * xh), ("dbeta", dy)):
        S = t.abs().sum(0)
        out[name] = t.sum(0)
        out["e_" + name] = gam(kP) * S + cc * U * S * (1 + gam(kP)) + f64(x.shape[0] + 8) * S
    return out


def exact_stats(x, eps):
    """{mean, rstd} of the fp32 rows in float64, rounded to fp32 once"""
    mu = x.mean(1)
    r = 1.0 / torch.sqrt(((x - mu[:, None]) ** 2).mean(1) + eps)
    return torch.stack([mu, r], 1).float()


def ref_per_sample(x, stats, dy, T, B, scale=1.0):
    """the per-sample gamma / beta gradients [B, D], their bounds, the squared norms [B] and theirs, the rows' bounds"""
    D = x.shape[1]
    xh = (x - stats[:, :1]) * stats[:, 1:]
    tw, tb = (dy * xh).view(T, B, D), dy.view(T, B, D)
    gw, gb = tw.sum(0), tb.sum(0)
    dw = gam(3) * tw.abs().sum(0) + f64(T + 8) * tw.abs().sum(0)
    db = f64(T + 8) * tb.abs().sum(0)
    out = dict(gw=gw, gb=gb, dw=dw, db=db)
    for k, g, d in (("w", gw, dw), ("b", gb, db)):
        out["sq" + k] = (g * g).sum(1)
        out["e_sq" + k] = (2 * g.abs() * d + d * d).sum(1) + f64(D + 16) * ((g.abs() + d) ** 2).sum(1)
        out["e_row" + k] = abs(scale) * d + U * abs(scale) * (g.abs() + d) + f64(4) * abs(scale) * g.abs()
    return out


def ratio_of(err, bound):
    live = bound > 0
    return float((err[live] / bound[live]).max()) if bool(live.any()) else 0.0


def violations(out, ref, bound):
    err = (out - ref).abs()
    bad = ~(err <= bound)
    ok = ~torch.isnan(err)
    return bad, ratio_of(err[ok], bound[ok])


def check(key, out, ref, bound, tag=""):
    bad, ratio = violations(out, ref, bound)
    WORST[key] = max(WORST.get(key, 0.0), ratio)
    assert not bool(bad.any()), (key, tag, ratio, int(bad.sum()))


def print_worst():
    for k in sorted(WORST):
        print("WORST %-10s %-13s %-9s %.4g" % (k[0], k[1], k[2], WORST[k]))


# ---- operands ----------------------------------------------------------------------------------------------------
def operands(rows, D, family, seed, device):
    """x, dy [rows, D], gamma, beta [D] float32"""
    g = torch.Generator(device=device).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device=device, dtype=torch.float64)
    x, dy, gamma, beta = rn(rows, D), rn(rows, D), rn(D), rn(D)
    gamma[torch.rand(D, generator=g, device=device) < 0.1] = 0.0           # zeros and negatives in every family
    if family == "offset":             # rows offset by +-100 standard deviations: the mean cancels
        x = x + 100.0 * torch.where(torch.rand(rows, 1, generator=g, device=device) < 0.5, -1.0, 1.0)
    elif family == "flat":             # variance at or below eps, every third row exactly constant
        c = rn(rows, 1) * 3.0
        x = c + 1e-4 * x
        x[::3] = c[::3]
    elif family == "outliers":         # 0.2 % of the entries at +-1e3
        hit = torch.rand(rows, D, generator=g, device=device) < 0.002
        x = torch.where(hit, 1e3 * torch.sign(x), x)
    elif family == "pow2":             # rows of x and dy scaled by 2^-20 .. 2^20
        e = lambda: torch.exp2(torch.randint(-20, 21, (rows, 1), generator=g, device=device).double())
        x, dy = x * e(), dy * e()
    elif family == "gamma0":           # half the gamma entries 0, the rest of both signs
        gamma[torch.rand(D, generator=g, device=device) < 0.5] = 0.0
    elif family == "zero-dy":          # padded time steps: dy zero on whole rows
        dy[torch.rand(rows, generator=g, device=device) < 0.3] = 0.0
    return x.float(), dy.float(), gamma.float(), beta.float()


# ---- CPU: the kernels' arithmetic in numpy float32, and mutations of it --------------------------------------------
f32 = np.float32


def fma(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(f32)


def butterfly(v):
    """warp_sum over the last axis (32 lanes); every lane ends with the same value"""
    for o in (16, 8, 4, 2, 1):
        v = (v + v[..., np.arange(32) ^ o]).astype(f32)
    return v[..., 0]


def lane_strided(t, D):
    """[rows, 32]: lane l's sequential sum of columns l, l + 32, ..."""
    acc = np.zeros(t.shape[:-1] + (32,), f32)
    for k in range(cdiv(D, 32)):
        n = min(32, D - 32 * k)
        acc[..., :n] = (acc[..., :n] + t[..., 32 * k:32 * k + n]).astype(f32)
    return acc


def lanes4(a, D, iters):
    """[rows, iters, 32, 4] float4 groups j = 4 lane + 128 it (zero past D or the kernel's reach), valid [iters, 32]"""
    rows = a.shape[0]
    w = 128 * iters
    p = np.zeros((rows, max(w, D)), f32)
    p[:, :D] = a
    valid = (4 * np.arange(32)[None, :] + 128 * np.arange(iters)[:, None]) < D
    return p[:, :w].reshape(rows, iters, 32, 4), valid


def emu_forward(x, g, b, eps, cls, iters=None):
    """y, stats as the class's kernel computes them (iters overrides the vector kernel's ITERS: mutation)"""
    rows, D = x.shape
    eps = f32(eps)
    if cls == GEN:
        s = butterfly(lane_strided(x, D))
        mean = (s / f32(D)).astype(f32)
        d = (x - mean[:, None]).astype(f32)
        q = np.zeros((rows, 32), f32)
        for k in range(cdiv(D, 32)):
            n = min(32, D - 32 * k)
            q[:, :n] = fma(d[:, 32 * k:32 * k + n], d[:, 32 * k:32 * k + n], q[:, :n])
        q = butterfly(q)
        rstd = (f32(1) / np.sqrt((q / f32(D)).astype(f32) + eps).astype(f32)).astype(f32)
        y = fma((d * rstd[:, None]).astype(f32), g[None, :], b[None, :])
        return y, np.stack([mean, rstd], 1)
    it = iters or cls
    v, valid = lanes4(x, D, it)
    s = np.zeros((rows, 32), f32)
    for k in range(it):
        pair = ((v[:, k, :, 0] + v[:, k, :, 1]).astype(f32) + (v[:, k, :, 2] + v[:, k, :, 3]).astype(f32)).astype(f32)
        s = (s + pair).astype(f32)
    mean = (butterfly(s) / f32(D)).astype(f32)
    d = (v - mean[:, None, None, None]).astype(f32)
    q = np.zeros((rows, 32), f32)
    for k in range(it):
        dk = d[:, k]
        pair = (fma(dk[..., 1], dk[..., 1], (dk[..., 0] * dk[..., 0]).astype(f32)) +
                fma(dk[..., 3], dk[..., 3], (dk[..., 2] * dk[..., 2]).astype(f32))).astype(f32)
        q = np.where(valid[k][None, :], (q + pair).astype(f32), q)
    rstd = (f32(1) / np.sqrt((butterfly(q) / f32(D)).astype(f32) + eps).astype(f32)).astype(f32)
    y = np.full((rows, max(D, 128 * it)), np.nan, f32)
    gg, _ = lanes4(g[None, :], D, it)
    bb, _ = lanes4(b[None, :], D, it)
    yv = fma((d * rstd[:, None, None, None]).astype(f32), gg, bb)
    for k in range(it):
        for lane in np.nonzero(valid[k])[0]:
            j = 4 * lane + 128 * k
            y[:, j:j + 4] = yv[:, k, lane]
    return y[:, :D], np.stack([mean, rstd], 1)


def colsum_emu(P, drop_last=False):
    """the grouped launch's column sum of partial rows P [chunks, D]: lane l adds rows l, l + 32, ..., then warp_sum"""
    if drop_last:
        P = P[:-1]
    acc = np.zeros((32, P.shape[1]), f32)
    for k in range(cdiv(P.shape[0], 32)):
        n = min(32, P.shape[0] - 32 * k)
        acc[:n] = (acc[:n] + P[32 * k:32 * k + n]).astype(f32)
    return butterfly(acc.T)


def emu_backward(x, stats, g, dy, cls, mask, mutation=None):
    """dx, dx_drop, dgamma, dbeta of the class's kernels.  mask [rows, D]: the multiplier dx_drop takes (None: none)"""
    rows, D = x.shape
    st = stats[:, ::-1] if mutation == "swap-stats" else stats
    m, r = st[:, 0:1].astype(f32), st[:, 1:2].astype(f32)
    xh = ((x - m).astype(f32) * r).astype(f32)
    gd = (dy * g[None, :]).astype(f32)
    hs = np.ones_like(xh) if mutation == "s2-from-g" else xh        # the factor s2 takes besides dy gamma
    if cls in FUSED:
        dv, valid = lanes4(dy, D, cls)
        gv, _ = lanes4(g[None, :], D, cls)
        hv, _ = lanes4(hs, D, cls)
        s1 = np.zeros((rows, 32), f32)
        s2 = np.zeros((rows, 32), f32)
        for k in range(cls):
            d, gg, h = dv[:, k], gv[:, k], hv[:, k]
            t = (d[..., 0] * gg[..., 0]).astype(f32)
            for e in (1, 2, 3):
                t = fma(d[..., e], gg[..., e], t)
            s1 = (s1 + t).astype(f32)
            dg = (d * gg).astype(f32)
            t = (dg[..., 0] * h[..., 0]).astype(f32)
            for e in (1, 2, 3):
                t = fma(dg[..., e], h[..., e], t)
            s2 = (s2 + t).astype(f32)
    elif cls == SVEC:
        gv, valid = lanes4(gd, D, cdiv(D, 128))
        hv, _ = lanes4(hs, D, cdiv(D, 128))
        s1 = np.zeros((rows, 32), f32)
        s2 = np.zeros((rows, 32), f32)
        for k in range(gv.shape[1]):
            for e in range(4):
                s1 = np.where(valid[k][None, :], (s1 + gv[:, k, :, e]).astype(f32), s1)
                s2 = np.where(valid[k][None, :], fma(gv[:, k, :, e], hv[:, k, :, e], s2), s2)
    else:
        s1 = lane_strided(gd, D)
        s2 = np.zeros((rows, 32), f32)
        for k in range(cdiv(D, 32)):
            n = min(32, D - 32 * k)
            s2[:, :n] = fma(gd[:, 32 * k:32 * k + n], hs[:, 32 * k:32 * k + n], s2[:, :n])
    s1 = (butterfly(s1) / f32(D)).astype(f32)[:, None]
    s2 = (butterfly(s2) / f32(D)).astype(f32)[:, None]
    dx = (r * fma(-xh, s2, fma(dy, g[None, :], -s1))).astype(f32)
    dxd = None if mask is None else (dx * mask).astype(f32)
    # the column sums' partial rows
    if cls in FUSED:
        R = bwd_rows_per_cta(D, cls)
        chunks = cdiv(rows, R)
        P = np.zeros((chunks, 2, D), f32)
        for c in range(chunks):
            warp_rows = [np.zeros((2, D), f32) for _ in range(8)]
            for rr in range(R):
                row = c * R + rr
                if row >= rows:
                    continue
                w = warp_rows[rr % 8]
                w[0] = fma(dy[row], xh[row], w[0])
                w[1] = (w[1] + dy[row]).astype(f32)
            acc = np.zeros((2, D), f32)
            for w in range(8):
                if mutation == "lost-warp" and w == 1:
                    continue
                acc = (acc + warp_rows[w]).astype(f32)
            P[c] = acc
    else:
        chunks = cdiv(rows, 256)
        P = np.zeros((chunks, 2, D), f32)
        for c in range(chunks):
            groups = []
            for y in range(8):
                acc = np.zeros((2, D), f32)
                for row in range(c * 256 + 32 * y, min(rows, c * 256 + 32 * y + 32)):
                    acc[0] = fma(dy[row], xh[row], acc[0])
                    acc[1] = (acc[1] + dy[row]).astype(f32)
                groups.append(acc)
            acc = groups[0]
            for y in range(1, 8):
                acc = (acc + groups[y]).astype(f32)
            P[c] = acc
    drop = mutation == "lost-chunk"
    return dict(dx=dx, dx_drop=dxd, dgamma=colsum_emu(P[:, 0], drop), dbeta=colsum_emu(P[:, 1], drop), chunks=chunks)


def emu_per_sample(x, stats, dy, T, B, scale, mutation=None):
    D = x.shape[1]
    xh = ((x - stats[:, :1]).astype(f32) * stats[:, 1:]).astype(f32)
    tw = (dy * xh).astype(f32).astype(np.float64).reshape(T, B, D)
    gw, gb = np.zeros((B, D)), np.zeros((B, D))
    for t in range(T):
        gw, gb = gw + tw[t], gb + dy.reshape(T, B, D)[t].astype(np.float64)
    s = 1.0 if mutation == "no-scale" else scale
    return dict(sqw=(gw * gw).sum(1), sqb=(gb * gb).sum(1), roww=(gw * s).astype(f32), rowb=(gb * s).astype(f32))


# ---- CPU: the emulations inside the bounds, the mutations outside ----------------------------------------------------
CPU_SEED, CPU_STEP, CPU_P = 1234567, 42, 0.3
# (rows, D, forward class, backward class): every class, tails of the fused CTAs (17 = 2 x 8 + 1, 33 = 32 + 1), two
# and more split chunks (257, 300), D not a multiple of 32 (the padded Philox index differs)
CPU_CASES = [(17, 84, V1, V1), (9, 152, V2, V2), (33, 260, V5, V5), (20, 644, GEN, SVEC), (300, 37, GEN, SSCAL),
             (9, 260, GEN, SSCAL), (257, 132, GEN, SVEC)]
CPU_FAMILIES = ["normal", "offset", "flat", "outliers", "pow2", "zero-dy"]
MUTATIONS = ["vec2-at-260", "keep-bit-off-by-one", "philox-padded-D", "swap-stats", "lost-warp", "s2-from-g",
             "lost-chunk", "no-scale"]


def philox_mask(rows, D, site, ld=None):
    from oracle.dropout_masks import dropout_mask_at
    ld = D if ld is None else ld
    idx = (np.arange(rows, dtype=np.uint64)[:, None] * np.uint64(ld) + np.arange(D, dtype=np.uint64)[None, :])
    return dropout_mask_at(CPU_SEED, CPU_STEP, site, idx, CPU_P)


def bits_mask(bits, D, p, shift=0):
    """the fused kernel's decode of keep words [rows, ld]: bit (j % 32) + shift of word j / 32"""
    j = np.arange(D)
    b = (bits[:, j // 32] >> ((j % 32 + shift) % 32).astype(np.uint32)) & np.uint32(1)
    ik = f32(1) / (f32(1) - f32(p))
    return np.where(b == 1, ik, f32(0)).astype(f32)


def pack_bits(keep, ld):
    """keep [rows, D] bool -> words [rows, ld] uint32"""
    rows, D = keep.shape
    k = np.zeros((rows, 32 * ld), np.uint64)
    k[:, :D] = keep
    return (k.reshape(rows, ld, 32) << np.arange(32, dtype=np.uint64)).sum(2).astype(np.uint32)


def cpu_run(case, family, mutation=None, eps=1e-5):
    """(bad, worst ratio) of one case: forward, backward on the forward's stats with the mask of the class's source,
    the per-sample kernels over rows = T*B"""
    rows, D, fc, bc = case
    x, dy, g, b = [t.numpy() for t in operands(rows, D, family, rows * 31 + D, "cpu")]
    eps32 = float(f32(eps))
    iters = 2 if mutation == "vec2-at-260" else None
    if mutation == "vec2-at-260" and not (fc == V5 and D == 260):
        return False, 0.0
    y, stats = emu_forward(x, g, b, eps32, fc, iters)
    xd, gd, bd, dyd = (torch.from_numpy(t).double() for t in (x, g, b, dy))
    rf = ref_forward(xd, gd, bd, eps32, fc)
    bad = []
    for out, key in ((y, "y"), (stats[:, 0], "mean"), (stats[:, 1], "rstd")):
        v, _ = violations(torch.from_numpy(out).double(), rf[key], rf["e_" + key])
        bad.append(bool(v.any()))
    # the mask: fused kernels read stored bits (= the Philox decisions), the split path draws Philox itself
    site = 32 + rows % 3
    pmask = philox_mask(rows, D, site)
    if bc in FUSED:
        ld = cdiv(D, 32) + 1
        words = pack_bits(pmask > 0, ld)
        words[:, -1] = 0xA5A5A5A5                    # a padding word the kernel must not read
        mask = bits_mask(words, D, CPU_P, 1 if mutation == "keep-bit-off-by-one" else 0)
        ref_mask = bits_mask(words, D, CPU_P)
    else:
        padded = cdiv(D, 32) * 32
        mask = philox_mask(rows, D, site, padded) if mutation == "philox-padded-D" else pmask
        ref_mask = pmask
    eb = emu_backward(x, stats, g, dy, bc, mask, mutation)
    rb = ref_backward(xd, torch.from_numpy(stats.copy()).double(), gd, dyd, bc, eb["chunks"],
                      torch.from_numpy(ref_mask).double())
    for key in ("dx", "dx_drop", "dgamma", "dbeta"):
        v, _ = violations(torch.from_numpy(eb[key]).double(), rb[key], rb["e_" + key])
        bad.append(bool(v.any()))
    # per sample: rows = T*B with B = the largest of 3, 2, 1 that divides rows
    B = next(k for k in (3, 2, 1) if rows % k == 0)
    T = rows // B
    ep = emu_per_sample(x, stats, dy, T, B, -0.75, mutation)
    rp = ref_per_sample(xd, torch.from_numpy(stats.copy()).double(), dyd, T, B, -0.75)
    for k in ("w", "b"):
        v, _ = violations(torch.from_numpy(ep["sq" + k]), rp["sq" + k], rp["e_sq" + k])
        bad.append(bool(v.any()))
        v, _ = violations(torch.from_numpy(ep["row" + k]).double(), -0.75 * rp["g" + k], rp["e_row" + k])
        bad.append(bool(v.any()))
    return any(bad), bad


@pytest.mark.parametrize("family", CPU_FAMILIES)
@pytest.mark.parametrize("eps", [1e-5, 1e-12, 1e-2])
def test_emulated_kernels_within_bound(family, eps):
    for case in CPU_CASES:
        bad, which = cpu_run(case, family, eps=eps)
        assert not bad, (case, family, eps, which)


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_bound_sees_each_mutation(mutation):
    assert any(cpu_run(case, family, mutation)[0] for case in CPU_CASES for family in CPU_FAMILIES), mutation


# ---- the debug entries' refusals (host checks only: nothing is launched) ---------------------------------------------
def ln_args(**kw):
    a = L.RdDebugLayernormArgs()
    for f in ("x", "gamma", "beta", "y", "stats", "dy", "dx", "dx_drop", "rng", "scratch", "dgamma", "dbeta"):
        setattr(a, f, FAKE)
    a.rows, a.D, a.eps, a.forward, a.backward = 100, 84, 1e-5, 1, 1
    a.scratch_floats = scratch_floats(100, 84)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("kw,what", [
    (dict(x=None), "NULL pointer"), (dict(gamma=None), "NULL pointer"), (dict(stats=None), "NULL pointer"),
    (dict(beta=None), "NULL pointer"), (dict(y=None), "NULL pointer"), (dict(dy=None), "NULL pointer"),
    (dict(dx=None), "NULL pointer"), (dict(scratch=None), "NULL pointer"), (dict(dgamma=None), "NULL pointer"),
    (dict(dbeta=None), "NULL pointer"), (dict(forward=0, backward=0), "neither half"),
    (dict(rows=0), "bad sizes"), (dict(D=0), "bad sizes"), (dict(rows=-5), "bad sizes"),
    (dict(scratch_floats=scratch_floats(100, 84) - 1), "scratch buffer of %d floats, it needs %d"
     % (scratch_floats(100, 84) - 1, scratch_floats(100, 84))),
    (dict(keep_bits=FAKE, keep_ld=2), "keep_ld 2 below ceil(D / 32) = 3"),
    (dict(drop_p=0.2, rng=None), "needs rng and dx_drop"), (dict(drop_p=0.2, dx_drop=None), "needs rng and dx_drop"),
    (dict(drop_p=1.0), "outside [0, 1)"), (dict(drop_p=-0.1), "outside [0, 1)"),
])
def test_layernorm_entry_refuses(kw, what):
    refused(lib().rd_debug_layernorm(C.byref(ln_args(**kw)), None), what)


def test_layernorm_entry_refuses_null_args_and_half_specific_pointers():
    refused(lib().rd_debug_layernorm(None, None), "NULL argument")
    # a backward-only call needs no beta / y, a forward-only call no dy / dx / scratch; both still refuse what they need
    refused(lib().rd_debug_layernorm(C.byref(ln_args(forward=0, dy=None)), None), "NULL pointer")
    refused(lib().rd_debug_layernorm(C.byref(ln_args(backward=0, y=None)), None), "NULL pointer")
    refused(lib().rd_debug_layernorm(C.byref(ln_args(backward=0, beta=None)), None), "NULL pointer")


@pytest.mark.parametrize("kw,what", [
    (dict(mode=L.RD_PS_ROTATED), "unknown mode"), (dict(mode=7), "unknown mode"), (dict(x=None), "NULL argument"),
    (dict(stats=None), "NULL argument"), (dict(dy=None), "NULL argument"), (dict(sq=None), "NULL argument"),
    (dict(mode=L.RD_PS_ROWS, G=None), "NULL argument"), (dict(T=0), "bad sizes"), (dict(B=0), "bad sizes"),
    (dict(D=0), "bad sizes"), (dict(fw=2), "outside nf"), (dict(fb=-1), "outside nf"),
    (dict(mode=L.RD_PS_ROWS, gw=300 - 83), "leave the row"), (dict(mode=L.RD_PS_ROWS, gb=-1), "leave the row"),
])
def test_per_sample_entry_refuses(kw, what):
    a = dict(mode=L.RD_PS_SQNORMS, x=FAKE, stats=FAKE, dy=FAKE, T=60, B=3, D=84, sq=FAKE, nf=2, fw=0, fb=1, G=FAKE,
             ldg=300, gw=0, gb=100)
    a.update(kw)
    refused(lib().rd_debug_per_sample_layernorm(a["mode"], a["x"], a["stats"], a["dy"], a["T"], a["B"], a["D"], a["sq"],
                                                a["nf"], a["fw"], a["fb"], a["G"], a["ldg"], a["gw"], a["gb"], 1.0,
                                                None), what)


# ---- GPU harness -----------------------------------------------------------------------------------------------------
GUARD = 32
F32_GUARD, F64_GUARD = 0x7FA5A5A5, 0x7FF4A5A5A5A5A5A5        # NaNs with payloads no kernel writes
PAD_ROWS = 3


class Guarded:
    """n elements at GUARD (+ shift) elements into a buffer filled with a NaN payload: 16-byte aligned unless shift"""

    def __init__(self, n, dtype=torch.float32, shift=0):
        self.bits = F32_GUARD if dtype == torch.float32 else F64_GUARD
        it = torch.int32 if dtype == torch.float32 else torch.int64
        self.buf = torch.full((n + 2 * GUARD + 1,), self.bits, dtype=it, device="cuda")
        self.lo, self.n = GUARD + shift, n
        self.t = self.buf[self.lo:self.lo + n].view(dtype)

    def ptr(self):
        return self.t.data_ptr()

    def guards_kept(self):
        return bool((self.buf[:self.lo] == self.bits).all() and (self.buf[self.lo + self.n:] == self.bits).all())

    def untouched(self):
        return bool((self.buf == self.bits).all())


def placed(t, shift=0, pad_rows=0):
    """a copy of t at `shift` floats past a 16-byte boundary, with pad_rows NaN rows after it"""
    rows = t.shape[0] if t.dim() > 1 else 1
    width = t.shape[-1]
    n = (rows + pad_rows) * width
    base = torch.full((n + 8,), float("nan"), device="cuda")
    v = base[4 + shift:4 + shift + n]
    v[:t.numel()] = t.reshape(-1)
    return base, v[:t.numel()].view(t.shape)


def rng_key(seed, step):
    return torch.tensor([seed, step], dtype=torch.int64, device="cuda")


def philox_mask_gpu(rng, site, rows, D, p):
    out = torch.empty(rows * D, device="cuda")
    L.check(lib().rd_debug_dropout_mask(rng.data_ptr(), site, rows * D, p, out.data_ptr(), L.stream_ptr()),
            "rd_debug_dropout_mask")
    return out.view(rows, D)


def to_i32(w):
    """uint32 values held in int64 -> the int32 words with the same bits"""
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32).contiguous()


def pack_bits_gpu(keep, ld):
    """keep [rows, D] bool -> int32 words [rows, ld] (bit j % 32 of word j / 32)"""
    rows, D = keep.shape
    k = torch.zeros(rows, 32 * ld, dtype=torch.int64, device="cuda")
    k[:, :D] = keep.long()
    return to_i32((k.view(rows, ld, 32) << torch.arange(32, device="cuda")).sum(2))


def mask_of_bits(words, D, p):
    j = torch.arange(D, device="cuda")
    b = (words.long()[:, j // 32] >> (j % 32)) & 1
    ik = float(np.float32(1) / (np.float32(1) - np.float32(p)))
    return torch.where(b == 1, ik, 0.0)


def run_ln(x, gamma, beta, dy, eps=1e-5, forward=True, backward=True, stats=None, drop_p=0.0, rng=None, site=32,
           keep=None, keep_ld=0, shift=(), dx_drop=True):
    """one rd_debug_layernorm call on placed operands (NaN rows past `rows` in x and dy; `shift`: the pointers moved by
    one float).  Every output is NaN-payload filled with guards, the scratch NaN-filled; the guards, and the outputs
    a half does not write, must keep their payload.  Returns the outputs (float64) and the written-back plan."""
    rows, D = x.shape
    s = lambda name: 1 if name in shift else 0
    _, xp = placed(x, s("x"), PAD_ROWS)
    _, dyp = placed(dy, s("dy"), PAD_ROWS)
    _, gp = placed(gamma, s("gamma"))
    _, bp = placed(beta, s("beta"))
    o = {k: Guarded(n, dt, s(k)) for k, n, dt in (("y", rows * D, torch.float32), ("dx", rows * D, torch.float32),
                                                   ("dx_drop", rows * D, torch.float32), ("dgamma", D, torch.float32),
                                                   ("dbeta", D, torch.float32))}
    st = Guarded(2 * rows)
    if stats is not None:
        st.t.copy_(stats.reshape(-1))
    nsc = scratch_floats(rows, D)
    scratch = torch.full((nsc,), float("nan"), device="cuda")
    a = L.RdDebugLayernormArgs()
    a.x, a.gamma, a.beta, a.dy, a.stats = xp.data_ptr(), gp.data_ptr(), bp.data_ptr(), dyp.data_ptr(), st.ptr()
    a.y, a.dx, a.dgamma, a.dbeta = o["y"].ptr(), o["dx"].ptr(), o["dgamma"].ptr(), o["dbeta"].ptr()
    a.dx_drop = o["dx_drop"].ptr() if dx_drop else None
    a.rng = rng.data_ptr() if rng is not None else None
    a.keep_bits = keep.data_ptr() if keep is not None else None
    a.keep_ld = keep_ld
    a.scratch, a.scratch_floats = scratch.data_ptr(), nsc
    a.rows, a.D, a.eps, a.drop_p, a.site = rows, D, eps, drop_p, site
    a.forward, a.backward = int(forward), int(backward)
    L.check(lib().rd_debug_layernorm(C.byref(a), L.stream_ptr()), "rd_debug_layernorm")
    torch.cuda.synchronize()
    for k, g in list(o.items()) + [("stats", st)]:
        assert g.guards_kept(), ("a write outside", k)
    if not forward:
        assert o["y"].untouched()
    if not backward:
        for k in ("dx", "dx_drop", "dgamma", "dbeta"):
            assert o[k].untouched(), k
    if backward and drop_p == 0.0:
        assert o["dx_drop"].untouched(), "dx_drop written at p = 0"
    out = {k: g.t.view(rows, D) if k in ("y", "dx", "dx_drop") else g.t for k, g in o.items()}
    out["stats"] = st.t.view(rows, 2)
    out = {k: v.clone() for k, v in out.items()}
    plan = dict(fwd=a.fwd_class, bwd=a.bwd_class, chunks=a.chunks, keep=a.keep_source)
    return out, plan


def check_forward(out, x, gamma, beta, eps, cls, family, tag=""):
    rf = ref_forward(x.double(), gamma.double(), beta.double(), float(np.float32(eps)), cls)
    path = CLASS_NAME[cls]
    check(("y", path, family), out["y"].double(), rf["y"], rf["e_y"], tag)
    check(("mean", path, family), out["stats"][:, 0].double(), rf["mean"], rf["e_mean"], tag)
    check(("rstd", path, family), out["stats"][:, 1].double(), rf["rstd"], rf["e_rstd"], tag)


def check_backward(out, plan, x, stats, gamma, dy, family, mask=None, tag=""):
    cls = plan["bwd"]
    rb = ref_backward(x.double(), stats.double(), gamma.double(), dy.double(), cls, plan["chunks"],
                      None if mask is None else mask.double())
    path = CLASS_NAME[cls]
    keys = ("dx", "dgamma", "dbeta") + (("dx_drop",) if mask is not None else ())
    for k in keys:
        check((k, path, family), out[k].double(), rb[k], rb["e_" + k], tag)
    if mask is not None:
        assert bool((out["dx_drop"][mask == 0] == 0).all()), (tag, "a dropped element is not 0")


def expect_plan(plan, rows, D, fwd=None, bwd=None, keep=None):
    if fwd is not None:
        assert plan["fwd"] == fwd, (plan, rows, D)
    if bwd is not None:
        assert plan["bwd"] == bwd, (plan, rows, D)
        assert plan["chunks"] == cdiv(rows, bwd_rows_per_cta(D, bwd)), (plan, rows, D)
    if keep is not None:
        assert plan["keep"] == keep, plan


# ---- GPU: every class and tail ---------------------------------------------------------------------------------------
TAIL_D = [1, 3, 4, 5, 124, 128, 129, 132, 252, 256, 257, 260, 636, 640, 641, 644, 1024]
TAIL_ROWS = [1, 7, 8, 9, 31, 32, 33, 255, 256, 257, 4097]


@pytest.mark.gpu
@pytest.mark.parametrize("D", TAIL_D)
def test_every_class_and_tail(D):
    """forward and backward in one call (the backward on the forward's stats, Philox dropout at p = 0.1), then the
    backward alone on exact stats; each class confirmed from the plan"""
    rng = rng_key(77, 5)
    for k, rows in enumerate(TAIL_ROWS):
        x, dy, gamma, beta = operands(rows, D, "normal", seed=D * 100 + k, device="cuda")
        site = 32 + k % 8
        out, plan = run_ln(x, gamma, beta, dy, drop_p=0.1, rng=rng, site=site)
        fc, bc = fwd_class(D), bwd_class(D)
        expect_plan(plan, rows, D, fc, bc, L.RD_LN_KEEP_PHILOX)
        tag = "D %d rows %d" % (D, rows)
        check_forward(out, x, gamma, beta, 1e-5, fc, "normal", tag)
        mask = philox_mask_gpu(rng, site, rows, D, 0.1)
        check_backward(out, plan, x, out["stats"], gamma, dy, "normal", mask, tag)
        ex = exact_stats(x.double(), float(np.float32(1e-5)))
        out2, plan2 = run_ln(x, gamma, beta, dy, forward=False, stats=ex)
        expect_plan(plan2, rows, D, None, bc, L.RD_LN_KEEP_NONE)
        check_backward(out2, plan2, x, ex, gamma, dy, "exact-stats", None, tag + " exact stats")
    print_worst()


@pytest.mark.gpu
@pytest.mark.parametrize("mis", ["beta", "dx_drop", "gamma", "x", "dy", "dx", "y"])
def test_one_pointer_misaligned(mis):
    """each pointer one float off in turn: beta alone (generic forward, fused backward), dx_drop alone (vector forward,
    split backward), gamma alone (both off), ..."""
    rng = rng_key(3, 9)
    for D in (84, 152, 528, 644):
        for rows in (9, 257):
            x, dy, gamma, beta = operands(rows, D, "normal", seed=rows + D, device="cuda")
            out, plan = run_ln(x, gamma, beta, dy, drop_p=0.2, rng=rng, site=64, shift=(mis,))
            f, b = plan_of((D, mis))
            if D <= 640:
                assert (f == GEN) == (mis in ("x", "y", "gamma", "beta"))
                assert (b in FUSED) == (mis in ("y", "beta"))
            expect_plan(plan, rows, D, f, b, L.RD_LN_KEEP_PHILOX)
            tag = "%s misaligned D %d rows %d" % (mis, D, rows)
            check_forward(out, x, gamma, beta, 1e-5, f, "misaligned", tag)
            check_backward(out, plan, x, out["stats"], gamma, dy, "misaligned",
                           philox_mask_gpu(rng, 64, rows, D, 0.2), tag)
    print_worst()


# ---- GPU: the keep masks ---------------------------------------------------------------------------------------------
def same_bits(a, b):
    it = torch.int32 if a.dtype == torch.float32 else torch.int64
    return torch.equal(a.contiguous().view(it), b.contiguous().view(it))


@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("layer", [0, 3])
def test_keep_masks(p, layer):
    """Philox at sites 32 + l and 64 + l; stored bits equal to the Philox decisions (padding words and the bits past
    D of the last word garbage) give the same bits as Philox on the fused and the split path; arbitrary bits are
    applied exactly on the fused path; the split path ignores them (it draws Philox)"""
    rng = rng_key(2024 + layer, 17)
    for site in (32 + layer, 64 + layer):
        for D, rows in ((84, 257), (152, 33), (528, 65), (100, 40)):
            x, dy, gamma, beta = operands(rows, D, "normal", seed=site * 7 + D, device="cuda")
            mask = philox_mask_gpu(rng, site, rows, D, p)
            ld = cdiv(D, 32) + 2
            g = torch.Generator(device="cuda").manual_seed(site + D)
            junk = torch.randint(0, 2 ** 32, (rows, ld), generator=g, device="cuda", dtype=torch.int64)
            w = pack_bits_gpu(mask > 0, ld).long() & 0xFFFFFFFF
            last, live = cdiv(D, 32) - 1, (1 << (D % 32 or 32)) - 1
            w[:, last] = (w[:, last] & live) | (junk[:, last] & (0xFFFFFFFF ^ live))    # garbage past D
            w[:, last + 1:] = junk[:, last + 1:]                                       # padding words
            words = to_i32(w)
            tag = "site %d D %d rows %d p %g" % (site, D, rows, p)
            for shift, path in (((), "fused"), (("dx_drop",), "split")):
                ph, pp = run_ln(x, gamma, beta, dy, drop_p=p, rng=rng, site=site, shift=shift)
                kb, pk = run_ln(x, gamma, beta, dy, drop_p=p, rng=rng, site=site, shift=shift, keep=words, keep_ld=ld)
                assert pp["keep"] == L.RD_LN_KEEP_PHILOX
                assert pk["keep"] == (L.RD_LN_KEEP_BITS if path == "fused" else L.RD_LN_KEEP_PHILOX), (pk, path)
                assert same_bits(ph["dx_drop"], kb["dx_drop"]), (tag, path, "stored Philox bits differ from Philox")
                check_backward(ph, pp, x, ph["stats"], gamma, dy, "keep-" + path, mask, tag)
            # arbitrary bits: the fused path applies exactly them, the split path still Philox
            arb = to_i32(torch.randint(0, 2 ** 32, (rows, ld), generator=g, device="cuda", dtype=torch.int64))
            amask = mask_of_bits(arb, D, p)
            fb, pf = run_ln(x, gamma, beta, dy, drop_p=p, rng=rng, site=site, keep=arb, keep_ld=ld)
            assert pf["keep"] == L.RD_LN_KEEP_BITS
            want = (fb["dx"] * amask).float()
            assert same_bits(fb["dx_drop"], want), (tag, "arbitrary bits not applied exactly")
            check_backward(fb, pf, x, fb["stats"], gamma, dy, "keep-bits", amask, tag)
            sb, ps = run_ln(x, gamma, beta, dy, drop_p=p, rng=rng, site=site, keep=arb, keep_ld=ld, shift=("dx_drop",))
            assert ps["keep"] == L.RD_LN_KEEP_PHILOX and ps["bwd"] == SSCAL
            sp, _ = run_ln(x, gamma, beta, dy, drop_p=p, rng=rng, site=site, shift=("dx_drop",))
            assert same_bits(sb["dx_drop"], sp["dx_drop"]), (tag, "the split path read the bits")
    print_worst()


# ---- GPU: operand families and production shapes ---------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("eps", [1e-5, 1e-12, 1e-2])
def test_operand_families(family, eps):
    rng = rng_key(11, 3)
    for D, rows in ((84, 300), (152, 257), (160, 64), (528, 129), (37, 100), (644, 70)):
        x, dy, gamma, beta = operands(rows, D, family, seed=D + rows, device="cuda")
        out, plan = run_ln(x, gamma, beta, dy, eps=eps, drop_p=0.2, rng=rng, site=33)
        tag = "%s eps %g D %d rows %d" % (family, eps, D, rows)
        check_forward(out, x, gamma, beta, eps, plan["fwd"], family, tag)
        check_backward(out, plan, x, out["stats"], gamma, dy, family, philox_mask_gpu(rng, 33, rows, D, 0.2), tag)
        ex = exact_stats(x.double(), float(np.float32(eps)))
        out2, plan2 = run_ln(x, gamma, beta, dy, forward=False, stats=ex)
        check_backward(out2, plan2, x, ex, gamma, dy, family + "-exact", None, tag + " exact stats")
    print_worst()


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["P19", "P12", "PAM", "LARGE"])
def test_production_shapes(config):
    D, rows = production_widths()[config]
    rng = rng_key(5, 1)
    fc, bc = PLAN_TABLE[(config, None)]
    for family in ("normal", "offset"):
        x, dy, gamma, beta = operands(rows, D, family, seed=rows, device="cuda")
        out, plan = run_ln(x, gamma, beta, dy, drop_p=0.2, rng=rng, site=65)
        expect_plan(plan, rows, D, fc, bc, L.RD_LN_KEEP_PHILOX)
        tag = "%s %s" % (config, family)
        check_forward(out, x, gamma, beta, 1e-5, fc, family, tag)
        check_backward(out, plan, x, out["stats"], gamma, dy, family, philox_mask_gpu(rng, 65, rows, D, 0.2), tag)
        del out
    print_worst()


@pytest.mark.gpu
def test_same_bits_across_runs():
    rng = rng_key(8, 8)
    for D, rows in ((84, 1000), (528, 300), (644, 300), (37, 300)):
        x, dy, gamma, beta = operands(rows, D, "normal", seed=D, device="cuda")
        a, _ = run_ln(x, gamma, beta, dy, drop_p=0.2, rng=rng, site=64)
        b, _ = run_ln(x, gamma, beta, dy, drop_p=0.2, rng=rng, site=64)
        for k in a:
            assert same_bits(a[k], b[k]), (D, k)


# ---- GPU: the per-sample kernels -------------------------------------------------------------------------------------
def run_per_sample(x, stats, dy, T, B, scale):
    """both modes; the NaN-payload guards, the unused field and every column of G outside the two fields must stay"""
    D = x.shape[1]
    _, xp = placed(x, 0, PAD_ROWS)
    _, dyp = placed(dy, 0, PAD_ROWS)
    _, sp = placed(stats, 0, PAD_ROWS)
    nf = 3
    sq = Guarded(B * nf, torch.float64)
    L.check(lib().rd_debug_per_sample_layernorm(L.RD_PS_SQNORMS, xp.data_ptr(), sp.data_ptr(), dyp.data_ptr(), T, B, D,
                                                sq.ptr(), nf, 2, 0, None, 0, 0, 0, 1.0, L.stream_ptr()),
            "rd_debug_per_sample_layernorm sqnorms")
    gw, gb = 3, 3 + D + 2
    ldg = gb + D + 1
    G = Guarded(B * ldg)
    L.check(lib().rd_debug_per_sample_layernorm(L.RD_PS_ROWS, xp.data_ptr(), sp.data_ptr(), dyp.data_ptr(), T, B, D,
                                                None, 0, 0, 0, G.ptr(), ldg, gw, gb, scale, L.stream_ptr()),
            "rd_debug_per_sample_layernorm rows")
    torch.cuda.synchronize()
    assert sq.guards_kept() and G.guards_kept()
    bits = sq.buf[sq.lo:sq.lo + B * nf].view(B, nf)
    assert bool((bits[:, 1] == F64_GUARD).all()), "a write to an unused field"
    gbits = G.buf[G.lo:G.lo + B * ldg].view(B, ldg)
    field = torch.zeros(ldg, dtype=torch.bool, device="cuda")
    field[gw:gw + D] = True
    field[gb:gb + D] = True
    assert bool((gbits[:, ~field] == F32_GUARD).all()), "a write outside the fields"
    s = sq.t.view(B, nf)
    Gv = G.t.view(B, ldg)
    return dict(sqw=s[:, 2].clone(), sqb=s[:, 0].clone(), roww=Gv[:, gw:gw + D].double(),
                rowb=Gv[:, gb:gb + D].double())


PS_SHAPES = [(T, B) for T in (1, 60, 215, 600) for B in (1, 3, 33, 128)]
PS_D = [84, 152, 160, 528, 3, 257]


@pytest.mark.gpu
@pytest.mark.parametrize("T,B", PS_SHAPES)
def test_per_sample_kernels(T, B):
    """against float64, then Sum_b of the scale-1 rows against rd_debug_layernorm's dgamma / dbeta on the same
    (x, stats, dy), and each row's squared norm against dp_ln_sqnorm, each within the sum of the two bounds"""
    D = PS_D[(T + B) % len(PS_D)]
    rows = T * B
    family = ("normal", "offset", "zero-dy", "pow2")[PS_SHAPES.index((T, B)) % 4]
    x, dy, gamma, beta = operands(rows, D, family, seed=T * 1000 + B, device="cuda")
    fw, _ = run_ln(x, gamma, beta, dy, backward=False)
    stats = fw["stats"].float()
    scale = -0.75
    o = run_per_sample(x, stats, dy, T, B, scale)
    r = ref_per_sample(x.double(), stats.double(), dy.double(), T, B, scale)
    tag = "T %d B %d D %d" % (T, B, D)
    check(("sqw", "per-sample", family), o["sqw"], r["sqw"], r["e_sqw"], tag)
    check(("sqb", "per-sample", family), o["sqb"], r["sqb"], r["e_sqb"], tag)
    check(("roww", "per-sample", family), o["roww"], scale * r["gw"], r["e_roww"], tag)
    check(("rowb", "per-sample", family), o["rowb"], scale * r["gb"], r["e_rowb"], tag)
    # cross-checks at scale 1
    o1 = run_per_sample(x, stats, dy, T, B, 1.0)
    r1 = ref_per_sample(x.double(), stats.double(), dy.double(), T, B, 1.0)
    bw, pb = run_ln(x, gamma, beta, dy, forward=False, stats=stats)
    rb = ref_backward(x.double(), stats.double(), gamma.double(), dy.double(), pb["bwd"], pb["chunks"])
    for k, name in (("w", "dgamma"), ("b", "dbeta")):
        diff = (o1["row" + k].sum(0) - bw[name].double()).abs()
        bound = r1["e_row" + k].sum(0) + rb["e_" + name] + f64(B + 4) * o1["row" + k].abs().sum(0)
        assert bool((diff <= bound).all()), (tag, k, ratio_of(diff, bound))
        WORST[("sum-rows-" + k, "cross", family)] = max(WORST.get(("sum-rows-" + k, "cross", family), 0.0),
                                                       ratio_of(diff, bound))
        rn2 = (o1["row" + k] ** 2).sum(1)
        d = r1["e_row" + k]
        g = r1["g" + k].abs()
        bound = r1["e_sq" + k] + (2 * g * d + d * d).sum(1) + f64(D + 8) * ((g + d) ** 2).sum(1)
        diff = (rn2 - o1["sq" + k]).abs()
        assert bool((diff <= bound).all()), (tag, k, "row norm vs sqnorm", ratio_of(diff, bound))
        WORST[("rownorm-" + k, "cross", family)] = max(WORST.get(("rownorm-" + k, "cross", family), 0.0),
                                                      ratio_of(diff, bound))
    o2 = run_per_sample(x, stats, dy, T, B, scale)
    for k in o:
        assert same_bits(o[k], o2[k]), (tag, k, "two runs differ")
    print_worst()
