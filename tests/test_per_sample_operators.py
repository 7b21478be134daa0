"""The per-sample gradient kernels on their own, element by element against float64.

DP-SGD, TracIn, TracIn-RP, EK-FAC and the Laplace approximation stand on three kernels of rd_dp.cu and rd_influence.cu:
  * dp_norm_tile_kernel + dp_norm_finalize_kernel: per-sample squared norms of a linear layer's weight and bias
    gradients, in the ghost form (64 x 64 tiles of the R x R Gram triangle, off-diagonal tiles counted twice) or the
    explicit form (64 x 64 tiles of the sample's [Nout, Kin + 1] product dY_b^T [X_b | 1], then sums of squares);
  * psg_tile_kernel<false / true>: the explicit product written out as gradient rows, times `scale`, rounded once;
    <true> (EK-FAC) reads Kin + 1 columns of an already rotated [X | 1] Q_A and appends no ones column;
  * psg_dot_kernel + psg_dot_reduce_kernel (rd_per_sample_grad_dot): the TracIn inner products on wgmma 3xTF32.
The linear items run here through rd_debug_per_sample_linear, one group launch exactly as the backward's gradient
consumer issues it, with the form forced or chosen (written back with tm, tn and the tiles per sample); the dot runs
through its public entry.  Every output is held to a bound DERIVED below, element by element or per norm.

Notation: u = 2^-24, gamma_k = k u / (1 - k u); x~ = [x | 1] (rotated mode: x~ = x, Kin + 1 columns); e = the exact
product P[m, n] = sum_r y_rm x~_rn over the sample's R rows; S[m, n] = sum_r |y_rm| |x~_rn|.  "fp64 terms" below are
bounded by k 2^-53 times the matching sum of magnitudes (k the number of fp64 operations in the chain) and are added
to every bound in that form; they also cover the float64 rounding of the reference itself.

Explicit form and rows.  The kernels sum each 16-row slice of the contraction with a chain of 16 fp32 fmaf (rows past
R load as exact zeros) and add the slices to fp64 accumulators.  A chain of k fmaf errs by at most gamma_k times the sum
of the magnitudes of its products, so
    |e^ - e| <= delta = gamma_16 S + fp64 terms.
  * Rows mode rounds scale * e^ (an fp64 product) to fp32 once:
    |G - scale e| <= |scale| delta + u |scale| (|e| + delta).
  * The norms add the squares in fp64: |e^2 - e^2| = |e^ - e| |e^ + e| <= 2 |e| delta + delta^2, so
    | ||W^||^2 - ||W||^2 | <= sum_mn (2 |e_mn| delta_mn + delta_mn^2) + fp64 terms (bias: over the ones column).
Ghost form.  Each Gram entry g_rr' = sum_k y_rk y_r'k (X: over the Kin columns of x, without the ones column) is summed
the same way along k, so |g^ - g| <= dg = gamma_16 a_rr' + fp64 terms with a_rr' = sum_k |y_rk| |y_r'k|.  The weight
norm is sum_rr' gy gx, the bias norm sum_rr' gy, added in fp64 tile by tile:
    weight: sum_rr' (dgy |gx| + |gy| dgx + dgy dgx) + fp64 terms  <= about 2 gamma_16 (sum_r ||y_r|| ||x_r||)^2
    bias:   sum_rr' dgy + fp64 terms                              <= gamma_16 (sum_r ||y_r||)^2
  (Cauchy-Schwarz gives the closed forms; the tests use the sums, which are tighter.)  These bounds are ABSOLUTE, not
  relative to the result: when a sample's rows cancel (sum_r y_r x~_r^T ~ 0, the "cancel" family) the norm is far
  below its bound and the ghost form may return it NEGATIVE (every term of the explicit form is a square, so that form
  never does).  The kernels do not clamp: the count of negative ghost norms on that family is printed, and DESIGN §3
  records it.  No model-level test meets one (test_dp_sgd.py holds the model's norms to 1e-5 relative); a clamp
  would wait for a model input that does.
The dot.  One CTA per (64 queries, 128 train rows, segment); each 32-column k-block of a segment is 3xTF32 with K = 32
into fresh accumulators (test_gemm_operators.py: (6 ceil(32/8) + 48) u S_k = 72 u S_k, train columns past the segment's
end zeroed), the k-block sums are folded in order in fp32 round-to-nearest (kb - 1 roundings after the exact first,
each below u times a running sum bounded by S (1 + 72 u); one more u S covers the second-order terms), and the reduce
adds the segments in order in fp64, times alpha, onto the scores:
    |score - (score0 + alpha sum_s P_s)| <= |alpha| sum_s (72 + kb_s) u S_s + fp64 terms,
  S_s = sum_{j in s} |gq_j| |gt_j|, kb_s = ceil(len_s / 32).
  Precondition (header of rd_per_sample_grad_dot): the train side is zeroed past a segment's end, but the query side
  is read up to the end of the segment's last k-block and multiplied by those zeros, so a NaN or Inf there poisons
  the score (0 * Inf = NaN).  Every caller passes finite rows (bucket padding is 0); the tests fill the columns
  outside every segment with finite +-1e30 in both operands, which must move no score.

CPU: a numpy emulation of both tile kernels (16-row fp32 slices, products exact in fp64 and rounded once per step, fp64
across slices, the kernel's triangle decode) stays inside the bounds on every operand family, and each of these
mutations breaks them on at least one case: (a) an off-diagonal ghost tile not doubled; (b) the triangle decode
skipping the last diagonal tile, or visiting (i, j) with j < i; (c) the ones column missing where it is alone in its
tile (tn = ceil(Kin / 64) instead of ceil((Kin + 1) / 64), Kin % 64 == 0); (d) the last partial 16-slice of the
contraction dropped; (e) the sample and row strides swapped; (f) rotated mode appending a ones column.  An emulation of
the dot stays inside its bound, and accumulating a whole segment in the tensor cores' truncating accumulator breaks it
on same-sign rows.  A restatement of dp_ghost, dp_norm_tiles and psg_tiles reproduces the DESIGN §3 form table, and
the debug entry's refusals are checked.
GPU: linear items at R in {1, 15, 16, 17, 63, 64, 65, 128, 129, 257} (ghost tm up to 5), Nout in {1, 63, 64, 65, 130},
Kin in {1, 62, 63, 64, 65, 127} (Kin = 63: the ones column last in tile 0; 64: alone in a new tile), B in {1, 3, 33},
both forced forms on each shape and the shape's own choice bit for bit; the encoder (sstride 1, rstride B) and ob-prop
(sstride R, rstride 1) layouts; NaN in the columns past Nout / Kin (/ Kin + 1 rotated), NaN-payload guards around every
output and in every column of G outside the items' fields; six operand families; the same bits alone, anywhere in a
group of 32 mixed items, and across runs.  The dot at Bq in {1, 63, 64, 65, 130} x Bt in {1, 63, 64, 65, 128, 129,
300}, segments of 1 to 4096 columns, adjacent and ending at an ldg that is not a multiple of 32, +-1e30 outside the
segments, lds > Bt with NaN canaries, += onto nonzero scores with alpha = -0.7, four families, and the same bits across
query and train sub-blocks and permutations.  The worst err / bound of each family is printed.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from raindrop_b200 import lib as L
from test_gemm_operators import FAKE, U, emulate_3xtf32, refused, tc_bound

TILE, SLICE, MAX_ITEMS = 64, 16, 32
GAMMA16 = 16 * U / (1 - 16 * U)
FAMILIES = ["random", "scaled", "relu", "zero", "tf32", "cancel"]
WORST = {}
NEGATIVE = {}       # family -> (negative ghost norms, ghost norms)


def lib():
    return L.load()


def f64(k):
    """k fp64 roundings, each below 2^-53 of the running magnitude (1 % covers the second-order terms)"""
    return k * 2.0 ** -53 * 1.01


def cdiv(a, b):
    return -(-a // b)


# ---- the tile plans, restated ----------------------------------------------------------------------------------------
def dp_ghost(R, nout, kin):
    return R * (nout + kin + 1) < nout * (kin + 1)


def dp_norm_tiles(R, nout, kin, ghost):
    """(tm, tn, tiles per sample) of the given form"""
    if ghost:
        tm = cdiv(R, TILE)
        return tm, tm, tm * (tm + 1) // 2
    tm, tn = cdiv(nout, TILE), cdiv(kin + 1, TILE)
    return tm, tn, tm * tn


def psg_tiles(nout, kin):
    tn = cdiv(kin + 1, TILE)
    return cdiv(nout, TILE), tn, cdiv(nout, TILE) * tn


def model_items(config):
    """(encoder items, ob-prop items) of a model config: (R, Nout, Kin) of each linear of one layer"""
    from raindrop_b200.synth import model_config
    c = model_config(config)
    D, nhid, T, N = c["d_model"] + 16, c["nhid"], c["max_len"], c["d_inp"]
    C_ = T * c["d_ob"]
    return [(T, 3 * D, D), (T, D, D), (T, nhid, D), (T, D, nhid)], [(N, C_, C_)]


# DESIGN §3: (encoder form, tiles per sample), (ob-prop form, tiles per sample)
FORM_TABLE = {"TINY": (("ghost", 1), ("ghost", 1)), "TINY8": (("ghost", 1), ("ghost", 1)),
              "P19": (("ghost", 1), ("ghost", 1)), "P12": (("explicit", None), ("ghost", 1)),
              "PAM": (("explicit", None), ("ghost", 1)), "LARGE": (("ghost", 10), ("ghost", 3))}


@pytest.mark.parametrize("config", sorted(FORM_TABLE))
def test_form_table_matches_design(config):
    enc, ob = model_items(config)
    for items, (form, tiles) in zip((enc, ob), FORM_TABLE[config]):
        for R, nout, kin in items:
            g = dp_ghost(R, nout, kin)
            assert ("ghost" if g else "explicit") == form, (config, R, nout, kin)
            if tiles is not None:
                assert dp_norm_tiles(R, nout, kin, g)[2] == tiles, (config, R, nout, kin)
    ob_rows = {"TINY": 5, "TINY8": 6, "P19": 34, "P12": 36, "PAM": 17, "LARGE": 128}
    assert ob[0][0] == ob_rows[config]


# ---- float64 references and bounds (torch, any device) --------------------------------------------------------------
def reference(Y, X, rotated):
    """Y [B, R, Nout], X [B, R, Kin] (rotated: Kin + 1 columns, the bias column included), float64.  Returns the product
    P = Y^T X~ [B, Nout, Kin + 1], the element bound d (delta of the module docstring, which also covers the reference's
    own fp64 rounding), the exact squared norms and both forms' norm bounds."""
    B, R, nout = Y.shape
    Xt = X if rotated else torch.cat([X, torch.ones(B, R, 1, dtype=X.dtype, device=X.device)], 2)
    kin = Xt.shape[2] - 1
    P = Y.transpose(1, 2) @ Xt
    S = Y.abs().transpose(1, 2) @ Xt.abs()
    d = (GAMMA16 + f64(2 * R + 4)) * S
    a = P.abs() + f64(R + 2) * S                      # >= |e|
    r = dict(P=P, S=S, d=d, a=a, kin=kin, w=(P[..., :kin] ** 2).sum((1, 2)), b=(P[..., kin] ** 2).sum(1))
    nterm = nout * (kin + 1) + 2 * TILE
    sq, big = 2 * a * d + d * d, (a + d) ** 2
    r["expl_w"] = sq[..., :kin].sum((1, 2)) + f64(nterm) * big[..., :kin].sum((1, 2))
    r["expl_b"] = sq[..., kin].sum(1) + f64(nterm) * big[..., kin].sum(1)
    if not rotated:
        gy, ay = Y @ Y.transpose(1, 2), Y.abs() @ Y.abs().transpose(1, 2)
        gx, ax = X @ X.transpose(1, 2), X.abs() @ X.abs().transpose(1, 2)
        dy, dx = (GAMMA16 + f64(2 * nout + 4)) * ay, (GAMMA16 + f64(2 * kin + 4)) * ax
        n2 = R * R + 2 * R + 2 * TILE
        r["ghost_w"] = ((dy * gx.abs() + gy.abs() * dx + dy * dx).sum((1, 2)) +
                        f64(n2) * ((ay + dy) * (ax + dx)).sum((1, 2)))
        r["ghost_b"] = dy.sum((1, 2)) + f64(n2) * (ay + dy).sum((1, 2))
        r["gram_scale"] = (ay.sum((1, 2)), (ay * ax).sum((1, 2)))
    return r


def row_bound(r, scale):
    return abs(scale) * r["d"] + (U + 2 * 2.0 ** -53) * abs(scale) * (r["a"] + r["d"])


def record(key, ratio):
    WORST[key] = max(WORST.get(key, 0.0), ratio)


def ratio_of(err, bound):
    live = bound > 0
    return float((err[live] / bound[live]).max()) if live.any() else 0.0


def norm_violations(w, b, r, ghost):
    """bool [B] per norm (NaN counts), and the worst err / bound"""
    bw, bb = (r["ghost_w"], r["ghost_b"]) if ghost else (r["expl_w"], r["expl_b"])
    ew, eb = (w - r["w"]).abs(), (b - r["b"]).abs()
    bad = ~(ew <= bw) | ~(eb <= bb)
    return bad, max(ratio_of(ew, bw), ratio_of(eb, bb))


def rows_violations(out, r, scale):
    """out [B, Nout, Kin + 1] (NaN where nothing was written counts)"""
    bound = row_bound(r, scale)
    err = (out - scale * r["P"]).abs()
    return ~(err <= bound), ratio_of(err[~torch.isnan(err)], bound[~torch.isnan(err)])


# ---- operands --------------------------------------------------------------------------------------------------------
def tf32_rn(x):
    return ((x.view(torch.int32) + 0x1000) & -8192).view(torch.float32)


def logical_operands(B, R, nout, kx, family, seed, device="cuda"):
    """Y [B, R, nout], X [B, R, kx] float32: sample b's rows in order"""
    g = torch.Generator(device=device).manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device=device, dtype=torch.float64)
    Y, X = rn(B, R, nout), rn(B, R, kx)
    if family == "scaled":             # rows and columns scaled by 2^-10 .. 2^10 each: elements over 2^-20 .. 2^20
        e = lambda *s: torch.exp2(torch.randint(-10, 11, s, generator=g, device=device).double())
        Y, X = Y * e(B, R, 1) * e(1, 1, nout), X * e(B, R, 1) * e(1, 1, kx)
    elif family == "relu":             # post-ReLU X, positive dY
        Y, X = Y.abs(), X.clamp_min(0.0)
    elif family == "zero":             # padded tokens: dY rows past each sample's length are 0 (sample 0 all 0)
        n = torch.randint(0, R + 1, (B, 1), generator=g, device=device)
        n[0] = 0 if B > 1 else n[0]
        Y = Y * (torch.arange(R, device=device)[None, :] < n)[..., None]
    elif family == "tf32":
        X = tf32_rn(X.float()).double()
    elif family == "cancel":           # rows in pairs (y, x), (-y + 1e-4 z, x): sum_r y_r x~_r^T ~ 1e-4 of its terms
        h = R // 2
        Y[:, h:2 * h] = -Y[:, :h] + 1e-4 * rn(B, h, nout)
        X[:, h:2 * h] = X[:, :h]
        if R % 2:
            Y[:, -1] = 0.0
    return Y.float(), X.float()


def sample_rows(B, R, sstride, rstride, device="cuda"):
    """[B, R] buffer row of sample b's row t"""
    return torch.arange(B, device=device)[:, None] * sstride + torch.arange(R, device=device)[None, :] * rstride


LAYOUTS = {"enc": lambda B, R: (1, B), "ob": lambda B, R: (R, 1)}


# ---- CPU: the tile kernels' arithmetic in numpy, and mutations of it ------------------------------------------------
def fma_step(c, a, b):
    """c + a b rounded to fp32 once: the product of two fp32 values is exact in fp64 (one rounding where the kernel's
    fmaf has one; the fp64 sum may round first, at most 2^-53 more)"""
    return (c.astype(np.float64) + np.multiply.outer(a.astype(np.float64), b.astype(np.float64))).astype(np.float32)


def emu_product(Yb, Xt, drop_tail=False):
    """[Nout, K] = Yb^T Xt as the explicit tiles sum it: 16-row fp32 fmaf chains, fp64 across slices"""
    R = Yb.shape[0]
    e = np.zeros((Yb.shape[1], Xt.shape[1]))
    stop = R - R % SLICE if drop_tail else R
    for r0 in range(0, stop, SLICE):
        c = np.zeros(e.shape, np.float32)
        for k in range(r0, min(r0 + SLICE, R)):
            c = fma_step(c, Yb[k], Xt[k])
        e += c
    return e


def emu_gram(P, drop_tail=False):
    """[R, R] = P P^T as gram_tile sums it: 16-column fp32 fmaf chains, fp64 across slices"""
    K = P.shape[1]
    g = np.zeros((P.shape[0], P.shape[0]))
    stop = K - K % SLICE if drop_tail else K
    for k0 in range(0, stop, SLICE):
        c = np.zeros(g.shape, np.float32)
        for k in range(k0, min(k0 + SLICE, K)):
            c = fma_step(c, P[:, k], P[:, k])
        g += c
    return g


def triangle(tm, mutation=None):
    """dp_norm_tile_kernel's decode of tile index -> (i, j); (b-last) one tile short, (b-lower) without j += i"""
    for tile in range(tm * (tm + 1) // 2 - (mutation == "b-last")):
        i, j = 0, tile
        while j >= tm - i:
            j -= tm - i
            i += 1
        yield (i, j) if mutation == "b-lower" else (i, j + i)


def emu_ghost(Yb, Xb, mutation=None):
    gy, gx = emu_gram(Yb, mutation == "d"), emu_gram(Xb, mutation == "d")
    w = b = 0.0
    for i, j in triangle(cdiv(Yb.shape[0], TILE), mutation):
        bi, bj = slice(i * TILE, (i + 1) * TILE), slice(j * TILE, (j + 1) * TILE)
        pw, pb = float((gy[bi, bj] * gx[bi, bj]).sum()), float(gy[bi, bj].sum())
        if i != j and mutation != "a":
            pw, pb = 2 * pw, 2 * pb
        w, b = w + pw, b + pb
    return w, b


def emu_tiles_product(Yb, Xb, kin, rotated, mutation, unwritten=np.nan):
    """the [Nout, Kin + 1] product of the explicit / rows tiles, `unwritten` where no tile runs"""
    ones = np.ones((Yb.shape[0], 1), np.float32)
    Xt = Xb if rotated else np.concatenate([Xb, ones], 1)
    if rotated and mutation == "f":
        Xt = np.concatenate([Xb[:, :kin], ones], 1)
    e = emu_product(Yb, Xt, mutation == "d")
    if mutation == "c":
        e[:, cdiv(kin, TILE) * TILE:] = unwritten
    return e


def emulate(item, mode, mutation=None, scale=1.0):
    """the outputs of one item: (w [B], b [B]) in sqnorms mode, rows [B, Nout, Kin + 1] in the rows modes"""
    Y, X, B, R, kin = item["Y"], item["X"], item["B"], item["R"], item["kin"]
    ss, rs = LAYOUTS[item["layout"]](B, R)
    if mutation == "e":
        ss, rs = rs, ss
    rows = sample_rows(B, R, ss, rs, "cpu").numpy() % (B * R)      # swapped strides may leave the buffer
    Yf, Xf = item["Ybuf"], item["Xbuf"]
    out = []
    for b in range(B):
        Yb, Xb = Yf[rows[b]], Xf[rows[b]]
        if mode == "sqnorms" and item["ghost"]:
            out.append(emu_ghost(Yb, Xb, mutation))
        else:
            e = emu_tiles_product(Yb, Xb, kin, mode == "rotated", mutation, 0.0 if mode == "sqnorms" else np.nan)
            if mode == "sqnorms":
                out.append(((e[:, :kin] ** 2).sum(), (e[:, kin] ** 2).sum()))
            else:
                out.append((e * scale).astype(np.float32))
    if mode == "sqnorms":
        return torch.tensor([o[0] for o in out]), torch.tensor([o[1] for o in out])
    return torch.from_numpy(np.stack(out)).double()


def cpu_item(B, R, nout, kin, family, layout, ghost=False, rotated=False, seed=0):
    kx = kin + 1 if rotated else kin
    Y, X = logical_operands(B, R, nout, kx, family, seed, "cpu")
    ss, rs = LAYOUTS[layout](B, R)
    rows = sample_rows(B, R, ss, rs, "cpu").reshape(-1)
    Ybuf, Xbuf = torch.zeros(B * R, nout), torch.zeros(B * R, kx)
    Ybuf[rows], Xbuf[rows] = Y.reshape(B * R, nout), X.reshape(B * R, kx)
    return dict(Y=Y, X=X, Ybuf=Ybuf.numpy(), Xbuf=Xbuf.numpy(), B=B, R=R, kin=kin, layout=layout, ghost=ghost,
                rotated=rotated, ref=reference(Y.double(), X.double(), rotated))


# (B, R, Nout, Kin, layout, mode, ghost): tm = 2 and 3 ghost triangles, partial slices of 4 / 5 / 8 and 15, Kin = 64
# (the ones column alone in tile 1), both layouts with B <= R (swapped strides stay inside the buffer)
CPU_CASES = [(2, 80, 20, 24, "enc", "sqnorms", True), (1, 150, 21, 8, "ob", "sqnorms", True),
             (3, 21, 20, 64, "enc", "sqnorms", False), (2, 37, 5, 64, "ob", "sqnorms", False),
             (3, 21, 20, 64, "enc", "rows", False), (2, 37, 5, 63, "ob", "rows", False),
             (3, 21, 20, 64, "enc", "rotated", False), (2, 17, 9, 63, "ob", "rotated", False)]
MUTATIONS = ["a", "b-last", "b-lower", "c", "d", "e", "f"]
CPU_SCALE = -3.0


def cpu_check(case, family, mutation=None):
    B, R, nout, kin, layout, mode, ghost = case
    it = cpu_item(B, R, nout, kin, family, layout, ghost, mode == "rotated", seed=R + nout + len(family))
    if mode == "sqnorms":
        bad, ratio = norm_violations(*emulate(it, mode, mutation), it["ref"], ghost)
    else:
        bad, ratio = rows_violations(emulate(it, mode, mutation, CPU_SCALE), it["ref"], CPU_SCALE)
    return bool(bad.any()), ratio


@pytest.mark.parametrize("family", FAMILIES)
def test_emulated_tiles_within_bound(family):
    for case in CPU_CASES:
        bad, ratio = cpu_check(case, family)
        assert not bad, (case, family, ratio)


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_bound_sees_each_mutation(mutation):
    hits = [(case, family) for case in CPU_CASES for family in FAMILIES if cpu_check(case, family, mutation)[0]]
    assert hits, mutation


def test_ghost_form_can_go_negative_on_cancelling_rows():
    """the ghost form's error is absolute: on cancelling rows the emulated norm lands on either side of zero (inside
    its bound), where the explicit form's sum of squares cannot"""
    neg = 0
    for seed in range(40):
        it = cpu_item(1, 6, 16, 16, "cancel", "enc", ghost=True, seed=seed)
        w, b = emulate(it, "sqnorms")
        bad, _ = norm_violations(w, b, it["ref"], True)
        assert not bad.any(), seed
        neg += int((w < 0).sum() + (b < 0).sum())
    print("negative ghost norms on cancelling rows: %d of 80" % neg)
    assert neg > 0


# the dot: k-blocks of 32 columns in fresh accumulators, folded in fp32 round-to-nearest, segments in fp64
def emulate_dot(Gq, Gt, segs, fresh=True):
    out = np.zeros((Gq.shape[0], Gt.shape[0]))
    for off, ln in segs:
        acc = np.zeros((Gt.shape[0], Gq.shape[0]), np.float32)
        if not fresh:                      # the whole segment in the tensor cores' truncating accumulator
            acc = emulate_3xtf32(Gt[:, off:off + ln], Gq[:, off:off + ln])
        else:
            for k0 in range(0, ln, 32):
                k1 = min(k0 + 32, ln)
                A = np.zeros((Gt.shape[0], 32), np.float32)
                A[:, :k1 - k0] = Gt[:, off + k0:off + k1]
                Bq = np.zeros((Gq.shape[0], 32), np.float32)
                Bq[:, :k1 - k0] = Gq[:, off + k0:off + k1]
                acc = (acc + emulate_3xtf32(A, Bq)).astype(np.float32)
        out += acc.T.astype(np.float64)
    return out


def dot_coef(ln):
    return tc_bound(32, True) + cdiv(ln, 32)


def dot_check_np(out, Gq, Gt, segs):
    q, t = Gq.astype(np.float64), Gt.astype(np.float64)
    P, bound = np.zeros(out.shape), np.zeros(out.shape)
    for off, ln in segs:
        s = slice(off, off + ln)
        P += q[:, s] @ t[:, s].T
        bound += (dot_coef(ln) * U + f64(ln + len(segs) + 4)) * (np.abs(q[:, s]) @ np.abs(t[:, s]).T)
    return np.abs(out - P) <= bound


@pytest.mark.parametrize("positive", [False, True])
def test_emulated_dot_within_bound(positive):
    rng = np.random.default_rng(3 + positive)
    draw = (lambda *s: rng.random(s)) if positive else (lambda *s: rng.standard_normal(s))
    Gq, Gt = draw(5, 1200).astype(np.float32), draw(6, 1200).astype(np.float32)
    segs = [(0, 1), (4, 33), (40, 64), (104, 1096)]
    assert dot_check_np(emulate_dot(Gq, Gt, segs), Gq, Gt, segs).all()


def test_dot_bound_sees_one_truncating_accumulator():
    """same-sign rows over a 4096-column segment: without the fresh accumulators the truncation drifts past the bound"""
    rng = np.random.default_rng(7)
    Gq, Gt = rng.random((3, 4096)).astype(np.float32), rng.random((4, 4096)).astype(np.float32)
    segs = [(0, 4096)]
    assert dot_check_np(emulate_dot(Gq, Gt, segs), Gq, Gt, segs).all()
    assert not dot_check_np(emulate_dot(Gq, Gt, segs, fresh=False), Gq, Gt, segs).all()


# ---- the debug entry's refusals --------------------------------------------------------------------------------------
def items_array(specs):
    arr = (L.RdDebugPerSampleItem * max(len(specs), 1))()
    for a, s in zip(arr, specs):
        for k, v in s.items():
            setattr(a, k, v)
    return arr


def fake_spec(**kw):
    s = dict(d_out=FAKE, x=FAKE, ld_out=64, ld_x=68, sstride=1, rstride=4, gw=0, gb=64 * 64, R=10, out_features=64,
             in_features=64, fw=0, fb=1, form=-1)
    s.update(kw)
    return s


def call(specs, mode=L.RD_PS_SQNORMS, B=4, nf=2, partial_bytes=1 << 30, ldg=64 * 65, sq=FAKE, partial=FAKE, G=FAKE,
         n=None, plan=True):
    n = len(specs) if n is None else n
    plans = (L.RdDebugPerSamplePlan * max(n, 1))()
    return lib().rd_debug_per_sample_linear(items_array(specs), n, B, mode, sq, nf, partial, partial_bytes, G, ldg,
                                            1.0, plans if plan else None, None)


@pytest.mark.parametrize("n", [0, MAX_ITEMS + 1])
def test_refuses_item_counts(n):
    refused(call([fake_spec()] * max(n, 1), n=n), "items, it takes 1 to 32")


@pytest.mark.parametrize("kw,mode,what", [
    (dict(), 3, "unknown mode"), (dict(), -1, "unknown mode"),
    (dict(form=2), L.RD_PS_SQNORMS, "unknown form"), (dict(form=-2), L.RD_PS_SQNORMS, "unknown form"),
    (dict(d_out=0), L.RD_PS_SQNORMS, "NULL pointer"), (dict(x=0), L.RD_PS_ROWS, "NULL pointer"),
    (dict(R=0), L.RD_PS_SQNORMS, "bad sizes"), (dict(out_features=0), L.RD_PS_ROWS, "bad sizes"),
    (dict(in_features=0), L.RD_PS_SQNORMS, "bad sizes"), (dict(sstride=0), L.RD_PS_SQNORMS, "bad sizes"),
    (dict(rstride=0), L.RD_PS_ROWS, "bad sizes"), (dict(ld_out=63), L.RD_PS_SQNORMS, "bad sizes"),
    (dict(ld_x=63), L.RD_PS_ROWS, "bad sizes"), (dict(ld_x=64), L.RD_PS_ROTATED, "bad sizes"),
    (dict(fw=2), L.RD_PS_SQNORMS, "outside nf"), (dict(fb=-1), L.RD_PS_SQNORMS, "outside nf"),
    (dict(gw=65), L.RD_PS_ROWS, "leave the row"), (dict(gb=64 * 64 + 1), L.RD_PS_ROTATED, "leave the row"),
    (dict(gw=-1), L.RD_PS_ROWS, "leave the row"),
])
def test_refuses_bad_items(kw, mode, what):
    spec = fake_spec()
    spec.update(kw)
    refused(call([fake_spec(), spec], mode), what)


def test_refuses_null_buffers_and_sizes():
    refused(call([fake_spec()], sq=None), "NULL argument")
    refused(call([fake_spec()], partial=None), "NULL argument")
    refused(call([fake_spec()], L.RD_PS_ROWS, G=None), "NULL argument")
    refused(call([fake_spec()], plan=False), "NULL argument")
    refused(lib().rd_debug_per_sample_linear(None, 1, 4, 0, FAKE, 2, FAKE, 1 << 30, FAKE, 64, 1.0,
                                             (L.RdDebugPerSamplePlan * 1)(), None), "NULL argument")
    refused(call([fake_spec()], B=0), "bad sizes")
    refused(call([fake_spec()], nf=0), "bad sizes")
    refused(call([fake_spec()], L.RD_PS_ROWS, ldg=0), "bad sizes")


@pytest.mark.parametrize("R,nout,kin,form", [(10, 64, 64, -1), (300, 130, 62, 1), (300, 130, 62, 0), (1, 1, 1, -1)])
def test_refuses_an_undersized_partial(R, nout, kin, form):
    """16 bytes per CTA: 16 B (sum of the items' tiles per sample)"""
    specs = [fake_spec(R=R, out_features=nout, in_features=kin, ld_out=nout, ld_x=kin, form=form),
             fake_spec(form=form)]
    tiles = sum(dp_norm_tiles(s["R"], s["out_features"], s["in_features"],
                              dp_ghost(s["R"], s["out_features"], s["in_features"]) if form < 0 else form == 1)[2]
                for s in specs)
    need = 16 * 4 * tiles
    refused(call(specs, partial_bytes=need - 1), "partial buffer of %d bytes, it needs %d" % (need - 1, need))


# ---- GPU harness -----------------------------------------------------------------------------------------------------
GUARD = 32
F32_GUARD, F64_GUARD = 0x7FA5A5A5, 0x7FF4A5A5A5A5A5A5        # NaNs with payloads no kernel writes


def guarded(n, dtype):
    bits = F32_GUARD if dtype == torch.float32 else F64_GUARD
    itype = torch.int32 if dtype == torch.float32 else torch.int64
    buf = torch.full((n + 2 * GUARD,), bits, dtype=itype, device="cuda")
    return buf, buf[GUARD:GUARD + n].view(dtype)


def assert_guards(buf, n):
    bits = F32_GUARD if buf.dtype == torch.int32 else F64_GUARD
    assert (buf[:GUARD] == bits).all() and (buf[GUARD + n:] == bits).all(), "a write outside the output"


def same_bits(a, b):
    it = torch.int32 if a.dtype == torch.float32 else torch.int64
    return torch.equal(a.contiguous().view(it), b.contiguous().view(it))


class Item:
    """one linear item: logical operands Y [B, R, Nout], X [B, R, Kin (+1)] scattered into NaN-padded buffers in the
    encoder or ob-prop layout"""

    def __init__(self, B, R, nout, kin, family="random", seed=0, layout="enc", pad=0, rotated=False):
        self.B, self.R, self.nout, self.kin = B, R, nout, kin
        self.family, self.layout, self.rotated = family, layout, rotated
        kx = kin + 1 if rotated else kin
        self.Y, self.X = logical_operands(B, R, nout, kx, family, seed)
        self.ss, self.rs = LAYOUTS[layout](B, R)
        self.ld_out = nout + pad
        self.ld_x = (-(-(kin + 1) // 4) * 4 + pad) if rotated else kin + pad
        rows = sample_rows(B, R, self.ss, self.rs).reshape(-1)
        self.ybuf = torch.full((B * R, self.ld_out), float("nan"), device="cuda")
        self.xbuf = torch.full((B * R, self.ld_x), float("nan"), device="cuda")
        self.ybuf[rows, :nout] = self.Y.reshape(B * R, nout)
        self.xbuf[rows, :kx] = self.X.reshape(B * R, kx)
        self._ref = None

    def ref(self):
        if self._ref is None:
            self._ref = reference(self.Y.double(), self.X.double(), self.rotated)
        return self._ref

    def name(self):
        return "%s %s B%d R%d %dx%d" % (self.family, self.layout, self.B, self.R, self.nout, self.kin)

    def spec(self, **kw):
        s = dict(d_out=self.ybuf.data_ptr(), x=self.xbuf.data_ptr(), ld_out=self.ld_out, ld_x=self.ld_x,
                 sstride=self.ss, rstride=self.rs, R=self.R, out_features=self.nout, in_features=self.kin)
        s.update(kw)
        return s


def run_sqnorms(items, form=-1):
    """one sqnorms-mode call over the items (same B): returns w [B, n], b [B, n] (float64) and the plan.  Fields 2i, 2i
    + 1 of nf = 2n + 1; the last field and the guards must keep their NaN payload."""
    B, n = items[0].B, len(items)
    nf = 2 * n + 1
    forms = form if isinstance(form, (list, tuple)) else [form] * n
    specs = [it.spec(fw=2 * i, fb=2 * i + 1, form=f) for i, (it, f) in enumerate(zip(items, forms))]
    plans = (L.RdDebugPerSamplePlan * n)()
    tiles = 0
    for it, f in zip(items, forms):
        g = dp_ghost(it.R, it.nout, it.kin) if f < 0 else f == 1
        tiles += dp_norm_tiles(it.R, it.nout, it.kin, g)[2]
    partial = torch.full((2 * B * tiles,), float("nan"), dtype=torch.float64, device="cuda")
    buf, sq = guarded(B * nf, torch.float64)
    L.check(lib().rd_debug_per_sample_linear(items_array(specs), n, B, L.RD_PS_SQNORMS, sq.data_ptr(), nf,
                                             partial.data_ptr(), 8 * partial.numel(), None, 0, 1.0, plans,
                                             L.stream_ptr()), "rd_debug_per_sample_linear sqnorms")
    torch.cuda.synchronize()
    assert_guards(buf, B * nf)
    bits = buf[GUARD:GUARD + B * nf].view(B, nf)
    assert (bits[:, -1] == F64_GUARD).all(), "a write to an unused field"
    sq = sq.view(B, nf)
    for i, (it, f) in enumerate(zip(items, forms)):
        g = dp_ghost(it.R, it.nout, it.kin) if f < 0 else f == 1
        p = plans[i]
        assert (p.ghost, (p.tm, p.tn, p.ntiles)) == (int(g), dp_norm_tiles(it.R, it.nout, it.kin, g)), i
    return sq[:, 0:2 * n:2].clone(), sq[:, 1:2 * n:2].clone(), plans


def run_rows(items, rotated=False, scale=1.0):
    """one rows-mode call: each item's weight and bias fields at their own offsets with 1-3 floats of padding between
    fields; returns [B, Nout, Kin + 1] per item (float64).  Every column outside the fields keeps its NaN payload."""
    B, n = items[0].B, len(items)
    offs, cur = [], 3
    for i, it in enumerate(items):
        gw = cur
        cur += it.nout * it.kin + 1 + i % 3
        offs.append((gw, cur))
        cur += it.nout + 1 + (i + 1) % 3
    ldg = cur + 2
    specs = [it.spec(gw=gw, gb=gb) for it, (gw, gb) in zip(items, offs)]
    plans = (L.RdDebugPerSamplePlan * n)()
    buf, G = guarded(B * ldg, torch.float32)
    L.check(lib().rd_debug_per_sample_linear(items_array(specs), n, B, L.RD_PS_ROTATED if rotated else L.RD_PS_ROWS,
                                             None, 0, None, 0, G.data_ptr(), ldg, scale, plans, L.stream_ptr()),
            "rd_debug_per_sample_linear rows")
    torch.cuda.synchronize()
    assert_guards(buf, B * ldg)
    bits = buf[GUARD:GUARD + B * ldg].view(B, ldg)
    field = torch.zeros(ldg, dtype=torch.bool, device="cuda")
    G = G.view(B, ldg)
    outs = []
    for i, (it, (gw, gb)) in enumerate(zip(items, offs)):
        assert (plans[i].tn, plans[i].ntiles) == psg_tiles(it.nout, it.kin)[1:], i
        field[gw:gw + it.nout * it.kin] = True
        field[gb:gb + it.nout] = True
        outs.append(torch.cat([G[:, gw:gw + it.nout * it.kin].reshape(B, it.nout, it.kin), G[:, gb:gb + it.nout, None]],
                              2).double())
    assert (bits[:, ~field] == F32_GUARD).all(), "a write between fields"
    return outs


def check_norms(tag, it, w, b, ghost):
    r = it.ref()
    bad, ratio = norm_violations(w, b, r, ghost)
    key = ("ghost" if ghost else "explicit", it.family)
    record(key, ratio)
    neg = int((w < 0).sum() + (b < 0).sum())
    if ghost:
        n0, t0 = NEGATIVE.get(it.family, (0, 0))
        NEGATIVE[it.family] = (n0 + neg, t0 + 2 * w.numel())
    print("%-58s %-8s worst err/bound %.3g%s" % (tag + " " + it.name(), key[0], ratio,
                                                 "  (%d negative)" % neg if neg else ""))
    assert not bad.any(), (tag, it.name(), key, ratio)
    if not ghost:
        assert (w >= 0).all() and (b >= 0).all()


def check_rows(tag, it, out, scale):
    bad, ratio = rows_violations(out, it.ref(), scale)
    key = ("rotated" if it.rotated else "rows", it.family)
    record(key, ratio)
    print("%-58s %-8s worst err/bound %.3g" % (tag + " " + it.name(), key[0], ratio))
    assert not bad.any(), (tag, it.name(), key, ratio, int(bad.sum()))


def print_worst():
    for k in sorted(WORST):
        print("WORST %-10s %-10s %.4g" % (k[0], k[1], WORST[k]))
    for f, (n, t) in sorted(NEGATIVE.items()):
        print("NEGATIVE ghost norms %-8s %d of %d" % (f, n, t))


def all_modes(items, tag, scale=-3.0):
    """both forced forms and the shape's own choice (bitwise that form), rows; the rotated twins in rotated mode"""
    plain = [it for it in items if not it.rotated]
    rot = [it for it in items if it.rotated]
    if plain:
        res = {f: run_sqnorms(plain, f) for f in (0, 1, -1)}
        for i, it in enumerate(plain):
            g = dp_ghost(it.R, it.nout, it.kin)
            for f in (0, 1):
                check_norms(tag, it, res[f][0][:, i], res[f][1][:, i], f == 1)
            chosen = res[1 if g else 0]
            assert same_bits(res[-1][0][:, i], chosen[0][:, i]) and same_bits(res[-1][1][:, i], chosen[1][:, i]), \
                (tag, it.name(), "auto differs from the form it picks")
        for it, out in zip(plain, run_rows(plain, False, scale)):
            check_rows(tag, it, out, scale)
    if rot:
        for it, out in zip(rot, run_rows(rot, True, scale)):
            check_rows(tag, it, out, scale)


# ---- GPU: tails, layouts and padding ---------------------------------------------------------------------------------
TAIL_R = [1, 15, 16, 17, 63, 64, 65, 128, 129, 257]
TAIL_NOUT = [1, 63, 64, 65, 130]
TAIL_KIN = [1, 62, 63, 64, 65, 127]


def tail_shapes():
    """a covering set: every R with three (Nout, Kin) pairs, every Nout and Kin with many R"""
    return [(R, TAIL_NOUT[(i + s) % 5], TAIL_KIN[(i + 2 * s) % 6]) for s in range(3) for i, R in enumerate(TAIL_R)]


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 3, 33])
def test_tails(B):
    shapes = tail_shapes()
    items = [Item(B, R, nout, kin, "random", seed=R * 7 + nout + kin, layout=("enc", "ob")[k % 2], pad=k % 3 * 2)
             for k, (R, nout, kin) in enumerate(shapes)]
    assert any(dp_norm_tiles(it.R, it.nout, it.kin, True)[0] == 5 for it in items)
    all_modes(items, "tails")
    rot = [Item(B, R, nout, kin, "random", seed=R + nout, layout=("ob", "enc")[k % 2], rotated=True)
           for k, (R, nout, kin) in enumerate(shapes)]
    all_modes(rot, "tails")
    print_worst()


@pytest.mark.gpu
@pytest.mark.parametrize("family", FAMILIES)
def test_operand_families(family):
    shapes = [(3, 65, 65, 64), (33, 17, 130, 63), (1, 129, 64, 127), (3, 257, 63, 1), (33, 64, 1, 62)]
    for k, (B, R, nout, kin) in enumerate(shapes):
        items = [Item(B, R, nout, kin, family, seed=11 * k + 1, layout=lay, pad=p)
                 for lay, p in (("enc", 3), ("ob", 0))]
        items += [Item(B, R, nout, kin, family, seed=11 * k + 2, layout="ob", rotated=True)]
        all_modes(items, "family")
    print_worst()


# ---- GPU: the result depends on the shapes alone ---------------------------------------------------------------
def mixed_items(B, seed=0):
    shapes = tail_shapes()
    out = []
    for k in range(MAX_ITEMS):
        R, nout, kin = shapes[(k * 7) % len(shapes)]
        out.append(Item(B, R, nout, kin, FAMILIES[k % 5], seed=seed + k, layout=("enc", "ob")[k % 2], pad=k % 4))
    return out


@pytest.mark.gpu
def test_bits_alone_and_anywhere_in_a_group():
    """the same bits alone, at any position of a 32-item group of mixed shapes (the blk0 item lookup), and across runs;
    sqnorms in every form, rows"""
    B = 3
    items = mixed_items(B)
    forms = [(-1, 0, 1)[k % 3] for k in range(MAX_ITEMS)]
    w, b, _ = run_sqnorms(items, forms)
    w2, b2, _ = run_sqnorms(items, forms)
    assert same_bits(w, w2) and same_bits(b, b2), "two runs differ"
    order = list(reversed(range(MAX_ITEMS)))
    wr, br, _ = run_sqnorms([items[i] for i in order], [forms[i] for i in order])
    rows = run_rows(items, False, 0.75)
    rows_r = run_rows([items[i] for i in order], False, 0.75)
    for k in range(MAX_ITEMS):
        it = items[k]
        g = dp_ghost(it.R, it.nout, it.kin) if forms[k] < 0 else forms[k] == 1
        check_norms("group", it, w[:, k], b[:, k], g)
        wa, ba, _ = run_sqnorms([it], forms[k])
        j = order.index(k)
        assert same_bits(wa[:, 0], w[:, k]) and same_bits(ba[:, 0], b[:, k]), (k, "alone vs group")
        assert same_bits(wr[:, j], w[:, k]) and same_bits(br[:, j], b[:, k]), (k, "position")
        ra = run_rows([it], False, 0.75)[0]
        assert same_bits(ra.float(), rows[k].float()) and same_bits(rows_r[j].float(), rows[k].float()), (k, "rows")
        check_rows("group", it, rows[k], 0.75)
    print_worst()


@pytest.mark.gpu
def test_rotated_bits_alone_and_in_a_group():
    B = 33
    shapes = tail_shapes()
    items = [Item(B, *shapes[(k * 5) % len(shapes)], FAMILIES[k % 6], seed=k, layout=("ob", "enc")[k % 2], rotated=True)
             for k in range(12)]
    rows = run_rows(items, True, -1.25)
    for k, it in enumerate(items):
        assert same_bits(run_rows([it], True, -1.25)[0].float(), rows[k].float()), k
        check_rows("rotated group", it, rows[k], -1.25)


# ---- GPU: the TracIn dot ---------------------------------------------------------------------------------------
FAR = 1e30


def dot_operands(Bq, Bt, ldg, segs, family, seed):
    """Gq [Bq, ldg], Gt [Bt, ldg] with +-1e30 in every column outside the segments"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device="cuda")
    Gq, Gt = rn(Bq, ldg), rn(Bt, ldg)
    if family == "scaled":
        e = lambda *s: torch.exp2(torch.randint(-10, 11, s, generator=g, device="cuda").float())
        Gq, Gt = Gq * e(Bq, 1) * e(1, ldg), Gt * e(Bt, 1) * e(1, ldg)
    elif family == "same-sign":
        Gq, Gt = Gq.abs(), Gt.abs()
    elif family == "tf32":
        Gq = tf32_rn(Gq)
    inside = torch.zeros(ldg, dtype=torch.bool, device="cuda")
    for off, ln in segs:
        inside[off:off + ln] = True
    sign = lambda *s: torch.where(torch.rand(*s, generator=g, device="cuda") < 0.5, -FAR, FAR)
    Gq[:, ~inside] = sign(Bq, int((~inside).sum()))
    Gt[:, ~inside] = sign(Bt, int((~inside).sum()))
    return Gq.contiguous(), Gt.contiguous()


def run_dot(Gq, Gt, segs, alpha, scores):
    """scores [Bq, lds] float64 (the first Bt columns live)"""
    Bq, Bt, ldg = Gq.shape[0], Gt.shape[0], Gq.shape[1]
    n = len(segs)
    offs = (C.c_int64 * n)(*[o for o, _ in segs])
    lens = (C.c_int64 * n)(*[ln for _, ln in segs])
    nb = lib().rd_per_sample_grad_dot_scratch_bytes(Bq, Bt, ldg, n)
    sc = torch.full(((nb + 3) // 4,), float("nan"), device="cuda")
    L.check(lib().rd_per_sample_grad_dot(Gq.data_ptr(), Bq, Gt.data_ptr(), Bt, ldg, offs, lens, n, alpha,
                                         scores.data_ptr(), scores.shape[1], sc.data_ptr(), L.stream_ptr()),
            "rd_per_sample_grad_dot")
    torch.cuda.synchronize()


def dot_reference(Gq, Gt, segs, alpha, s0):
    q, t = Gq.double(), Gt.double()
    P, bound = s0.clone(), f64(4) * s0.abs()
    for off, ln in segs:
        sl = slice(off, off + ln)
        Ss = q[:, sl].abs() @ t[:, sl].abs().T
        P += alpha * (q[:, sl] @ t[:, sl].T)
        bound += abs(alpha) * (dot_coef(ln) * U + f64(ln + len(segs) + 4)) * Ss
    return P, bound


def check_dot(tag, family, Gq, Gt, segs, alpha=-0.7, lds_pad=3):
    """+= onto nonzero scores with NaN canaries between Bt and lds; returns the scores"""
    Bq, Bt = Gq.shape[0], Gt.shape[0]
    lds = Bt + lds_pad
    g = torch.Generator(device="cuda").manual_seed(Bq * 1000 + Bt)
    s0 = torch.randn(Bq, Bt, generator=g, device="cuda", dtype=torch.float64)
    buf, flat = guarded(Bq * lds, torch.float64)
    scores = flat.view(Bq, lds)
    scores[:, :Bt] = s0
    run_dot(Gq, Gt, segs, alpha, scores)
    assert_guards(buf, Bq * lds)
    gap = buf[GUARD:GUARD + Bq * lds].view(Bq, lds)[:, Bt:]
    assert (gap == F64_GUARD).all(), (tag, "a write between Bt and lds")
    out = scores[:, :Bt]
    P, bound = dot_reference(Gq, Gt, segs, alpha, s0)
    err = (out - P).abs()
    ratio = ratio_of(err, bound - f64(4) * s0.abs())
    record(("dot", family), ratio)
    print("%-58s worst err/bound %.3g" % ("dot %s %s Bq %d Bt %d" % (tag, family, Bq, Bt), ratio))
    assert (err <= bound).all(), (tag, family, Bq, Bt, ratio)
    return out.clone()


def layout_segments(lengths, gaps, tail):
    """segments of the given lengths at 4-aligned offsets, `gaps[i]` extra columns after segment i; the row ends
    `tail` columns after the last segment (ldg % 4 == 0)"""
    segs, cur = [], 0
    for ln, gp in zip(lengths, gaps):
        segs.append((cur, ln))
        cur = -(-(cur + ln) // 4) * 4 + gp
    return segs, -(-(cur - gaps[-1]) // 4) * 4 + tail


SEG_LENGTHS = [1, 4, 31, 32, 33, 64, 96, 4095, 4096, 44]
DOT_SIZES = [(q, t) for q in (1, 63, 64, 65, 130) for t in (1, 63, 64, 65, 128, 129, 300)]


@pytest.mark.gpu
def test_dot_sizes():
    """partial query and train tiles, an idle second warpgroup (Bt <= 64), over short segments"""
    segs, ldg = layout_segments([33, 64, 4, 1, 96], [0, 0, 8, 4, 0], 0)
    assert ldg % 32 != 0
    for k, (Bq, Bt) in enumerate(DOT_SIZES):
        fam = ("random", "scaled", "same-sign", "tf32")[k % 4]
        check_dot("sizes", fam, *dot_operands(Bq, Bt, ldg, segs, fam, seed=k), segs)
    print_worst()


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["random", "scaled", "same-sign", "tf32"])
def test_dot_segments(family):
    """1, 2 and 3+ k-blocks and both parities of the final fold; segments that are adjacent (a k-block runs into the
    next segment); gaps of +-1e30; the last segment ending at an ldg that is not a multiple of 32"""
    segs, ldg = layout_segments(SEG_LENGTHS, [0, 0, 12, 0, 0, 0, 0, 4, 0, 0], 0)
    assert ldg % 32 != 0 and segs[-1][0] + segs[-1][1] == ldg
    assert any(a[0] + a[1] == b[0] and a[1] % 32 for a, b in zip(segs, segs[1:]))     # a k-block into the next
    for Bq, Bt in [(65, 129), (1, 300), (130, 64)]:
        check_dot("segments", family, *dot_operands(Bq, Bt, ldg, segs, family, seed=Bq + Bt), segs)
    print_worst()


@pytest.mark.gpu
def test_dot_far_columns_move_no_score():
    """the same scores bit for bit with the columns outside every segment at +-1e30 or at 0"""
    segs, ldg = layout_segments([33, 4095, 1, 36], [4, 8, 0, 0], 0)
    Gq, Gt = dot_operands(65, 129, ldg, segs, "random", seed=5)
    a = check_dot("far", "random", Gq, Gt, segs)
    inside = torch.zeros(ldg, dtype=torch.bool, device="cuda")
    for off, ln in segs:
        inside[off:off + ln] = True
    Gq0, Gt0 = Gq.clone(), Gt.clone()
    Gq0[:, ~inside], Gt0[:, ~inside] = 0.0, 0.0
    assert same_bits(a, check_dot("far zeroed", "random", Gq0, Gt0, segs))


@pytest.mark.gpu
def test_dot_bits_across_blocks_and_permutations():
    """each score is the same bits computed in any query / train sub-block (rows starting mid-tile, single rows) and
    with the rows of both operands permuted"""
    segs, ldg = layout_segments([4096, 33, 64, 1], [0, 3 * 4, 0, 0], 4)
    Bq, Bt = 130, 300
    Gq, Gt = dot_operands(Bq, Bt, ldg, segs, "random", seed=9)
    check_dot("blocks", "random", Gq, Gt, segs)
    whole = torch.zeros(Bq, Bt, dtype=torch.float64, device="cuda")
    run_dot(Gq, Gt, segs, 1.0, whole)
    for q0, q1, t0, t1 in [(0, 64, 0, 128), (1, 66, 7, 300), (129, 130, 299, 300), (63, 130, 128, 257)]:
        sub = torch.zeros(q1 - q0, t1 - t0, dtype=torch.float64, device="cuda")
        run_dot(Gq[q0:q1], Gt[t0:t1], segs, 1.0, sub)
        assert same_bits(sub, whole[q0:q1, t0:t1]), (q0, q1, t0, t1)
    g = torch.Generator(device="cuda").manual_seed(0)
    pq, pt = torch.randperm(Bq, generator=g, device="cuda"), torch.randperm(Bt, generator=g, device="cuda")
    perm = torch.zeros(Bq, Bt, dtype=torch.float64, device="cuda")
    run_dot(Gq[pq].contiguous(), Gt[pt].contiguous(), segs, 1.0, perm)
    assert same_bits(perm, whole[pq][:, pt])
