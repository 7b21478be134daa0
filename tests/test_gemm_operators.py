"""The forward GEMM engines on their own, element by element against float64.

tc_nt_kernel (rd_tc_gemm.cu, wgmma) runs the encoder projections and their input gradients in error-compensated
3xTF32 and the ob-prop layers in single-pass TF32 or 3xTF32; gemm_f32_kernel (rd_gemm.cu, CUDA cores) runs attention's
batched products, the head, the fallback shapes and the split-K weight gradients.  Both are called here through the
debug entries rd_debug_tc_nt / rd_debug_gemm_f32, which take a forced tile plan or split count per call.  Every output
element is compared with the float64 product P = A.B^T (or A.B) followed by the epilogue restated in float64 in the
kernel's order, against a COMPONENTWISE bound in units of u = 2^-24 times S = |A|.|B|^T.  A normwise tolerance
(max|d| / max|ref|) cannot see a wrong small-magnitude slice; these bounds can.

Bounds (derived, not fitted).  Write x = hi + lo with hi = trunc19(x), the top 19 bits (sign, exponent and 10 mantissa
bits: TF32), lo = x - hi exact in fp32 and |lo| < 2^-10 |x|.  The tensor core multiplies TF32 operands exactly (11 x 11
significand bits fit in fp32) and reads an fp32 operand as its top 19 bits.

  3xTF32 (B_lo != NULL).  Per k8 step the kernel issues lo.hi, hi.lo, hi.hi (A split in registers, B_lo precomputed).
  * Operands: the product is approximated by Ah.Bh + trunc19(Al).Bh + Ah.trunc19(Bl).  Dropped: Al.Bl, below
    2^-20 |a||b| = 16u |a||b|; and the reads of the remainders, |Al - trunc19(Al)| < 2^-10 |Al| < 2^-20 |a|, so each of
    the two costs below 16u |a||b|.  Summed over k: below 48u S.
  * Accumulation: each wgmma k8 step adds 8 exact products to the fp32 accumulator with one truncating (round toward
    zero) normalisation whose error is below one unit in the last place of the running magnitude, i.e. below 2u S.
    Three steps per k8: below 6 ceil(K/8) u S.
  => |C - P| <= (6 ceil(K/8) + 48) u S.
  Single pass (B_lo == NULL) on operands the test has RN-rounded to TF32: products exact, one truncating accumulation per
  k8 step, plus 4u S for the first step's alignment of the 8 products and the final conversion:
  => |C - P| <= (2 ceil(K/8) + 4) u S.
  gemm_f32: a chain of K fmaf (each a single rounding below u of the running magnitude, bounded by S), nsplit - 1
  additions of the split partials (below u S each), alpha and the store: |C - P| <= (K + nsplit + 2) u S.

The epilogue (bias, scale, gate, dropout, resid) is restated in float64: each fp32 operation adds at most u of its
result's magnitude, multiplications scale the product's bound, ReLU is non-expansive (so a pre-activation within the bound
of zero may go either way and still lies inside it) and the TF32 rounding of round_out adds 2^-11 of |out|.  Every
other disagreement fails, NaN included.  The worst err / (u S) of each case (product bound only) is printed.

CPU: a numpy emulation of the 3xTF32 arithmetic stays inside its bound and, with one lo.hi term dropped, breaks it; the
host refusals of the debug entries (split-K with an epilogue, uninstantiated epilogues and widths, K / N / lda not
multiples of 4, unaligned pointers).  GPU: every instantiated (epilogue, mode), every width, over-wide plans, M = 1,
K < 32, K = N = 2400, positive and random operands, unaligned bases (bitwise against aligned copies), keep bits bit for
bit, the permuted store, NaN canaries around C; gemm_f32 in all four operand layouts, batched, with transposed C, every
epilogue field and split-K; split_weights bitwise and colsum within its bound.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle.dropout_masks import dropout_mask_at
from raindrop_b200 import lib as L

U = 2.0 ** -24
F_RELU, F_SCALE, F_GATE, F_DROP, F_RESID, F_ROUND, F_PERM, F_REP = 1, 2, 4, 8, 16, 32, 64, 128
# the (flags, exact) combinations tc_nt instantiates (RD_NT_CASE in rd_tc_gemm.cu)
NT_CASES = [(F_PERM | F_RELU | F_SCALE, False), (F_RELU | F_SCALE | F_ROUND, False), (F_RELU | F_SCALE, False),
            (F_GATE | F_SCALE, False), (F_PERM | F_RELU | F_SCALE, True), (F_RELU | F_SCALE, True),
            (F_GATE | F_SCALE, True), (0, True), (F_RESID, True), (F_DROP, True), (F_DROP | F_RESID, True),
            (F_GATE, True), (F_RELU, True), (F_RELU | F_DROP, True), (F_DROP | F_RESID | F_REP, True),
            (F_RELU | F_DROP | F_REP, True)]
EXACT_WIDTHS = [48, 80, 96, 120, 136, 152, 184, 232]
FAST_WIDTHS = [64, 96, 128, 160, 192, 224, 240, 256]
SEED, STEP = 0x1234_5678_9ABC, 77
WORST = {}


def lib():
    return L.load()


def tc_bound(K, exact):
    return (6 * math.ceil(K / 8) + 48) if exact else (2 * math.ceil(K / 8) + 4)


# ---- numpy formulas of the operand splits ------------------------------------------------------------------------
def trunc19(a):
    return (np.ascontiguousarray(a, dtype=np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def tf32_rna(a):
    """cvt.rna.tf32.f32: round the low 13 mantissa bits to nearest, ties away from zero."""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def f32_toward_zero(x):
    f = x.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(x)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f


def emulate_3xtf32(A, B, skip_lo_hi_step=None):
    """tc_nt's error-compensated arithmetic: per k8 step lo.hi, hi.lo, hi.hi, each summed exactly and added to the fp32
    accumulator with truncation; remainders read as their top 19 bits.  skip_lo_hi_step drops one step's lo.hi."""
    Ah, Bh = trunc19(A), trunc19(B)
    Al, Bl = trunc19(A - Ah), trunc19(B - Bh)
    acc = np.zeros((A.shape[0], B.shape[0]), np.float32)
    for s, k0 in enumerate(range(0, A.shape[1], 8)):
        ks = slice(k0, k0 + 8)
        for term, (a, b) in enumerate(((Al, Bh), (Ah, Bl), (Ah, Bh))):
            if term == 0 and s == skip_lo_hi_step:
                continue
            acc = f32_toward_zero(acc.astype(np.float64) + a[:, ks].astype(np.float64) @ b[:, ks].astype(np.float64).T)
    return acc


@pytest.mark.parametrize("positive", [True, False])
def test_3xtf32_bound_holds_and_discriminates(positive):
    rng = np.random.default_rng(5 + positive)
    M, N, K = 24, 20, 40
    draw = (lambda *s: rng.random(s)) if positive else (lambda *s: rng.standard_normal(s))
    A, B = draw(M, K).astype(np.float32), draw(N, K).astype(np.float32)
    P = A.astype(np.float64) @ B.astype(np.float64).T
    S = np.abs(A.astype(np.float64)) @ np.abs(B.astype(np.float64)).T
    bound = tc_bound(K, True) * U * S
    ok = np.abs(emulate_3xtf32(A, B) - P)
    assert (ok <= bound).all(), (ok / (U * S)).max()
    for step in (0, K // 8 - 1):        # the first and the last (tail) k-step
        bad = np.abs(emulate_3xtf32(A, B, skip_lo_hi_step=step) - P)
        assert (bad > bound).any(), (step, (bad / (U * S)).max())


# ---- the debug entries ---------------------------------------------------------------------------------------------
def nt_args(**kw):
    a = L.RdDebugTcNtArgs()
    a.scale_mod, a.gate_scale = 1, 1.0
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def gemm_args(**kw):
    a = L.RdDebugGemmArgs()
    a.nz, a.nz_inner, a.nsplit, a.alpha, a.rowscale_mod, a.gate_scale, a.sCj = 1, 1, 1, 1.0, 1, 1.0, 1
    for k, v in kw.items():
        setattr(a, k, v)
    return a


FAKE = 1 << 20      # a 16-byte aligned address the host checks see but never dereference


def refused(rc, what):
    assert rc == -2, rc
    msg = lib().rd_last_error_string().decode()
    assert what in msg, msg


@pytest.mark.parametrize("field,value", [("bias", FAKE), ("relu", 1), ("rowscale", FAKE), ("gate", FAKE),
                                         ("drop_p", 0.5), ("resid", FAKE), ("perm", 1)])
def test_gemm_split_k_refuses_epilogue(field, value):
    a = gemm_args(A=FAKE, B=FAKE, C=FAKE, M=64, N=64, K=4096, tb=1, sAi=4096, sBj=4096, sCi=64, nsplit=4,
                  rng=FAKE, rowscale_mod=1, pB=1, pN=64, pdob=1, pD=64)
    setattr(a, field, value)
    refused(lib().rd_debug_gemm_f32(C.byref(a), C.c_void_p(FAKE), None), "split-K")


@pytest.mark.parametrize("sCi,sCj", [(65, 1), (1, 64)])
def test_gemm_split_k_refuses_strided_c(sCi, sCj):
    a = gemm_args(A=FAKE, B=FAKE, C=FAKE, M=64, N=64, K=4096, tb=1, sAi=4096, sBj=4096, sCi=sCi, sCj=sCj, nsplit=4)
    refused(lib().rd_debug_gemm_f32(C.byref(a), C.c_void_p(FAKE), None), "contiguously")


def test_gemm_split_k_plan_is_written_back():
    a = gemm_args(A=FAKE, B=FAKE, C=FAKE, M=64, N=64, K=4096, tb=1, sAi=4096, sBj=4096, sCi=64, nsplit=0, bias=FAKE)
    refused(lib().rd_debug_gemm_f32(C.byref(a), None, None), "partial buffer")
    assert a.nsplit == 64 and a.partial_floats == 64 * (64 * 64 + 64), (a.nsplit, a.partial_floats)
    refused(lib().rd_debug_gemm_f32(C.byref(a), C.c_void_p(FAKE), None), "split-K applies alpha only")


def nt_plain(**kw):
    base = dict(A=FAKE, B=FAKE, B_lo=FAKE, C=FAKE, lda=64, M=256, N=64, K=64, BN=80, n_tiles=1)
    base.update(kw)
    return nt_args(**base)


@pytest.mark.parametrize("kw,what", [
    (dict(relu=1, gate=FAKE, gate_ld=64), "not instantiated"),                    # relu + gate: no such epilogue
    (dict(B_lo=0, BN=64, resid=FAKE, resid_ld=64), "not instantiated"),                  # single pass + residual
    (dict(B_lo=0, BN=80), "unsupported tiling"),                                  # an exact-mode width, single pass
    (dict(BN=64), "unsupported tiling"),                                          # a single-pass width, exact mode
    (dict(BN=48, n_tiles=1), "unsupported tiling"),                               # BN * n_tiles < N
    (dict(K=62, lda=64), "unsupported tiling"),
    (dict(N=66, BN=80), "unsupported tiling"),
    (dict(lda=66), "unsupported tiling"),
    (dict(A=FAKE + 4), "16-byte aligned"), (dict(B=FAKE + 8), "16-byte aligned"), (dict(B_lo=FAKE + 12), "16-byte aligned"),
    (dict(C=FAKE + 4), "16-byte aligned"), (dict(gate=FAKE + 8, gate_ld=64), "16-byte aligned"),
    (dict(resid=FAKE + 4, resid_ld=64), "16-byte aligned"),
    (dict(resid=FAKE, resid_ld=63), "bad epilogue"), (dict(drop_p=0.5), "bad epilogue"),
    (dict(drop_p=0.5, rng=FAKE, drop_mask=FAKE, drop_mask_ld=1), "bad epilogue"),
])
def test_tc_nt_refusals(kw, what):
    refused(lib().rd_debug_tc_nt(C.byref(nt_plain(**kw)), None), what)


# ---- GPU harness ---------------------------------------------------------------------------------------------------
CANARY = 64          # NaN floats before and after C


def dev(x):
    return torch.as_tensor(x).cuda()


def at_offset(t, byte_off):
    """A copy of t whose data starts byte_off bytes past a 128-byte boundary (torch's blocks are 512-byte aligned)."""
    n = t.numel() + 64
    buf = torch.empty(n, dtype=t.dtype, device=t.device)
    assert buf.data_ptr() % 128 == 0
    v = buf[byte_off // 4: byte_off // 4 + t.numel()].view(t.shape)
    v.copy_(t)
    return v


def canaried(n):
    buf = torch.full((n + 2 * CANARY,), float("nan"), device="cuda")
    return buf, buf[CANARY:CANARY + n]


def assert_canaries(buf):
    assert torch.isnan(buf[:CANARY]).all() and torch.isnan(buf[-CANARY:]).all(), "a write outside C"


def rng_tensor():
    return torch.tensor([SEED, STEP], dtype=torch.int64, device="cuda")


def drop_scale(rows, N, p, site, rep=None):
    """float64 [rows, N]: the kernels' keep scale of element (row, col), index row*N + col or through rep_remap."""
    r = np.arange(rows, dtype=np.int64)[:, None]
    c = np.arange(N, dtype=np.int64)[None, :]
    if not rep:
        return dropout_mask_at(SEED, STEP, site, (r * N + c).astype(np.uint64), p).astype(np.float64)
    B, Bc = rep
    t, j = r // Bc, r % Bc
    m, b = j // B, j % B
    out = np.empty((rows, N), np.float64)
    for mm in np.unique(m):
        sel = (m == mm)[:, 0]
        idx = ((t[sel] * B + b[sel]) * N + c).astype(np.uint64)
        out[sel] = dropout_mask_at(SEED, STEP + int(mm), site, idx, p)
    return out


class Epi:
    """The epilogue in float64, in the kernels' order, with a running bound of the fp32 rounding it adds (ep) and the
    factor the product's error is multiplied by (mult)."""

    def __init__(self, P):
        self.v = P.clone()
        self.ep = torch.zeros_like(P)
        self.mult = torch.ones_like(P)

    def _round(self):
        self.ep = self.ep + U * self.v.abs()

    def mul(self, f):
        self.v = self.v * f
        self.ep = self.ep * f.abs()
        self.mult = self.mult * f.abs()
        self._round()

    def add(self, a):
        self.v = self.v + a
        self._round()

    def relu(self):
        self.v = self.v.clamp_min(0.0)


def check(name, out, epi, S, coef, round_out=False):
    """|out - ref| <= coef u S mult + ep (+ 2^-11 |ref| with round_out), NaN failing; records err / (u S mult)."""
    out = out.double()
    err = (out - epi.v).abs()
    tol = coef * U * S * epi.mult + epi.ep + (2.0 ** -11 * epi.v.abs() if round_out else 0.0)
    bad = ~(err <= tol)
    scale = U * S * epi.mult
    live = scale > 0
    ratio = float((err[live] / scale[live]).max()) if live.any() else 0.0
    WORST[name] = max(WORST.get(name, 0.0), ratio)
    print("%-58s worst err/(u S) %8.2f   bound %d%s" % (name, ratio, coef, "  (+ TF32 rounding)" if round_out else ""))
    assert not bad.any(), (name, int(bad.sum()), float(err[bad].max()), ratio, coef)


def lo_of(B):
    return B - (B.view(torch.int32) & -8192).view(torch.float32)


def run_tc_nt(A, B, K, exact, flags=0, bias=None, BN=0, n_tiles=0, *, lda=None, scale_mod=7, gate_scale=1.5, p=0.25,
              site=33, rep=None, perm=None, gen=None, gate=None, resid=None, scale=None, name=""):
    """One rd_debug_tc_nt call: A [M, lda] (first K columns used), B [N, K] (device fp32).  Returns (out, epi, S, coef,
    extras) with out [M, N] in (row, col) order (the permuted store unpermuted) and the canaries checked."""
    M, N = A.shape[0], B.shape[0]
    lda = A.stride(0)
    Bl = lo_of(B) if exact else None
    if gen is None:
        gen = torch.Generator(device="cuda").manual_seed(M * 7 + N)
    if flags & F_SCALE and scale is None:
        scale = 0.5 + torch.rand(scale_mod, device="cuda", generator=gen)
    if flags & F_GATE and gate is None:
        gate = torch.randn(M, N, device="cuda", generator=gen)
    if flags & F_RESID and resid is None:
        resid = torch.randn(M, N + 4, device="cuda", generator=gen)[:, :N]      # resid_ld = N + 4
    rng = rng_tensor() if flags & F_DROP else None
    words = (N + 31) // 32
    mask = torch.full((M, words + 1), -1, dtype=torch.int32, device="cuda") if flags & F_DROP else None
    if flags & F_PERM:
        pB, pN = perm
        pD = 4 * pN + 16
        cbuf, cview = canaried((N // 4) * pB * pD)
    else:
        cbuf, cview = canaried(M * N)
    a = nt_args(A=A.data_ptr(), lda=lda, B=B.data_ptr(), B_lo=L.ptr(Bl), M=M, N=N, K=K, BN=BN, n_tiles=n_tiles,
                C=cview.data_ptr(), bias=L.ptr(bias), relu=int(bool(flags & F_RELU)), scale=L.ptr(scale),
                scale_mod=scale_mod, gate=L.ptr(gate), gate_ld=N, gate_scale=gate_scale,
                drop_p=p if flags & F_DROP else 0.0, rng=L.ptr(rng), drop_site=site,
                rep_B=rep[0] if flags & F_REP else 0, rep_Bc=rep[1] if flags & F_REP else 0,
                drop_mask=L.ptr(mask), drop_mask_ld=words + 1 if mask is not None else 0,
                resid=L.ptr(resid), resid_ld=resid.stride(0) if resid is not None else 0,
                round_out=int(bool(flags & F_ROUND)), perm=int(bool(flags & F_PERM)))
    if flags & F_PERM:
        a.pB, a.pN, a.pD = pB, pN, pD
    L.check(lib().rd_debug_tc_nt(C.byref(a), L.stream_ptr()), "rd_debug_tc_nt " + name)
    torch.cuda.synchronize()
    assert_canaries(cbuf)
    if flags & F_PERM:
        img = cview.view(N // 4, pB, pD)
        assert torch.isnan(img[:, :, 4 * pN:]).all(), "the permuted store wrote past n*4 + 3"
        out = img[:, :, :4 * pN].reshape(N // 4, pB, pN, 4).permute(1, 2, 0, 3).reshape(M, N)
    else:
        out = cview.view(M, N)
    Ad, Bd = A[:, :K].double(), B.double()
    epi = Epi(Ad @ Bd.T)
    S = Ad.abs() @ Bd.abs().T
    if bias is not None:
        epi.add(bias.double()[None, :])
    if flags & F_RELU:
        epi.relu()
    if flags & F_SCALE:
        epi.mul(scale.double()[torch.arange(M, device="cuda") % scale_mod][:, None].expand(M, N))
    if flags & F_GATE:
        epi.mul(torch.where(gate > 0, gate_scale, 0.0).double())
    keep = None
    if flags & F_DROP:
        keep = dev(drop_scale(M, N, p, site, rep if flags & F_REP else None))
        epi.mul(keep)
    if flags & F_RESID:
        epi.add(resid.double())
    if flags & F_ROUND:
        o = out.cpu().numpy()
        assert (o.view(np.uint32) & 0x1FFF == 0).all(), "round_out left bits below TF32"
    check(name, out, epi, S, tc_bound(K, exact), round_out=bool(flags & F_ROUND))
    if mask is not None:
        check_keep_bits(mask, keep, M, N)
    return out


def check_keep_bits(mask, keep, M, N):
    """Words 0 .. ceil(N/32)-1 of every row hold bit col % 32 of the keep decision, zeros past N; the ld padding word
    keeps its canary."""
    words = (N + 31) // 32
    bits = np.zeros((M, 32 * words), np.uint64)
    bits[:, :N] = (keep.cpu().numpy() > 0)
    w = (bits.reshape(M, words, 32) << np.arange(32, dtype=np.uint64)).sum(-1).astype(np.uint32)
    want = np.full((M, words + 1), 0xFFFFFFFF, np.uint32)
    want[:, :words] = w
    got = mask.cpu().numpy().view(np.uint32)
    assert (got == want).all(), ("keep bits", int((got != want).sum()), np.argwhere(got != want)[:4])


def operands(M, N, K, lda, positive, exact, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if positive:
        A = torch.rand(M, lda, device="cuda", generator=g)
        B = torch.rand(N, K, device="cuda", generator=g)
    else:
        A = torch.randn(M, lda, device="cuda", generator=g)
        B = torch.randn(N, K, device="cuda", generator=g)
    if not exact:     # single pass reads TF32-representable operands
        A = dev(tf32_rna(A.cpu().numpy()))
        B = dev(tf32_rna(B.cpu().numpy()))
    A[:, K:] = float("nan")       # the lda padding is never read
    return A, B


def flag_name(flags):
    names = ["relu", "scale", "gate", "drop", "resid", "round", "perm", "rep"]
    return "|".join(n for i, n in enumerate(names) if flags >> i & 1) or "plain"


@pytest.mark.gpu
@pytest.mark.parametrize("flags,exact", NT_CASES, ids=["%s-%s" % (flag_name(f), "exact" if e else "fast") for f, e in NT_CASES])
@pytest.mark.parametrize("with_bias", [False, True])
def test_tc_nt_every_epilogue_at_tail_shape(flags, exact, with_bias):
    M, N, K = 129, 236, 36
    A, B = operands(M, N, K, K + 4, False, exact, seed=flags * 2 + exact)
    bias = torch.randn(N, device="cuda") if with_bias else None
    run_tc_nt(A, B, K, exact, flags, bias, perm=(3, 43), rep=(43, 129),
              name="tc_nt %s %s%s M129 N236 K36" % (flag_name(flags), "exact" if exact else "fast",
                                                   " +bias" if with_bias else ""))


@pytest.mark.gpu
@pytest.mark.parametrize("exact,bn", [(True, w) for w in EXACT_WIDTHS] + [(False, w) for w in FAST_WIDTHS])
def test_tc_nt_every_width(exact, bn):
    M, K = 4318, 64
    N = 2 * bn + 4
    A, B = operands(M, N, K, K, bn % 3 == 0, exact, seed=bn)
    # single pass has no plain-product epilogue: relu + scale (the ob-prop layer's)
    run_tc_nt(A, B, K, exact, 0 if exact else F_RELU | F_SCALE, None, BN=bn, n_tiles=-(-N // bn),
              name="tc_nt width %d %s M4318 N%d" % (bn, "exact" if exact else "fast", N))


@pytest.mark.gpu
@pytest.mark.parametrize("exact,bn,N,n_tiles", [(True, 48, 100, 5), (True, 232, 236, 3), (False, 64, 132, 6)])
def test_tc_nt_overwide_plan(exact, bn, N, n_tiles):
    M, K = 300, 40
    A, B = operands(M, N, K, K, False, exact, seed=n_tiles)
    run_tc_nt(A, B, K, exact, F_RELU | F_SCALE, torch.randn(N, device="cuda"), BN=bn, n_tiles=n_tiles,
              name="tc_nt over-wide %d x %d %s N%d" % (n_tiles, bn, "exact" if exact else "fast", N))


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,positive", [(1, 152, 64, False), (1, 40, 4, True), (200, 96, 4, False),
                                            (200, 96, 20, True), (256, 2400, 2400, True), (256, 2400, 2400, False)])
@pytest.mark.parametrize("exact", [True, False])
def test_tc_nt_edge_shapes(M, N, K, positive, exact):
    A, B = operands(M, N, K, K, positive, exact, seed=M + N + K)
    run_tc_nt(A, B, K, exact, 0 if exact else F_RELU | F_SCALE, None,
              name="tc_nt M%d N%d K%d %s %s" % (M, N, K, "pos" if positive else "rand", "exact" if exact else "fast"))


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [F_DROP | F_RESID, F_GATE, F_RELU | F_DROP | F_REP])
def test_tc_nt_unaligned_bases_are_bitwise_aligned(flags):
    M, N, K = 129, 236, 36
    A, B = operands(M, N, K, K, False, True, seed=flags)
    g = torch.Generator(device="cuda").manual_seed(3)
    gate = torch.randn(M, N, device="cuda", generator=g)
    resid = torch.randn(M, N, device="cuda", generator=g)
    bias = torch.randn(N, device="cuda", generator=g)
    kw = dict(rep=(43, 129), gate=gate if flags & F_GATE else None, resid=resid if flags & F_RESID else None)
    ref = run_tc_nt(at_offset(A, 0), at_offset(B, 0), K, True, flags, bias, name="tc_nt aligned %s" % flag_name(flags),
                    **kw)
    for off in (16, 48, 80, 112):
        kw = dict(rep=(43, 129), gate=at_offset(gate, off) if flags & F_GATE else None,
                  resid=at_offset(resid, off) if flags & F_RESID else None)
        got = run_tc_nt(at_offset(A, off), at_offset(B, off), K, True, flags, bias,
                        name="tc_nt +%d bytes %s" % (off, flag_name(flags)), **kw)
        assert torch.equal(got.view(torch.int32), ref.view(torch.int32)), off


# ---- gemm_f32 ------------------------------------------------------------------------------------------------------
def run_gemm(M, N, K, *, ta=0, tb=0, nz=1, nz_inner=1, c_t=False, nsplit=1, asum=False, alpha=1.0, bias=False,
             relu=False, rowscale_mod=0, gate=False, p=0.0, rep=None, resid=False, pdob=0, positive=False, seed=0,
             name=""):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rnd = (lambda *s: torch.rand(*s, device="cuda", generator=g)) if positive else \
        (lambda *s: torch.randn(*s, device="cuda", generator=g))
    # operands in their storage layouts, padded strides; logical A(z) [M, K], B(z) [K, N]
    Aw, Bw = (M + 5 if ta else K + 3), (K + 1 if tb else N + 2)
    Ast = rnd(nz, (K if ta else M), Aw)
    Bst = rnd(nz, (N if tb else K), Bw)
    Al = (Ast[:, :, :M].transpose(1, 2) if ta else Ast[:, :, :K])
    Bl = (Bst[:, :, :K].transpose(1, 2) if tb else Bst[:, :, :N])
    a = gemm_args(A=Ast.data_ptr(), B=Bst.data_ptr(), M=M, N=N, K=K, ta=ta, tb=tb, nz=nz, nz_inner=nz_inner,
                  alpha=alpha, nsplit=nsplit)
    if ta: a.sAk, a.sAi = Aw, 1
    else: a.sAi, a.sAk = Aw, 1
    if tb: a.sBj, a.sBk = Bw, 1
    else: a.sBk, a.sBj = Bw, 1
    zs = lambda st: (nz_inner * st, st)
    a.sAzo, a.sAzi = zs(Ast.stride(0))
    a.sBzo, a.sBzi = zs(Bst.stride(0))
    P = torch.einsum("zik,zkj->zij", Al.double(), Bl.double())
    S = torch.einsum("zik,zkj->zij", Al.double().abs(), Bl.double().abs())
    epi = Epi(P)
    if alpha != 1.0:
        epi.mul(torch.full_like(P, alpha))
    ext = {}
    if bias:
        ext["bias"] = rnd(N)
        a.bias = ext["bias"].data_ptr()
        epi.add(ext["bias"].double())
    if relu:
        a.relu = 1
        epi.relu()
    if rowscale_mod:
        ext["rs"] = 0.5 + torch.rand(rowscale_mod, device="cuda", generator=g)
        a.rowscale, a.rowscale_mod = ext["rs"].data_ptr(), rowscale_mod
        epi.mul(ext["rs"].double()[torch.arange(M, device="cuda") % rowscale_mod][None, :, None].expand_as(P))
    if gate:
        ext["gate"] = torch.randn(M, N + 3, device="cuda", generator=g)
        a.gate, a.gate_ld, a.gate_scale = ext["gate"].data_ptr(), N + 3, 1.25
        epi.mul(torch.where(ext["gate"][:, :N] > 0, 1.25, 0.0).double()[None].expand_as(P))
    if p > 0:
        ext["rng"] = rng_tensor()
        a.drop_p, a.rng, a.drop_site = p, ext["rng"].data_ptr(), 50
        if rep:
            a.rep_B, a.rep_Bc = rep
        epi.mul(dev(drop_scale(M, N, p, 50, rep))[None].expand_as(P))
    if resid:
        ext["resid"] = torch.randn(M, N + 1, device="cuda", generator=g)
        a.resid, a.resid_ld = ext["resid"].data_ptr(), N + 1
        epi.add(ext["resid"][:, :N].double())
    if pdob:
        pN = 5
        pB, T = M // pN, N // pdob
        pD = pN * pdob + 3
        a.perm, a.pB, a.pN, a.pdob, a.pD = 1, pB, pN, pdob, pD
        cbuf, cview = canaried(T * pB * pD)
    else:
        Cz = M * N + 8            # per-z slab with a gap the kernel must not touch
        cbuf, cview = canaried(nz * Cz)
        a.sCzo, a.sCzi = nz_inner * Cz, Cz
        if c_t: a.sCi, a.sCj = 1, M
        else: a.sCi, a.sCj = N, 1
    a.C = cview.data_ptr()
    asum_t = torch.full((M,), float("nan"), device="cuda") if asum else None
    a.asum = L.ptr(asum_t)
    partial = None
    if nsplit == 0:
        rc = lib().rd_debug_gemm_f32(C.byref(a), None, L.stream_ptr())
        assert rc == (-2 if a.partial_floats > 0 else 0), (rc, a.nsplit, a.partial_floats)
        if a.partial_floats > 0:
            partial = torch.empty(a.partial_floats, device="cuda")
    elif nsplit > 1:
        partial = torch.empty(nsplit * (M * N + M), device="cuda")
    if nsplit != 0 or partial is not None:
        L.check(lib().rd_debug_gemm_f32(C.byref(a), L.ptr(partial), L.stream_ptr()), "rd_debug_gemm_f32 " + name)
    torch.cuda.synchronize()
    assert_canaries(cbuf)
    if pdob:
        img = cview.view(T, pB, pD)
        assert torch.isnan(img[:, :, pN * pdob:]).all(), "the permuted store wrote past n*pdob + pdob - 1"
        out = img[:, :, :pN * pdob].reshape(T, pB, pN, pdob).permute(1, 2, 0, 3).reshape(1, M, N)
    else:
        slabs = cview.view(nz, -1)
        assert torch.isnan(slabs[:, M * N:]).all(), "a write between the z slabs"
        out = slabs[:, :M * N].reshape(nz, N, M).transpose(1, 2) if c_t else slabs[:, :M * N].reshape(nz, M, N)
    ns = max(a.nsplit, 1)
    check(name, out, epi, S, K + ns + 2)
    if asum:
        ref = Al[0].double().sum(1)
        s_abs = Al[0].double().abs().sum(1)
        err = (asum_t.double() - ref).abs()
        assert (err <= (K + ns + 2) * U * s_abs).all(), float((err / (U * s_abs)).max())
    return a


@pytest.mark.gpu
@pytest.mark.parametrize("ta,tb", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_gemm_f32_operand_layouts(ta, tb):
    run_gemm(77, 131, 45, ta=ta, tb=tb, seed=ta * 2 + tb, name="gemm_f32 ta%d tb%d M77 N131 K45" % (ta, tb))
    run_gemm(130, 66, 300, ta=ta, tb=tb, positive=True, seed=9, name="gemm_f32 ta%d tb%d M130 N66 K300 pos" % (ta, tb))


@pytest.mark.gpu
@pytest.mark.parametrize("c_t", [False, True])
def test_gemm_f32_batched_and_transposed_c(c_t):
    run_gemm(70, 68, 33, ta=0, tb=1, nz=6, nz_inner=3, c_t=c_t, alpha=0.75, seed=4,
             name="gemm_f32 nz6/3 %s" % ("C^T" if c_t else "C"))
    if c_t:
        run_gemm(65, 129, 17, ta=1, tb=0, c_t=True, seed=5, name="gemm_f32 ta1 C^T")


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [dict(bias=True), dict(relu=True, bias=True), dict(rowscale_mod=7),
                                dict(rowscale_mod=1, alpha=-0.5), dict(gate=True), dict(p=0.3),
                                dict(p=0.3, rep=(5, 15)), dict(resid=True),
                                dict(alpha=0.5, bias=True, relu=True, rowscale_mod=3, gate=True, p=0.2, resid=True)],
                         ids=["bias", "bias+relu", "rowscale7", "alpha+rowscale1", "gate", "drop", "drop-rep", "resid",
                              "all"])
def test_gemm_f32_every_epilogue_field(kw):
    run_gemm(75, 132, 70, ta=0, tb=1, seed=len(kw), name="gemm_f32 " + ",".join(sorted(kw)), **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("pdob", [1, 3, 4, 16])
def test_gemm_f32_permuted_store(pdob):
    run_gemm(35, 48, 40, ta=0, tb=1, pdob=pdob, bias=True, relu=True, seed=pdob, name="gemm_f32 perm pdob=%d" % pdob)


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,nsplit", [(37, 45, 5000, 0), (130, 70, 20000, 0), (37, 45, 33, 2), (37, 45, 65, 3),
                                          (37, 45, 97, 7), (37, 45, 4081, 256), (37, 45, 1000, 7)])
def test_gemm_f32_split_k(M, N, K, nsplit):
    if nsplit > 1:      # K just above (nsplit - 1) chunks except the last case
        chunk = -(-(-(-K // nsplit)) // 16) * 16
        assert (nsplit - 1) * chunk < K
    a = run_gemm(M, N, K, ta=1, tb=0, nsplit=nsplit, asum=True, alpha=0.5 if nsplit == 7 else 1.0, seed=K,
                 positive=K % 2 == 1, name="gemm_f32 split-K M%d N%d K%d ns%d" % (M, N, K, nsplit))
    if nsplit == 0:
        assert a.nsplit > 1, a.nsplit


# ---- split_weights and colsum --------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols", [(37, 52), (240, 240), (1, 5)])
def test_split_weights_bitwise(rows, cols):
    g = np.random.default_rng(rows)
    w = (g.standard_normal((rows, cols)) * np.exp2(g.integers(-20, 20, (rows, cols)))).astype(np.float32)
    flat = w.reshape(-1)
    flat[:3] = [0.0, -0.0, 1.0]
    n_ties = min(8, flat.size - 3)      # exact RN ties: the low 13 bits are 0x1000
    flat[3:3 + n_ties] = ((g.integers(1 << 23, 1 << 30, n_ties).astype(np.uint32) & ~np.uint32(0x1FFF)) |
                          np.uint32(0x1000)).view(np.float32)
    wd = dev(w)
    outs = [torch.full((rows * cols,), float("nan"), device="cuda") for _ in range(5)]
    L.check(lib().rd_debug_split_weights(wd.data_ptr(), rows, cols, *[o.data_ptr() for o in outs], L.stream_ptr()),
            "rd_debug_split_weights")
    lo, t, t_lo, rn, rn_t = (o.cpu().numpy().view(np.uint32) for o in outs)
    want_lo = (w - trunc19(w))
    assert (lo == want_lo.reshape(-1).view(np.uint32)).all()
    assert (t == np.ascontiguousarray(w.T).reshape(-1).view(np.uint32)).all()
    assert (t_lo == np.ascontiguousarray(want_lo.T).reshape(-1).view(np.uint32)).all()
    assert (rn == tf32_rna(w).reshape(-1).view(np.uint32)).all()
    assert (rn_t == np.ascontiguousarray(tf32_rna(w).T).reshape(-1).view(np.uint32)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols,ld", [(1000, 37, 41), (31, 200, 200), (4097, 3, 4)])
def test_colsum_bound(rows, cols, ld):
    g = torch.Generator(device="cuda").manual_seed(rows)
    x = torch.randn(rows, ld, device="cuda", generator=g)
    x[:, cols:] = float("nan")
    chunks = -(-rows // 32)
    scratch = torch.empty(chunks * cols, device="cuda")
    outb, out = canaried(cols)
    L.check(lib().rd_debug_colsum(x.data_ptr(), rows, cols, ld, out.data_ptr(), scratch.data_ptr(), L.stream_ptr()),
            "rd_debug_colsum")
    torch.cuda.synchronize()
    assert_canaries(outb)
    xd = x[:, :cols].double()
    err = (out.double() - xd.sum(0)).abs()
    bound = (32 + chunks) * U * xd.abs().sum(0)
    assert (err <= bound).all(), float((err / (U * xd.abs().sum(0))).max())
