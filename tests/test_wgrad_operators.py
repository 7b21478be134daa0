"""The weight-gradient launch on its own, element by element against float64.

One grouped launch computes every weight and bias gradient of a training step: tc_wgrad_kernel (rd_tc_gemm.cu, wgmma)
writes dW = dY^T X and db = sum_r dY[r, :] (a ones column appended to X) per (m tile, n tile, row split) into partial
slabs, and wgrad_reduce_kernel sums the slabs in split order, together with the column sums riding along in the same
launch (the LayerNorm dgamma / dbeta partial rows, ColsumItem).  Here the pair runs through rd_debug_wgrad_group: exactly
one tc_wgrad_kernel launch (none for n = 0) and one reduce launch, every problem the tensor-core kernel does not take
refused, and the plan that ran written back (tile width, rows target, each problem's nsplit and rows_per_split).  Every
output element is compared with the float64 product P = dY^T X (db: P's ones column) against a COMPONENTWISE bound in
units of u = 2^-24 times S = |dY|^T |X|, built from the written-back plan.  A normwise tolerance cannot see a wrong
small-magnitude slice (a lost lo image of one column group, a swapped row that dominates its k-block, a split counted
twice); these bounds can.

Bounds (derived, not fitted; the 3xTF32 step is derived in test_gemm_operators.py).
  * One split s of R_s <= rows_per_split rows is tc_nt's error-compensated product with K = R_s: A = dY^T split into
    hi / lo in registers, B = X^T split by the transposing producer (hi = trunc19, lo = the exact remainder, which the
    MMA reads as its top 19 bits), per k8 step lo.hi, hi.lo, hi.hi added to an fp32 accumulator with truncation.  Rows
    past R_s arrive as zeros and add exact zeros.  |D_s - P_s| <= (6 ceil(R_s/8) + 48) u S_s.
  * The reduce copies slab 0 (0 + D_0 is exact) and adds the other nsplit - 1 slabs one by one in slab order, fp32
    round to nearest (eight loads in flight, still added in order; the zeros that pad the last batch of eight add
    nothing).  Each addition errs by at most u times a running sum bounded by sum_s |D_s| <= S (1 + 64 ceil(R/8) u):
    (nsplit - 1) u S to first order, and one more u S covers the second-order terms at these sizes.
    => |dW - P| <= (6 ceil(rows_per_split/8) + 48 + nsplit) u S.
    The bias uses the same bound: the ones column is exact in TF32 (hi = 1, lo = 0), S = sum_r |dY[r, m]|.
  * Column sums (kind 1): lane l adds partial rows l, l + 32, ... in order (ceil(nsplit/32) - 1 roundings after the
    exact first), then a 5-level butterfly: at most ceil(nsplit/32) + 4 roundings, each below u sum |partial|; one more
    u covers the second-order terms.  => |out - sum| <= (ceil(nsplit/32) + 5) u sum |partial|.
  * The CUDA-core split-K path that rd_linear_wgrad_group takes for other shapes: (K + nsplit + 2) u S with
    nsplit <= 256 (test_gemm_operators.py).
Every other disagreement fails, NaN included.  The worst err / (u S) of each case is printed.

CPU: a numpy emulation of the launch's arithmetic (row splits, emulate_3xtf32 per split, the sequential slab sum) stays
inside the bound on every operand family, and each of these mutations breaks it on at least one element of every family
that can show it: (a) one split's lo.hi dropped on one k-step, (b) the lo term of one 16-column group of X zeroed, (c)
one split left out of the reduce / one added twice, (d) the ones column missing the last row of a split, (e) two
adjacent rows swapped inside each 32-row k-block.  And the debug entry's refusals.
GPU: every tile width against tails (Nout 16 / 68 / 132 with an empty second MMA warpgroup / 200; Kin 16, 156, the width
and twice the width, where the last n tile holds only the ones column; 1 to 513 rows), nsplit 1, 7, 8, 9, 17 and a
capped count; the ten problems of the P19, PAM and LARGE steps; the operand families (random, positive, power-of-two row
and column scales, post-ReLU X, TF32-rounded X, zero and dropout rows of dY); NaN footprints, rows past `rows` that
change no bit, NaN-filled partial slabs and untouched guards; the scalar dW store, db = NULL, dY = X, column sums next
to weight problems and alone; and rd_linear_wgrad_group across a WG_MAX flush with CUDA-core problems mixed in.
"""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from raindrop_b200 import lib as L
from test_gemm_operators import FAKE, U, emulate_3xtf32, refused, tc_bound, trunc19

WIDTHS = [32, 64, 96, 128, 144, 160]
WG_MAX, CS_MAX = 12, 36
SPLITK_MAX = 256            # the CUDA-core split-K path's largest split count (gemm_splitk_plan)
BATCH = {"P19": 128, "PAM": 256, "LARGE": 512}
WORST = {}


def lib():
    return L.load()


def wgrad_coef(rows_per_split, nsplit):
    return tc_bound(rows_per_split, True) + nsplit


def colsum_coef(nsplit):
    return math.ceil(nsplit / 32) + 5


# ---- CPU: the launch's arithmetic in numpy, and mutations of it ---------------------------------------------------
def emulate_launch(dY, X, rows_per_split, mutation=None):
    """dW, db as the launch computes them: per row split the 3xTF32 product of dY^T and [X | 1]^T, then the slabs
    added in order in fp32.  `mutation` names one of the errors (a) - (e) of the module docstring; split 1 is the one
    it hits where it hits one."""
    rows, kin = X.shape
    Xo = np.concatenate([X, np.ones((rows, 1), np.float32)], 1)
    slabs = []
    for s, r0 in enumerate(range(0, rows, rows_per_split)):
        A = np.ascontiguousarray(dY[r0:r0 + rows_per_split].T)          # [Nout, R_s]
        B = np.ascontiguousarray(Xo[r0:r0 + rows_per_split].T)          # [Kin + 1, R_s]
        skip = None
        if mutation == "a" and s == 1:
            skip = A.shape[1] // 8 - 1
        if mutation == "b":                   # X's lo image of columns 16 .. 31 lost: the MMA sees hi only
            B[16:32] = trunc19(B[16:32])
        if mutation == "d" and s == 1:
            B[kin, -1] = 0.0
        if mutation == "e":
            for k0 in range(0, A.shape[1] - 3, 32):
                A[:, [k0 + 2, k0 + 3]] = A[:, [k0 + 3, k0 + 2]]
        slabs.append(emulate_3xtf32(A, B, skip_lo_hi_step=skip))
    if mutation == "c-":
        del slabs[1]
    if mutation == "c+":
        slabs.insert(2, slabs[1])
    acc = np.zeros_like(slabs[0])
    for sl in slabs:
        acc = (acc + sl).astype(np.float32)
    return acc[:, :kin], acc[:, kin]


def np_operands(rows, nout, kin, family, seed):
    rng = np.random.default_rng(seed)
    if family == "positive":
        dY, X = rng.random((rows, nout)), rng.random((rows, kin))
    else:
        dY, X = rng.standard_normal((rows, nout)), rng.standard_normal((rows, kin))
    if family == "scaled":           # one row dominates each k-block; columns spread too: 2^-12 .. 2^12 per element
        e = lambda *s: np.exp2(rng.integers(-6, 7, s))
        dY, X = dY * e(rows, 1) * e(1, nout), X * e(rows, 1) * e(1, kin)
    if family == "relu":
        X = np.maximum(X, 0.0)
    if family == "tf32":
        X = trunc19(X.astype(np.float32) + np.float32(0))      # representable in TF32: lo is all zeros
    if family == "dropout":
        dY[rng.random(rows) < 0.3] = 0.0
        dY = dY * (rng.random((rows, nout)) > 0.2) / 0.8
    return dY.astype(np.float32), X.astype(np.float32)


CPU_SHAPE = (100, 20, 36, 32)        # rows, Nout, Kin, rows per split: splits of 32, 32, 32 and 4 rows
FAMILIES = ["random", "positive", "scaled", "relu", "tf32", "dropout"]
# (b) cannot show on TF32-rounded X, whose lo image is zero to begin with
MUTATIONS = [(m, f) for m in ("a", "b", "c-", "c+", "d", "e") for f in FAMILIES if (m, f) != ("b", "tf32")]


def np_check(dW, db, dY, X, coef):
    d, x = dY.astype(np.float64), X.astype(np.float64)
    P, S = d.T @ x, np.abs(d).T @ np.abs(x)
    Pb, Sb = d.sum(0), np.abs(d).sum(0)
    err = np.concatenate([np.abs(dW - P), np.abs(db - Pb)[:, None]], 1)
    scale = np.concatenate([S, Sb[:, None]], 1)
    return ~(err <= coef * U * scale), err / np.where(scale > 0, U * scale, 1.0)


@pytest.mark.parametrize("family", FAMILIES)
def test_emulated_launch_within_bound(family):
    rows, nout, kin, rps = CPU_SHAPE
    dY, X = np_operands(rows, nout, kin, family, seed=len(family))
    bad, ratio = np_check(*emulate_launch(dY, X, rps), dY, X, wgrad_coef(rps, -(-rows // rps)))
    assert not bad.any(), ratio.max()


@pytest.mark.parametrize("mutation,family", MUTATIONS)
def test_bound_sees_each_mutation(mutation, family):
    rows, nout, kin, rps = CPU_SHAPE
    dY, X = np_operands(rows, nout, kin, family, seed=len(family))
    bad, ratio = np_check(*emulate_launch(dY, X, rps, mutation), dY, X, wgrad_coef(rps, -(-rows // rps)))
    assert bad.any(), (mutation, family, ratio.max())


@pytest.mark.parametrize("mutation", ["a", "b", "c-", "c+", "d", "e"])
def test_scaled_family_sees_each_mutation_at_a_step_split(mutation):
    """At the step's split length (544 rows) one lost lo.hi k-step hides under the bound of random, positive, ReLU and
    dropout operands; with one row dominating each k-block it does not."""
    rows, nout, kin, rps = 1100, 20, 36, 544
    dY, X = np_operands(rows, nout, kin, "scaled", seed=6)
    coef = wgrad_coef(rps, -(-rows // rps))
    assert not np_check(*emulate_launch(dY, X, rps), dY, X, coef)[0].any()
    bad, ratio = np_check(*emulate_launch(dY, X, rps, mutation), dY, X, coef)
    assert bad.any(), (mutation, ratio.max())
    if mutation == "a":
        r = np_operands(rows, nout, kin, "random", seed=6)
        assert not np_check(*emulate_launch(*r, rps, mutation), *r, coef)[0].any()


# ---- the debug entry and its refusals ------------------------------------------------------------------------------
def wgrad_items(specs):
    """specs: dicts of rd_wgrad_item fields plus 'bytes' (the partial buffer's size)"""
    n = len(specs)
    items, sizes = (L.RdWgradItem * max(n, 1))(), (C.c_uint64 * max(n, 1))()
    for i, s in enumerate(specs):
        for k, v in s.items():
            if k == "bytes":
                sizes[i] = v
            else:
                setattr(items[i], k, v)
    return items, sizes


def colsum_items(specs):
    cs = (L.RdDebugColsumItem * max(len(specs), 1))()
    for i, s in enumerate(specs):
        for k, v in s.items():
            setattr(cs[i], k, v)
    return cs


def fake_item(rows=300, nout=64, kin=64, **kw):
    s = dict(d_out=FAKE, x=FAKE, rows=rows, out_features=nout, in_features=kin, d_weight=FAKE, d_bias=FAKE,
             partial=FAKE, bytes=lib().rd_linear_wgrad_partial_bytes(rows, nout, kin))
    s.update(kw)
    return s


def call(specs, cs_specs=(), plan=None):
    items, sizes = wgrad_items(specs)
    plan = plan or L.RdDebugWgradPlan()
    return lib().rd_debug_wgrad_group(items, sizes, len(specs), colsum_items(cs_specs), len(cs_specs), C.byref(plan),
                                      None)


FAKE_CS = dict(partial=FAKE, out=FAKE, stride=64, nsplit=3, ncols=64)


@pytest.mark.parametrize("n,ncs", [(WG_MAX + 1, 0), (0, CS_MAX + 1), (WG_MAX + 1, CS_MAX + 1)])
def test_refuses_too_many_items(n, ncs):
    refused(call([fake_item()] * n, [FAKE_CS] * ncs), "at most 12 problems and 36 column sums")


@pytest.mark.parametrize("kw,what", [
    (dict(out_features=66), "tensor-core kernel"), (dict(in_features=62), "tensor-core kernel"),
    (dict(out_features=12), "tensor-core kernel"), (dict(in_features=12), "tensor-core kernel"),
    (dict(d_out=FAKE + 4), "tensor-core kernel"), (dict(x=FAKE + 8), "tensor-core kernel"),
    (dict(partial=FAKE + 12), "tensor-core kernel"),
    (dict(d_out=0), "NULL pointer"), (dict(d_weight=0), "NULL pointer"), (dict(rows=0), "no rows"),
])
def test_refuses_what_the_tensor_cores_do_not_take(kw, what):
    spec = fake_item()
    spec.update(kw)
    refused(call([fake_item(), spec]), what)


@pytest.mark.parametrize("rows,nout,kin", [(300, 64, 64), (100000, 2400, 2400), (1, 16, 16)])
def test_refuses_an_undersized_partial(rows, nout, kin):
    need = lib().rd_linear_wgrad_partial_bytes(rows, nout, kin)
    refused(call([fake_item(rows, nout, kin, bytes=need - 4)]), "partial buffer of %d bytes" % (need - 4))


def test_refuses_a_bad_column_sum():
    refused(call([], [dict(FAKE_CS, nsplit=0)]), "bad column sum 0")
    refused(call([], [FAKE_CS, dict(FAKE_CS, stride=63)]), "bad column sum 1")


# ---- GPU harness ---------------------------------------------------------------------------------------------------
GUARD = 32                                   # guard floats before and after every output
GUARD_BITS = 0x7FA5A5A5                      # a NaN with a payload no kernel writes


def guarded(n, off=0):
    """(buffer, view): n floats starting off floats past a 128-byte boundary, GUARD_BITS around them"""
    buf = torch.full((n + 2 * GUARD + off,), GUARD_BITS, dtype=torch.int32, device="cuda")
    assert buf.data_ptr() % 128 == 0
    return buf, buf[GUARD + off:GUARD + off + n].view(torch.float32)


def assert_guards(buf, n, off=0):
    head, tail = buf[:GUARD + off], buf[GUARD + off + n:]
    assert (head == GUARD_BITS).all() and (tail == GUARD_BITS).all(), "a write outside the output"


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def operands(rows, nout, kin, family="random", seed=0, pad=0, pad_value=float("nan")):
    """dY [rows, nout], X [rows, kin] on the device as views of [rows + pad, .] buffers whose last pad rows hold
    pad_value (the kernel must never read them)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    R = rows + pad
    draw = torch.rand if family == "positive" else torch.randn
    dY, X = draw(R, nout, device="cuda", generator=g), draw(R, kin, device="cuda", generator=g)
    if family == "scaled":
        e = lambda *s: torch.exp2(torch.randint(-6, 7, s, device="cuda", generator=g).float())
        dY, X = dY * e(R, 1) * e(1, nout), X * e(R, 1) * e(1, kin)
    if family == "relu":
        X = X.clamp_min(0.0)
    if family == "tf32":
        X = ((X.view(torch.int32) + 0x1000) & -8192).view(torch.float32)
    if family == "dropout":
        dY[torch.rand(R, device="cuda", generator=g) < 0.3] = 0.0
        dY = dY * (torch.rand(R, nout, device="cuda", generator=g) > 0.2) / 0.8
    dY[rows:], X[rows:] = pad_value, pad_value
    return dY[:rows], X[:rows]


class Prob:
    """one weight-gradient problem: operands, guarded outputs, a NaN-filled partial buffer"""

    def __init__(self, dY, X, *, bias=True, dw_off=0):
        self.dY, self.X = dY, X
        self.rows, self.nout = dY.shape
        self.kin = X.shape[1]
        self.dw_off = dw_off
        self.wbuf, self.dW = guarded(self.nout * self.kin, dw_off)
        self.dW = self.dW.view(self.nout, self.kin)
        self.bbuf, self.db = guarded(self.nout) if bias else (None, None)
        self.bytes = lib().rd_linear_wgrad_partial_bytes(self.rows, self.nout, self.kin)
        self.partial = torch.full((self.bytes // 4,), float("nan"), device="cuda")

    def spec(self):
        return dict(d_out=self.dY.data_ptr(), x=self.X.data_ptr(), rows=self.rows, out_features=self.nout,
                    in_features=self.kin, d_weight=self.dW.data_ptr(), d_bias=L.ptr(self.db),
                    partial=self.partial.data_ptr(), bytes=self.bytes)

    def assert_guards(self):
        assert_guards(self.wbuf, self.nout * self.kin, self.dw_off)
        if self.bbuf is not None:
            assert_guards(self.bbuf, self.nout)


class Colsum:
    """out[c] = sum_s partial[s * stride + c]: a guarded output over a slice of a [nsplit, stride] block"""

    def __init__(self, part, col0, ncols):
        self.part, self.col0, self.ncols = part, col0, ncols
        self.buf, self.out = guarded(ncols)

    def spec(self):
        return dict(partial=self.part.data_ptr() + 4 * self.col0, out=self.out.data_ptr(), stride=self.part.shape[1],
                    nsplit=self.part.shape[0], ncols=self.ncols)


def run(probs, colsums=(), bn=None):
    """one rd_debug_wgrad_group call; returns the written-back plan"""
    items, sizes = wgrad_items([p.spec() for p in probs])
    cs = colsum_items([c.spec() for c in colsums])
    plan = L.RdDebugWgradPlan()
    if bn is not None:
        os.environ["RD_TC_WGRAD_BN"] = str(bn)
    try:
        L.check(lib().rd_debug_wgrad_group(items, sizes, len(probs), cs, len(colsums), C.byref(plan), L.stream_ptr()),
                "rd_debug_wgrad_group")
        torch.cuda.synchronize()
    finally:
        os.environ.pop("RD_TC_WGRAD_BN", None)
    for p in probs:
        p.assert_guards()
    for c in colsums:
        assert_guards(c.buf, c.ncols)
    if bn is not None and probs:
        assert plan.BN == bn, (plan.BN, bn)
    assert (plan.BN == 0) == (not probs), plan.BN
    return plan


def reference(dY, X, chunk=8192):
    """float64 P = dY^T [X | 1] and S = |dY|^T |[X | 1]| ([Nout, Kin + 1]) in row chunks on the device"""
    nout, kin = dY.shape[1], X.shape[1]
    P = torch.zeros(nout, kin + 1, dtype=torch.float64, device="cuda")
    S = torch.zeros_like(P)
    for r0 in range(0, dY.shape[0], chunk):
        d = dY[r0:r0 + chunk].double()
        x = torch.cat([X[r0:r0 + chunk].double(), torch.ones(d.shape[0], 1, dtype=torch.float64, device="cuda")], 1)
        P.addmm_(d.T, x)
        S.addmm_(d.abs().T, x.abs())
    return P, S


def check(name, dW, db, ref, coef, nan_mask=None):
    """|[dW | db] - P| <= coef u S element by element, NaN failing (except where nan_mask expects exactly NaN)"""
    P, S = ref
    out = dW.double() if db is None else torch.cat([dW.double(), db.double()[:, None]], 1)
    P, S = P[:, :out.shape[1]], S[:, :out.shape[1]]
    err = (out - P).abs()
    bad = ~(err <= coef * U * S)
    live = S > 0
    if nan_mask is not None:
        nan_mask = nan_mask[:, :out.shape[1]]
        assert torch.equal(torch.isnan(out), nan_mask), (name, "NaN footprint", int(torch.isnan(out).sum()),
                                                         int(nan_mask.sum()))
        bad &= ~nan_mask
        live &= ~nan_mask
    ratio = float((err[live] / (U * S[live])).max()) if live.any() else 0.0
    WORST[name] = max(WORST.get(name, 0.0), ratio)
    fin = ~torch.isnan(P)
    normwise = float(err[fin].max() / P[fin].abs().max()) if fin.any() else 0.0
    print("%-62s worst err/(u S) %8.2f   bound %5d   normwise %.1e" % (name, ratio, coef, normwise))
    assert not bad.any(), (name, int(bad.sum()), ratio, coef)
    return ratio


def check_prob(name, p, plan, k, ref=None, nan_mask=None):
    ref = ref if ref is not None else reference(p.dY, p.X)
    return check(name, p.dW, p.db, ref, wgrad_coef(plan.rows_per_split[k], plan.nsplit[k]), nan_mask)


def check_colsum(name, c):
    x = c.part[:, c.col0:c.col0 + c.ncols].double()
    err = (c.out.double() - x.sum(0)).abs()
    s = x.abs().sum(0)
    coef = colsum_coef(c.part.shape[0])
    ratio = float((err / (U * s)).max())
    WORST[name] = max(WORST.get(name, 0.0), ratio)
    print("%-62s worst err/(u S) %8.2f   bound %d" % (name, ratio, coef))
    assert (err <= coef * U * s).all(), (name, ratio, coef)


# ---- rd_linear_wgrad_group, held to its engines' bounds (the other wgrad test files use this) ---------------------
def takes_tensor_cores(dY, X):
    """the problems rd_linear_wgrad_group queues for the grouped tensor-core launch; the others go to split-K"""
    rows, nout = dY.shape
    kin = X.shape[1]
    aligned = (dY.data_ptr() | X.data_ptr()) % 16 == 0
    return rows >= 256 and nout % 4 == 0 and kin % 4 == 0 and nout >= 16 and kin >= 16 and aligned


def check_public(ops, outs, tag, bn=None):
    """outs [(dW, db)] of one rd_linear_wgrad_group call over ops [(dY, X)], element by element: the tensor-core
    problems, in the groups of at most WG_MAX the call flushes, run again through rd_debug_wgrad_group, which must give
    the same bits and the plan their bound is built from; the CUDA-core problems to split-K's bound"""
    tc = [i for i, (dY, X) in enumerate(ops) if takes_tensor_cores(dY, X)]
    for grp in [tc[j:j + WG_MAX] for j in range(0, len(tc), WG_MAX)]:
        probs = [Prob(*ops[i]) for i in grp]
        plan = run(probs, bn=bn)
        for k, (i, p) in enumerate(zip(grp, probs)):
            dW, db = outs[i]
            assert same_bits(dW, p.dW) and same_bits(db, p.db), (tag, i, "differs from the debug entry's launch")
            name = "%s: %d x %d, %d rows, %d x %d rows" % (tag, p.nout, p.kin, p.rows, plan.nsplit[k],
                                                          plan.rows_per_split[k])
            check(name, dW, db, reference(*ops[i]), wgrad_coef(plan.rows_per_split[k], plan.nsplit[k]))
    for i in sorted(set(range(len(ops))) - set(tc)):
        dY, X = ops[i]
        check("%s: %d x %d, %d rows (CUDA cores)" % (tag, dY.shape[1], X.shape[1], dY.shape[0]), *outs[i],
              reference(dY, X), dY.shape[0] + SPLITK_MAX + 2)


# ---- tails and widths ----------------------------------------------------------------------------------------------
TAIL_ROWS = {1: "random", 31: "positive", 33: "scaled", 256: "relu", 513: "tf32"}


@pytest.mark.gpu
@pytest.mark.parametrize("bn", WIDTHS)
def test_tails_every_width(bn):
    """Nout 16 and 132 leave an m tile's second MMA warpgroup without rows; Kin = width and 2 x width put the ones
    column alone into the last n tile"""
    shapes = [(nout, kin) for nout in (16, 68, 132, 200) for kin in (16, 156, bn, 2 * bn)]
    for rows, family in TAIL_ROWS.items():
        for half in (shapes[:8], shapes[8:]):
            probs = [Prob(*operands(rows, nout, kin, family, seed=rows + nout + kin, pad=5)) for nout, kin in half]
            plan = run(probs, bn=bn)
            for k, p in enumerate(probs):
                check_prob("tails w%d %s %d x %d, %d rows" % (bn, family, p.nout, p.kin, rows), p, plan, k)


@pytest.mark.gpu
@pytest.mark.parametrize("bn", [None] + WIDTHS)
def test_split_counts(bn):
    """nsplit 1, 7, 8, 9 (the reduce's batches of eight slabs: one, exactly one, one and one more) and 17 in one group,
    and a problem whose split count the partial-buffer cap lowers"""
    shapes = [(512, 64, 64, "random"), (7 * 512, 64, 64, "positive"), (8 * 512, 68, 60, "scaled"),
              (8 * 512 + 1, 64, 64, "random"), (17 * 512 - 5, 64, 36, "positive")]
    probs = [Prob(*operands(r, n, k, f, seed=r)) for r, n, k, f in shapes]
    plan = run(probs, bn=bn)
    assert list(plan.nsplit[:5]) == [1, 7, 8, 9, 17] and plan.rows_target == 512, (list(plan.nsplit), plan.rows_target)
    for k, p in enumerate(probs):
        check_prob("split counts w%s nsplit %d (%d rows)" % (bn or "default", plan.nsplit[k], p.rows), p, plan, k)
    capped = Prob(*operands(20000, 1024, 636, "positive", seed=9))
    plan = run([capped], bn=bn)
    assert plan.nsplit[0] < -(-20000 // plan.rows_target), (plan.nsplit[0], plan.rows_target)
    check_prob("capped w%s nsplit %d x %d rows" % (bn or "default", plan.nsplit[0], plan.rows_per_split[0]), capped,
               plan, 0)


# ---- the training step's problems ----------------------------------------------------------------------------------
def step_shapes(config):
    from raindrop_b200.synth import model_config
    cfg = model_config(config)
    B = BATCH[config]
    D, nhid, C_ = cfg["d_model"] + 16, cfg["nhid"], cfg["max_len"] * cfg["d_ob"]
    m2, m1 = cfg["max_len"] * B, B * cfg["d_inp"]
    enc = [(m2, D, nhid), (m2, nhid, D), (m2, D, D), (m2, 3 * D, D)]     # linear1, linear2, out_proj, in_proj
    return enc + enc + [(m1, C_, C_)] * 2


def step_group(config, family, seed=1):
    """the step's ten problems; the second encoder layer and the second ob-prop layer read the same operands as the
    first (a step's memory at LARGE): their results must be the same bits"""
    shapes = step_shapes(config)
    ops = {}
    for i, (rows, nout, kin) in enumerate(shapes):
        if (rows, nout, kin) not in ops:
            ops[(rows, nout, kin)] = operands(rows, nout, kin, family, seed=seed + i)
    return [Prob(*ops[s]) for s in shapes], shapes


def check_step(config, family, probs, shapes, plan, refs, tag):
    first = {}
    for k, (p, s) in enumerate(zip(probs, shapes)):
        if s in first:
            q = probs[first[s]]
            assert same_bits(p.dW, q.dW) and same_bits(p.db, q.db), (tag, s)
            continue
        first[s] = k
        if s not in refs:
            refs[s] = reference(p.dY, p.X)
        check_prob("%s %s %s %d x %d, %d x %d rows" % (config, tag, family, p.nout, p.kin, plan.nsplit[k],
                                                       plan.rows_per_split[k]), p, plan, k, refs[s])


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["P19", "PAM", "LARGE"])
def test_step_problems(config):
    probs, shapes = step_group(config, "random")
    plan = run(probs)
    refs = {}
    check_step(config, "random", probs, shapes, plan, refs, "default width %d" % plan.BN)
    if config != "P19":
        return
    ref_bits = [(p.dW.clone(), p.db.clone()) for p in probs]
    for bn in WIDTHS:
        plan = run(probs, bn=bn)
        for p, (w, b) in zip(probs, ref_bits):
            assert same_bits(p.dW, w) and same_bits(p.db, b), (bn, p.nout, p.kin)
        check_step(config, "random", probs, shapes, plan, refs, "width %d" % bn)


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["positive", "scaled", "relu", "tf32", "dropout"])
def test_step_problems_operand_families(family):
    probs, shapes = step_group("P19", family, seed=7)
    plan = run(probs)
    check_step("P19", family, probs, shapes, plan, {}, "")


# ---- NaN footprints, rows past `rows`, partial slabs ---------------------------------------------------------------
@pytest.mark.gpu
def test_nan_footprint():
    """a NaN at dY[r, m] makes exactly row m of dW and db[m] NaN; one at X[r, k] exactly column k of dW"""
    a = Prob(*operands(700, 132, 100, seed=1))
    b = Prob(*operands(1030, 68, 52, "scaled", seed=2))
    ref_a, ref_b = reference(a.dY, a.X), reference(b.dY, b.X)
    a.dY[600, 70] = float("nan")
    b.X[900, 45] = float("nan")
    plan = run([a, b])
    assert plan.nsplit[0] > 1 and plan.nsplit[1] > 1, list(plan.nsplit)      # the NaNs sit in a later split
    mask_a = torch.zeros(132, 101, dtype=torch.bool, device="cuda")
    mask_a[70, :] = True
    mask_b = torch.zeros(68, 53, dtype=torch.bool, device="cuda")
    mask_b[:, 45] = True
    check_prob("NaN at dY[600, 70]", a, plan, 0, ref_a, mask_a)
    check_prob("NaN at X[900, 45]", b, plan, 1, ref_b, mask_b)


@pytest.mark.gpu
@pytest.mark.parametrize("bn", [32, 160])
def test_rows_past_the_end_change_no_bit(bn):
    shapes = [(513, 132, 100), (33, 68, 156), (1000, 200, 16)]
    res = []
    for pad_value in (0.0, float("nan")):
        probs = [Prob(*operands(r, n, k, seed=r, pad=40, pad_value=pad_value)) for r, n, k in shapes]
        plan = run(probs, bn=bn)
        res.append([(p.dW.clone(), p.db.clone()) for p in probs])
    for k, p in enumerate(probs):
        check_prob("NaN rows past the end w%d %d x %d, %d rows" % (bn, p.nout, p.kin, p.rows), p, plan, k)
    for (w0, b0), (w1, b1) in zip(*res):
        assert same_bits(w0, w1) and same_bits(b0, b1)


# ---- reduce paths --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_scalar_store_no_bias_and_shared_operand():
    """dW 4, 8 and 12 bytes past a 16-byte boundary (the scalar store), db = NULL, and dY = X (the K-FAC factors)"""
    ops = operands(1500, 84, 84, "scaled", seed=3)
    ref = reference(*ops)
    probs = [Prob(*ops), Prob(*ops, dw_off=1), Prob(*ops, dw_off=2), Prob(*ops, dw_off=3, bias=False),
             Prob(ops[0], ops[0])]
    plan = run(probs)
    for k, p in enumerate(probs[:4]):
        assert same_bits(p.dW, probs[0].dW), k
        check_prob("dW +%d bytes%s" % (4 * p.dw_off, ", db NULL" if p.db is None else ""), p, plan, k, ref)
    assert probs[4].dY.data_ptr() == probs[4].X.data_ptr()
    check_prob("dY = X (X^T X)", probs[4], plan, 4)


def colsum_set(seed):
    """column sums over nsplit 1, 31, 32, 33, 100 and ncols 1, 33, 640, and a LayerNorm pair (stride 2D, beta at +D)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for ns in (1, 31, 32, 33, 100):
        for nc in (1, 33, 640):
            part = torch.randn(ns, nc + 3, device="cuda", generator=g) * torch.exp2(
                torch.randint(-8, 9, (ns, 1), device="cuda", generator=g).float())
            out.append(Colsum(part, 2 if nc < 640 else 0, nc))
    D = 84
    ln = torch.rand(33, 2 * D, device="cuda", generator=g)
    return out + [Colsum(ln, 0, D), Colsum(ln, D, D)]


@pytest.mark.gpu
@pytest.mark.parametrize("with_weights", [False, True])
def test_column_sums(with_weights):
    probs = [Prob(*operands(700, 132, 100, seed=4)), Prob(*operands(3000, 64, 36, "positive", seed=5))] \
        if with_weights else []
    cs = colsum_set(seed=int(with_weights))
    plan = run(probs, cs)
    for c in cs:
        check_colsum("colsum %s nsplit %d ncols %d" % ("next to weights" if probs else "alone", c.part.shape[0],
                                                      c.ncols), c)
    for k, p in enumerate(probs):
        check_prob("weights next to column sums %d x %d" % (p.nout, p.kin), p, plan, k)


@pytest.mark.gpu
def test_thirty_six_column_sums_alone():
    g = torch.Generator(device="cuda").manual_seed(6)
    cs = []
    for i in range(CS_MAX // 2):
        D = 16 + 12 * i
        ln = torch.randn(1 + 7 * i, 2 * D, device="cuda", generator=g)
        cs += [Colsum(ln, 0, D), Colsum(ln, D, D)]
    run([], cs)
    for c in cs:
        check_colsum("36 colsums: nsplit %d D %d" % (c.part.shape[0], c.ncols), c)


# ---- the public entry across a WG_MAX flush ------------------------------------------------------------------------
@pytest.mark.gpu
def test_public_group_crosses_wg_max():
    """13 tensor-core problems (a flush after twelve) and three CUDA-core ones: 255 rows, Nout 12, Kin 18"""
    shapes = [(256, 64, 64), (255, 64, 64), (300, 12, 64), (300, 64, 18)] + \
             [(300 + 97 * i, 16 + 20 * i, 156 - 8 * i) for i in range(12)]
    ops = [operands(r, n, k, ("random", "positive", "scaled")[i % 3], seed=i) for i, (r, n, k) in enumerate(shapes)]
    assert sum(takes_tensor_cores(*o) for o in ops) == WG_MAX + 1
    items = (L.RdWgradItem * len(ops))()
    outs, keep = [], []
    for it, (dY, X) in zip(items, ops):
        rows, nout = dY.shape
        kin = X.shape[1]
        dW = torch.full((nout, kin), float("nan"), device="cuda")
        db = torch.full((nout,), float("nan"), device="cuda")
        part = torch.full((lib().rd_linear_wgrad_partial_bytes(rows, nout, kin) // 4,), float("nan"), device="cuda")
        it.d_out, it.x, it.rows, it.out_features, it.in_features = dY.data_ptr(), X.data_ptr(), rows, nout, kin
        it.d_weight, it.d_bias, it.partial = dW.data_ptr(), db.data_ptr(), part.data_ptr()
        outs.append((dW, db))
        keep.append(part)
    L.check(lib().rd_linear_wgrad_group(items, len(ops), L.stream_ptr()), "rd_linear_wgrad_group")
    torch.cuda.synchronize()
    check_public(ops, outs, "public")
