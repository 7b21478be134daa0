"""GPU: the weight-gradient kernel loads dY by TMA (one tensor map per problem, 32 x 32 boxes, 128B swizzle) from one
thread that runs up to two k-blocks ahead of the transposing producer across work items, and transposes X with 16-byte
stores.

Every problem here has at least 256 rows, so it goes to tc_wgrad_kernel rather than the CUDA-core path.  Under each forced
width the test also reads the kernel's per-CTA k-block counts (rd_debug_wgrad_timing) and checks that they add up to
every problem's m tiles x n tiles x ceil(rows / 32) k-blocks: all of them ran through the kernel.

  * groups whose problems have rows just past a multiple of their row split (8705 = 17 x 512 + 1, 8737 = 17 x 512 + 33,
    ...), so their last split is one or two k-blocks long, next to long problems.  With enough items that CTAs take
    several each (and more at narrow widths), the issue cursor reaches such an item and crosses into the next one inside
    its lookahead.  Every width gives the same bits, within 2e-5 normwise of an fp64 product;
  * Nout just past a multiple of the 128-row m tile (the last tile's second MMA warpgroup has no rows; its dY boxes
    arrive as zeros) and Nout not a multiple of 32, with dY and X starting 16 bytes past a 128-byte boundary: the same
    bits as 128-byte aligned copies, under every width.
"""
import ctypes
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

WIDTHS = [32, 64, 96, 128, 144, 160]


def cdiv(a, b):
    return -(-a // b)


def run(operands, bn=None):
    """dW, db of every problem through one rd_linear_wgrad_group call, and the k-blocks the kernel's CTAs produced"""
    from raindrop_b200 import lib as L
    lib = L.load()
    items = (L.RdWgradItem * len(operands))()
    outs, keep = [], []
    for i, (dY, X) in enumerate(operands):
        rows, nout = dY.shape
        kin = X.shape[1]
        assert rows >= 256                      # below, the library uses the CUDA-core path instead
        dW = torch.full((nout, kin), float("nan"), device="cuda")
        db = torch.full((nout,), float("nan"), device="cuda")
        part = torch.empty(max(1, lib.rd_linear_wgrad_partial_bytes(rows, nout, kin) // 4), device="cuda")
        it = items[i]
        it.d_out, it.x, it.rows, it.out_features, it.in_features = dY.data_ptr(), X.data_ptr(), rows, nout, kin
        it.d_weight, it.d_bias, it.partial = dW.data_ptr(), db.data_ptr(), part.data_ptr()
        outs.append((dW, db))
        keep.append(part)
    dbg = torch.zeros(torch.cuda.get_device_properties(0).multi_processor_count, 16, dtype=torch.int64, device="cuda")
    if bn is not None:
        os.environ["RD_TC_WGRAD_BN"] = str(bn)
    lib.rd_debug_wgrad_timing(ctypes.c_void_p(dbg.data_ptr()))
    try:
        L.check(lib.rd_linear_wgrad_group(items, len(operands), L.stream_ptr()), "rd_linear_wgrad_group")
        torch.cuda.synchronize()
    finally:
        lib.rd_debug_wgrad_timing(None)
        os.environ.pop("RD_TC_WGRAD_BN", None)
    return outs, int(dbg[:, 8].sum())


def kernel_kblocks(operands, bn):
    """k-blocks of every (m tile, n tile, row split) item at width bn: splits are multiples of 32 rows, so per tile pair
    they add up to ceil(rows / 32) whatever the split plan"""
    return sum(cdiv(dY.shape[1], 128) * cdiv(X.shape[1] + 1, bn) * cdiv(dY.shape[0], 32) for dY, X in operands)


def same_bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def normwise(a, ref):
    return ((a.double() - ref).norm() / ref.norm()).item()


def check_fp64(operands, outs, tag):
    for (dY, X), (dW, db) in zip(operands, outs):
        assert normwise(dW, dY.double().T @ X.double()) < 2e-5, (tag, tuple(dW.shape))
        assert normwise(db, dY.double().sum(0)) < 2e-5, (tag, tuple(dW.shape))


def make(shapes, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(r, n, generator=g).cuda(), torch.randn(r, k, generator=g).cuda()) for r, n, k in shapes]


@pytest.mark.parametrize("shapes", [
    # 544-row splits (the group's item count raises the target): last splits of 33 rows (2 k-blocks) for the 8737-row
    # problems and 32 rows for the 12000-row one.  255 items at width 160, so on 132 SMs CTAs take two; in 6 the cursor
    # crosses from a 2-k-block item into a 17-k-block one (8 at width 144, 27 at width 32)
    [(8737, 200, 200), (1057, 200, 16), (4097, 64, 152), (8737, 200, 152), (8737, 64, 64), (12000, 200, 200),
     (4129, 200, 200)],
    # 512-row splits: last splits of 1 row (1 k-block) and 33 rows next to a 2000-row problem; at widths 64 and 32 the
    # CTAs take two or three items and the cursor crosses out of 1-k-block items (4 and 8 CTAs)
    [(8705, 132, 100), (8737, 128, 152), (8705, 256, 36), (8737, 96, 96), (2000, 128, 140)],
])
def test_short_last_splits_every_width(shapes):
    ops = make(shapes, seed=len(shapes))
    ref, _ = run(ops)
    check_fp64(ops, ref, "default")
    for bn in WIDTHS:
        got, kblocks = run(ops, bn)
        assert kblocks == kernel_kblocks(ops, bn), (bn, kblocks)
        check_fp64(ops, got, bn)
        for (a, b), (c, d) in zip(got, ref):
            assert same_bits(a, c) and same_bits(b, d), (bn, tuple(a.shape))


def offset_copy(t, skip_floats):
    buf = torch.empty(t.numel() + 32, device="cuda")
    assert buf.data_ptr() % 128 == 0
    v = buf[skip_floats:skip_floats + t.numel()].view_as(t)
    v.copy_(t)
    return v


@pytest.mark.parametrize("bn", WIDTHS)
def test_m_tails_unaligned_dy(bn):
    ops = make([(700, 132, 52), (1030, 196, 100), (300, 260, 16), (513, 20, 148)], seed=5)
    shifted = [(offset_copy(dY, 4 + 8 * (i % 2)), offset_copy(X, 12)) for i, (dY, X) in enumerate(ops)]
    for dY, X in shifted:
        assert dY.data_ptr() % 16 == 0 and dY.data_ptr() % 128 != 0
    ref, _ = run(ops, bn)
    got, kblocks = run(shifted, bn)
    assert kblocks == kernel_kblocks(ops, bn), (bn, kblocks)
    check_fp64(ops, got, bn)
    for (a, b), (c, d) in zip(got, ref):
        assert same_bits(a, c) and same_bits(b, d), (bn, tuple(a.shape))
