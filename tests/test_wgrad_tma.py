"""GPU: the grouped weight-gradient kernel reads X through one TMA tensor map per problem (dims {Kin, rows}, 32 x 32
boxes, 128B swizzle) and dY by cp.async.  A tensor map needs a 16-byte aligned base, not a 128-byte aligned one, so
operands that start 16, 48, 80 or 112 bytes past a 128-byte boundary must give the same bits as aligned copies of the
same data, under every tile width, and stay within 2e-5 normwise of an fp64 product.  The shapes have k-block tails
(rows not a multiple of 32), Kin not a multiple of 32 and n tiles that end past Kin (zero-filled by TMA, apart from the
ones column of the bias gradient).
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

WIDTHS = [32, 64, 96, 128, 144, 160]
SHAPES = [(1000, 68, 100), (4352, 240, 240), (7680, 152, 272), (333, 200, 16)]      # (rows, Nout, Kin)


def offset_copy(t, skip_floats):
    """a copy of t whose first element lies skip_floats floats past the 128-byte aligned start of its allocation"""
    buf = torch.empty(t.numel() + 32, device="cuda")
    assert buf.data_ptr() % 128 == 0
    v = buf[skip_floats:skip_floats + t.numel()].view_as(t)
    v.copy_(t)
    return v


def run(lib, L, operands, bn):
    items = (L.RdWgradItem * len(operands))()
    outs, keep = [], []
    for i, (dY, X) in enumerate(operands):
        rows, nout = dY.shape
        kin = X.shape[1]
        dW = torch.full((nout, kin), float("nan"), device="cuda")
        db = torch.full((nout,), float("nan"), device="cuda")
        part = torch.empty(max(1, lib.rd_linear_wgrad_partial_bytes(rows, nout, kin) // 4), device="cuda")
        it = items[i]
        it.d_out, it.x, it.rows, it.out_features, it.in_features = dY.data_ptr(), X.data_ptr(), rows, nout, kin
        it.d_weight, it.d_bias, it.partial = dW.data_ptr(), db.data_ptr(), part.data_ptr()
        outs.append((dW, db))
        keep.append(part)
    os.environ["RD_TC_WGRAD_BN"] = str(bn)
    try:
        L.check(lib.rd_linear_wgrad_group(items, len(operands), L.stream_ptr()), "rd_linear_wgrad_group")
        torch.cuda.synchronize()
    finally:
        os.environ.pop("RD_TC_WGRAD_BN", None)
    return outs


def same_bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("bn", WIDTHS)
def test_unaligned_bases_match_aligned(bn):
    from raindrop_b200 import lib as L
    lib = L.load()
    g = torch.Generator().manual_seed(11)
    aligned = [(torch.randn(r, n, generator=g).cuda(), torch.randn(r, k, generator=g).cuda()) for r, n, k in SHAPES]
    shifted = [(offset_copy(dY, 4 + 8 * (i % 4)), offset_copy(X, 28 - 8 * (i % 4))) for i, (dY, X) in enumerate(aligned)]
    for dY, X in shifted:
        assert dY.data_ptr() % 16 == 0 and dY.data_ptr() % 128 != 0
        assert X.data_ptr() % 16 == 0 and X.data_ptr() % 128 != 0
    ref = run(lib, L, aligned, bn)
    got = run(lib, L, shifted, bn)
    for (dY, X), (dW, db), (rW, rb) in zip(aligned, got, ref):
        assert same_bits(dW, rW) and same_bits(db, rb), (bn, tuple(dW.shape))
        full = dY.double().T @ X.double()
        assert ((dW.double() - full).norm() / full.norm()).item() < 2e-5, (bn, tuple(dW.shape))
        bsum = dY.double().sum(0)
        assert ((db.double() - bsum).norm() / bsum.norm()).item() < 2e-5, (bn, tuple(dW.shape))
