"""GPU: how the grouped weight-gradient launch folds its row splits into dW / db.

Each work item of tc_wgrad_kernel stores one row split of one (m tile, n tile) into that split's partial slab, and the
group's split sums add the slabs of each element in split order.  This file checks that the fold depends on nothing
but the operands:
  * the same group launched again and again on the same partial buffers, eagerly and as a captured CUDA graph replayed
    three times, gives the bits of the first launch every time (the outputs are overwritten with NaN in between, so
    each launch writes every element);
  * a group whose problems have a single row split (the tile's own slab is the whole sum) next to problems with 12 or
    more splits gives the same bits under every tile width, every element within its componentwise bound of an fp64
    product (test_wgrad_operators.check_public).
"""
import os

import pytest
import torch

from test_wgrad_operators import check_public

pytestmark = pytest.mark.gpu

WIDTHS = [32, 64, 96, 128, 144, 160]


def make(shapes, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(r, n, generator=g).cuda(), torch.randn(r, k, generator=g).cuda()) for r, n, k in shapes]


class Group:
    """one rd_linear_wgrad_group call over fixed operands, outputs and partial buffers"""

    def __init__(self, operands):
        from raindrop_b200 import lib as L
        self.L, self.lib = L, L.load()
        self.items = (L.RdWgradItem * len(operands))()
        self.outs, self.keep = [], []
        for i, (dY, X) in enumerate(operands):
            rows, nout = dY.shape
            kin = X.shape[1]
            assert rows >= 256                      # below, the library uses the CUDA-core path instead
            dW, db = torch.empty(nout, kin, device="cuda"), torch.empty(nout, device="cuda")
            part = torch.empty(max(1, self.lib.rd_linear_wgrad_partial_bytes(rows, nout, kin) // 4), device="cuda")
            it = self.items[i]
            it.d_out, it.x, it.rows, it.out_features, it.in_features = dY.data_ptr(), X.data_ptr(), rows, nout, kin
            it.d_weight, it.d_bias, it.partial = dW.data_ptr(), db.data_ptr(), part.data_ptr()
            self.outs.append((dW, db))
            self.keep.append(part)
        self.n = len(operands)

    def poison(self):
        for dW, db in self.outs:
            dW.fill_(float("nan"))
            db.fill_(float("nan"))

    def launch(self):
        self.L.check(self.lib.rd_linear_wgrad_group(self.items, self.n, self.L.stream_ptr()), "rd_linear_wgrad_group")

    def snapshot(self):
        torch.cuda.synchronize()
        return [(dW.clone(), db.clone()) for dW, db in self.outs]


def same_bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def assert_same(got, ref, tag):
    for (a, b), (c, d) in zip(got, ref):
        assert same_bits(a, c) and same_bits(b, d), (tag, tuple(a.shape))


def test_repeated_launches_eager_and_graph():
    ops = make([(7680, 152, 272), (7680, 456, 152), (4352, 240, 240), (300, 64, 36)], seed=11)
    grp = Group(ops)
    grp.poison()
    grp.launch()
    first = grp.snapshot()
    check_public(ops, first, "fold first")
    for k in range(3):
        grp.poison()
        grp.launch()
        assert_same(grp.snapshot(), first, "eager %d" % k)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):            # warm-up off the default stream before capture, as torch recommends
        grp.launch()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        grp.launch()
    for k in range(3):
        grp.poison()
        graph.replay()
        assert_same(grp.snapshot(), first, "replay %d" % k)


def test_single_split_next_to_many_splits_every_width():
    # 300 and 512 rows: one split per tile; 16384 and 12288 rows on small tiles: 16 to 32 splits of 512 - 1024 rows
    shapes = [(300, 200, 152), (16384, 64, 60), (512, 132, 100), (12288, 96, 36), (8192, 128, 128)]
    ops = make(shapes, seed=3)
    ref = Group(ops)
    ref.launch()
    ref_out = ref.snapshot()
    check_public(ops, ref_out, "fold default")
    for bn in WIDTHS:
        os.environ["RD_TC_WGRAD_BN"] = str(bn)
        try:
            grp = Group(ops)
            grp.poison()
            grp.launch()
            got = grp.snapshot()
        finally:
            os.environ.pop("RD_TC_WGRAD_BN", None)
        assert_same(got, ref_out, bn)
