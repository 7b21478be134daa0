"""GPU: tc_nt_kernel's epilogue at every tile width with every epilogue of the mode.

The epilogue runs in chunks of 8-column groups whose global loads and dropout draws are issued before the chunk's
stores; the chunk length depends on the flags and the tile width (nt_epi_chunk in rd_tc_gemm.cu), so each (flags,
width) pair has its own chunk boundaries.  The dropout lanes t and t^1 draw one Philox block each, for rows 8 (t & 1)
of their pair, and swap the keep bits.  Each case is checked element by element against the float64 product and
epilogue (the bounds of test_gemm_operators), and the keep bits exactly, at
  * M = 196: the last 64-row half of the second tile holds rows 192 .. 195 only, so in its first warp some lanes' row
    + 8 is past M while row is not (one lane of a dropout pair draws, the other does not);
  * N = 2 BN + 4 in three tiles: the last tile holds 4 columns, a tail inside its first chunk, and the keep-bit bytes
    past N are zeroed by that tile (the tile widths 48, 80, 120, 136, 152, 184 and 232 are not multiples of 32).
"""
import pytest
import torch

from test_gemm_operators import (EXACT_WIDTHS, F_DROP, F_PERM, F_REP, FAST_WIDTHS, NT_CASES, flag_name, operands,
                                 run_tc_nt)

pytestmark = pytest.mark.gpu

CASES = [(f, e, bn) for f, e in NT_CASES for bn in (EXACT_WIDTHS if e else FAST_WIDTHS)]


@pytest.mark.parametrize("flags,exact,bn", CASES,
                         ids=["%s-%s-%d" % (flag_name(f), "exact" if e else "fast", bn) for f, e, bn in CASES])
def test_tc_nt_epilogue_every_width(flags, exact, bn):
    M, K = 196, 24
    N = 2 * bn + 4
    A, B = operands(M, N, K, K + 4, False, exact, seed=flags * 7 + bn)
    bias = torch.randn(N, device="cuda", generator=torch.Generator(device="cuda").manual_seed(bn))
    run_tc_nt(A, B, K, exact, flags, bias, BN=bn, n_tiles=3, p=0.4 if flags & F_DROP else 0.25,
              perm=(4, 49) if flags & F_PERM else None, rep=(49, 196) if flags & F_REP else None,
              name="tc_nt %s %s width %d M%d N%d" % (flag_name(flags), "exact" if exact else "fast", bn, M, N))
