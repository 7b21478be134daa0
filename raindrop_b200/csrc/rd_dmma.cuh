// DMMA (mma.sync m16n8k16 f64) tiles of 64 x 64 fp64 outputs from fp32 operands staged to shared memory as fp64, shared
// by the TRAK Gram and rotation (rd_trak.cu) and the kNN-Shapley similarities (rd_valuation.cu).  Products of fp32 inputs
// are exact in fp64, and every output element of a launch sums its k-blocks in the same order.
#pragma once

#include "rd_tc_common.cuh"

namespace rd {
namespace {

constexpr int TK_TILE = 64, TK_BK = 32, TK_THREADS = 128;
constexpr int TK_LD = TK_TILE + 8;                 // doubles per staged row: a fragment's 4 k-rows land 16 banks apart
constexpr int TK_OPERAND = TK_BK * TK_LD;          // doubles of one staged operand [k][m]
constexpr int TK_STAGE = 2 * TK_OPERAND;
constexpr int TK_SMEM = 2 * TK_STAGE * 8;          // bytes: two stages
constexpr int TK_OUT_LD = TK_TILE + 1;             // the Gram tile's staging rows (column reads conflict-free)
static_assert(TK_TILE * TK_OUT_LD <= 2 * TK_STAGE, "the Gram tile is staged in the operand buffers");

__device__ __forceinline__ void dmma16816(double (&d)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
      "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
      : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

// One k-block of a 64 x 64 tile from staged operands sA[k][m], sB[k][n].  Warp w owns rows 32 (w & 1) + [0, 32) and
// columns 32 (w >> 1) + [0, 32).  Fragments (m16n8k16 f64): a_i = A(g + 8 (i & 1), t + 4 (i >> 1)), b_i = B(t + 4 i, g),
// c = C(g, 2t), C(g, 2t + 1), C(g + 8, 2t), C(g + 8, 2t + 1).
__device__ __forceinline__ void tk_mma_block(const double* sA, const double* sB, int warp, int lane,
                                             double (&acc)[2][4][4]) {
  const int g = lane >> 2, t = lane & 3, m0 = (warp & 1) * 32, n0 = (warp >> 1) * 32;
#pragma unroll
  for (int ks = 0; ks < TK_BK; ks += 16) {
    double a[2][8], b[4][4];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int i = 0; i < 8; ++i) a[mi][i] = sA[(ks + t + 4 * (i >> 1)) * TK_LD + m0 + 16 * mi + g + 8 * (i & 1)];
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int i = 0; i < 4; ++i) b[ni][i] = sB[(ks + t + 4 * i) * TK_LD + n0 + 8 * ni + g];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) dmma16816(acc[mi][ni], a[mi], b[ni]);
  }
}

// The k-block pipeline shared by both kernels: Load(kb) fetches k-block kb into registers, Store(stage) writes them to
// the stage's operands.  The next k-block's global loads are in flight while the current one multiplies.
template <typename Load, typename Store>
__device__ __forceinline__ void tk_mainloop(double* smem, int k_blocks, Load load, Store store, double (&acc)[2][4][4]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[mi][ni][e] = 0.0;
  load(0);
  store(smem);
  __syncthreads();
  for (int kb = 0; kb < k_blocks; ++kb) {
    double* cur = smem + (kb & 1) * TK_STAGE;
    if (kb + 1 < k_blocks) load(kb + 1);
    tk_mma_block(cur, cur + TK_OPERAND, warp, lane, acc);
    if (kb + 1 < k_blocks) store(smem + ((kb + 1) & 1) * TK_STAGE);
    __syncthreads();
  }
}

}  // namespace
}  // namespace rd
