// Tensor-core GEMMs on Hopper (sm_90a).
//
// tc_nt: C = epi(A . B^T), A [M, K] and B [N, K] both row-major ("K-major").  It serves the encoder projections
// (code/models_rd.py:232-237,358 -> nn.TransformerEncoder) and their input gradients in error-compensated form, and the
// observation-propagation layer (rd_obprop_tc.cu) in single-pass or error-compensated form.  One persistent CTA per SM:
//   warpgroup 2   TMA producer (one thread): A tile [128 x 32] and B tile [BN x 32] (+ its precomputed remainder B_lo)
//                 per k-block into a <= 4-stage ring of 128B-swizzled shared memory, one mbarrier per stage and
//                 direction.  It hands its registers to the MMA warpgroups (setmaxnreg 40 / 232).
//   warpgroups    0 and 1, rows 0-63 and 64-127 of the tile: one wgmma.m64nBNk8 TF32 per k-step and term across the
//                 whole tile width (BN a template parameter), A from REGISTERS and B from shared memory, fp32
//                 accumulators in registers (BN / 2 per thread).  A is split into hi = top 19 bits and lo = the exact
//                 remainder in registers, so the error-compensated mode needs no remainder image of the activations:
//                 every k-step issues lo.hi + hi.lo + hi.hi.  One wgmma group stays in flight while the A fragments of
//                 the next k-block are loaded into a second register buffer.  The epilogue (bias,
//                 relu, row scale, gate, dropout + keep bits, residual, TF32 rounding, permuted store) runs on the
//                 accumulator registers and stores straight to global memory; meanwhile the producer already fills
//                 the ring for the next tile.
//
// tc_wgrad_group: dW = dY^T X (+ db) for up to WG_MAX problems in one launch.  Both operands are activations whose
// contraction index runs over their ROWS; wgmma's TF32 form only reads K-major operands from shared memory, so dY^T is
// gathered into registers from a row-major stage, and X is transposed in shared memory by a producer warpgroup into the
// K-major swizzled image wgmma reads (tc_wgrad_kernel below); both arrive by TMA several k-blocks ahead.  A fixed-order
// split-K reduce follows.
#include <stdlib.h>

#include "rd_tc_common.cuh"
#include "rd_tc_gemm.cuh"
#include "rd_wgmma_tf32.cuh"

namespace rd {
using namespace tc;
namespace {

constexpr int BM = 128, BK = 32, MAX_STAGES = 4;
constexpr int NT_THREADS = 384;            // warpgroups 0, 1: MMA + epilogue; warpgroup 2: TMA producer
constexpr int A_TILE = BM * BK * 4;        // 16 KB
constexpr int MAX_BN = 160;                // weight gradients: widest n tile

// F_REP: dropout of replicate-major rows (rep_remap), instantiated only with F_DROP for the Monte Carlo dropout forward
enum : int { F_RELU = 1, F_SCALE = 2, F_GATE = 4, F_DROP = 8, F_RESID = 16, F_ROUND = 32, F_PERM = 64, F_REP = 128 };

struct NtP {
  long long M; int N, K, n_tiles, m_tiles, k_blocks, nstages;
  float* C; long long ldc;
  const float* bias;
  const float* scale; int scale_mod;
  const float* gate; long long gate_ld; float gate_scale;
  float drop_p; const uint64_t* rng; uint32_t drop_site; DropRep rep;
  uint32_t* drop_mask; int drop_mask_ld;
  const float* resid; long long resid_ld;
  int pB, pN, pD;
  unsigned long long* dbg;     // optional %globaltimer stamps [CTA][8] (rd_debug_gemm_timing, slots in tc_nt_kernel)
};

__device__ __forceinline__ void gstamp(const NtP& p, int slot) {
  if (p.dbg) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    p.dbg[(size_t)blockIdx.x * 8 + slot] = t;
  }
}

__device__ __forceinline__ float lds_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}

// 8-column groups per epilogue chunk: the registers a group holds across the chunk (bias 2, gate 4, residual 4, keep
// bits and the Philox state 7, 2 more with the replicate rows' keys) beside the BN / 2 accumulators, within a budget
// fitted to ptxas's allocation
__host__ __device__ constexpr int nt_epi_chunk(int F, int BN) {
  const int per_group = 2 + 4 * !!(F & F_GATE) + 4 * !!(F & F_RESID) + 7 * !!(F & F_DROP) + 2 * !!(F & F_REP);
  const int jc = (128 - BN / 2) / per_group;
  return jc > 8 ? 8 : (jc < 2 ? 2 : jc);
}

// one k-block: per 8-wide k-step one wgmma across the whole tile width per term, small terms first (lo.hi, hi.lo, hi.hi)
template <int BN, bool EXACT>
__device__ __forceinline__ void issue_kblock(float (&acc)[BN / 2], const uint32_t (&ah)[BK / 8][4],
                                             const uint32_t (&al)[BK / 8][4], uint32_t sb, uint32_t b_tile) {
#pragma unroll
  for (int e = 0; e < BN / 2; ++e) fence_operand(acc[e]);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < BK / 8; ++ks) {
    const uint32_t bo = sb + (uint32_t)ks * 32u;
    const uint64_t bh = wgmma_desc_sw128(bo);
    if (EXACT) {
      wgmma_tf32<BN>(acc, al[ks], bh);
      wgmma_tf32<BN>(acc, ah[ks], wgmma_desc_sw128(bo + b_tile));
    }
    wgmma_tf32<BN>(acc, ah[ks], bh);
  }
  wgmma_commit();
}

// A fragments of one k-block from the swizzled stage, split into hi / lo in the error-compensated mode
template <bool EXACT>
__device__ __forceinline__ void load_afrag(uint32_t sa, int arow, int t, uint32_t (&ah)[BK / 8][4], uint32_t (&al)[BK / 8][4]) {
#pragma unroll
  for (int ks = 0; ks < BK / 8; ++ks) {
    const int col = ks * 8 + t;
    const float x0 = lds_f32(sa + sw128_offset(arow, col)), x1 = lds_f32(sa + sw128_offset(arow + 8, col));
    const float x2 = lds_f32(sa + sw128_offset(arow, col + 4)), x3 = lds_f32(sa + sw128_offset(arow + 8, col + 4));
    if (EXACT) {
      ah[ks][0] = tf32_hi(x0); ah[ks][1] = tf32_hi(x1); ah[ks][2] = tf32_hi(x2); ah[ks][3] = tf32_hi(x3);
      al[ks][0] = tf32_lo(x0); al[ks][1] = tf32_lo(x1); al[ks][2] = tf32_lo(x2); al[ks][3] = tf32_lo(x3);
    } else {   // single pass: the producers keep these operands TF32-representable
      ah[ks][0] = __float_as_uint(x0); ah[ks][1] = __float_as_uint(x1);
      ah[ks][2] = __float_as_uint(x2); ah[ks][3] = __float_as_uint(x3);
    }
  }
}

template <int F, bool EXACT, int BN>
__global__ void __launch_bounds__(NT_THREADS, 1)
tc_nt_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
             const __grid_constant__ CUtensorMap tmBlo, const NtP p) {
  // %globaltimer stamps when p.dbg is set, per CTA: 5 entry, 0 after the grid dependency wait, 1 the first full stage
  // seen by MMA thread 0, 2 its last wgmma retired, 3 / 4 the epilogue end of warpgroup 0 / 1, 7 the end of thread 0
  extern __shared__ uint8_t smem_raw[];
  if (threadIdx.x == 0) gstamp(p, 5);
  pdl_launch_dependents();
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr uint32_t b_tile = (uint32_t)BN * 128u;
  constexpr uint32_t stage_bytes = (uint32_t)A_TILE + (EXACT ? 2u : 1u) * b_tile;     // A | B hi [| B lo]
  const uint32_t bar_base = base + (uint32_t)p.nstages * stage_bytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (MAX_STAGES + s); };

  if (warp == 8 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    if (EXACT) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmBlo) : "memory");
    for (int s = 0; s < MAX_STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();          // everything above is private to this CTA; the previous kernel's output is first touched below
  if (threadIdx.x == 0) gstamp(p, 0);
  const int total_tiles = p.m_tiles * p.n_tiles;

  if (warp >= 8) {
    // ===== TMA producer ==========================================================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 8 && lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int m_t = tile / p.n_tiles, n_t = tile - m_t * p.n_tiles;
        for (int kb = 0; kb < p.k_blocks; ++kb) {
          mbar_wait(empty_bar(stage), phase ^ 1u);
          mbar_expect_tx(full_bar(stage), stage_bytes);
          const uint32_t sa = base + (uint32_t)stage * stage_bytes;
          tma_load_2d(&tmA, full_bar(stage), sa, kb * BK, m_t * BM);
          tma_load_2d(&tmB, full_bar(stage), sa + A_TILE, kb * BK, n_t * BN);
          if (EXACT) tma_load_2d(&tmBlo, full_bar(stage), sa + A_TILE + b_tile, kb * BK, n_t * BN);
          if (++stage == p.nstages) { stage = 0; phase ^= 1u; }
        }
      }
    }
    return;
  }

  // ===== warpgroups 0, 1: MMA and epilogue ========================================================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  const int wg = warp >> 2, wq = warp & 3, g = lane >> 2, t = lane & 3;
  const int arow = wg * 64 + wq * 16 + g;              // tile-local row of fragment elements a0 / a2
  const float ik = p.drop_p > 0.f ? 1.f / (1.f - p.drop_p) : 1.f;
  const RngKey key = load_rng_key((F & F_DROP) ? p.rng : nullptr);
  int stage = 0, rstage = 0; uint32_t phase = 0;
  // the next full stage -> A fragments; returns the stage's B tile address
  auto acquire = [&](uint32_t (&ah)[BK / 8][4], uint32_t (&al)[BK / 8][4]) {
    mbar_wait(full_bar(stage), phase);
    const uint32_t sa = base + (uint32_t)stage * stage_bytes;
    load_afrag<EXACT>(sa, arow, t, ah, al);
    if (++stage == p.nstages) { stage = 0; phase ^= 1u; }
    return sa + (uint32_t)A_TILE;
  };
  // the oldest stage still held: every wgmma that read it has retired
  auto release = [&]() {
    __syncwarp();
    if (lane == 0) mbar_arrive(empty_bar(rstage));
    if (++rstage == p.nstages) rstage = 0;
  };
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int m_t = tile / p.n_tiles, n_t = tile - m_t * p.n_tiles;
    float acc[BN / 2];
#pragma unroll
    for (int e = 0; e < BN / 2; ++e) acc[e] = 0.f;
    // k-blocks in pairs over two register buffers of A fragments: while the group of k-block kb runs, the fragments of
    // kb + 1 are loaded and split into the other buffer (its previous group retired at the wait<1> before)
    uint32_t ah0[BK / 8][4], al0[BK / 8][4], ah1[BK / 8][4], al1[BK / 8][4];
    uint32_t sb0 = acquire(ah0, al0), sb1 = 0;
    if (threadIdx.x == 0 && tile == blockIdx.x) gstamp(p, 1);
    for (int kb = 0; kb < p.k_blocks; kb += 2) {
      issue_kblock<BN, EXACT>(acc, ah0, al0, sb0, b_tile);
      wgmma_wait<1>();
      if (kb > 0) release();
      if (kb + 1 >= p.k_blocks) break;
      sb1 = acquire(ah1, al1);
      issue_kblock<BN, EXACT>(acc, ah1, al1, sb1, b_tile);
      wgmma_wait<1>();
      release();
      if (kb + 2 < p.k_blocks) sb0 = acquire(ah0, al0);
    }
    wgmma_wait<0>();
#pragma unroll
    for (int e = 0; e < BN / 2; ++e) fence_operand(acc[e]);
    release();
    if (threadIdx.x == 0) gstamp(p, 2);

    // ---- epilogue on the accumulator registers: element (row0 + 8i, col0 + 8j + 2t + {0, 1}) ----
    const long long row0 = (long long)m_t * BM + arow;
    const int col0 = n_t * BN;
    RngKey rkey[2] = {key, key};      // replicate rows: key and B-row index of column 0 of this thread's two rows
    uint64_t rbase[2] = {0, 0};
    if (F & F_REP) {
#pragma unroll
      for (int i = 0; i < 2; ++i) rbase[i] = rep_remap(p.rng, p.rep, (uint32_t)(row0 + 8 * i), (uint64_t)p.N, 0, &rkey[i]);
    }
    float sc[2] = {1.f, 1.f};
    if (F & F_SCALE) {
#pragma unroll
      for (int i = 0; i < 2; ++i) sc[i] = row0 + 8 * i < p.M ? __ldg(p.scale + ((row0 + 8 * i) % p.scale_mod)) : 0.f;
    }
    // In chunks of JC 8-column groups: first every global load of the chunk (bias, gate, residual) and its dropout
    // draws, then the arithmetic and the stores.  The compiler keeps a load after any store that may alias it, so with
    // loads and stores interleaved per group every group cost one memory round trip.  JC is as many groups as fit
    // next to the accumulators in the 168 registers ptxas allocates for this launch shape (no spills at any width).
    constexpr int NJ = BN / 8;
    constexpr int JC = nt_epi_chunk(F, BN);
#pragma unroll
    for (int j0 = 0; j0 < NJ; j0 += JC) {
      float2 bv[JC], gv[JC][2], rv[JC][2];
      uint32_t keep2[JC][2];     // keep bits of this lane's two columns, per row
#pragma unroll
      for (int jj = 0; jj < JC && j0 + jj < NJ; ++jj) {
        const int col = col0 + 8 * (j0 + jj) + 2 * t;
        const bool col_ok = col < p.N;               // N even, col even: the pair is all in or all out
        // plain loads, not ld.global.nc: a non-coherent load may be scheduled after the chunk's stores, and ptxas
        // sinks it to its use there, which brings back one round trip per group
        bv[jj] = make_float2(0.f, 0.f);
        if (p.bias && col_ok) bv[jj] = make_float2(p.bias[col], p.bias[col + 1]);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const long long row = row0 + 8 * i;
          const bool ok = col_ok && row < p.M;
          if (F & F_GATE) gv[jj][i] = ok ? *reinterpret_cast<const float2*>(p.gate + row * p.gate_ld + col) : make_float2(0.f, 0.f);
          if (F & F_RESID) rv[jj][i] = ok ? *reinterpret_cast<const float2*>(p.resid + row * p.resid_ld + col) : make_float2(0.f, 0.f);
        }
        if (F & F_DROP) {
          // element index row*N + col (or through the replicate rows); N % 4 == 0, so lanes t and t^1 share the Philox
          // block of their 4-column group in each of their two rows.  Lane t draws the block of row 8 (t & 1) only and
          // hands its partner the keep bits of the partner's two columns: same block, word and decision per element.
          const int ir = t & 1;             // the row this lane draws; its own columns are words 2 ir, 2 ir + 1
          const long long row = row0 + 8 * ir;
          uint32_t own = 0u, other = 0u;
          if (col_ok && row < p.M) {
            const uint64_t idx = (F & F_REP) ? rbase[ir] + (uint64_t)col : (uint64_t)row * (uint64_t)p.N + (uint64_t)col;
            const uint4 u = dropout_block((F & F_REP) ? rkey[ir] : key, p.drop_site, idx);
            const uint32_t lo = (keep_scale(u.x, p.drop_p, ik) > 0.f ? 1u : 0u) | (keep_scale(u.y, p.drop_p, ik) > 0.f ? 2u : 0u);
            const uint32_t hi = (keep_scale(u.z, p.drop_p, ik) > 0.f ? 1u : 0u) | (keep_scale(u.w, p.drop_p, ik) > 0.f ? 2u : 0u);
            own = ir ? hi : lo;
            other = ir ? lo : hi;
          }
          keep2[jj][ir] = own;
          keep2[jj][ir ^ 1] = __shfl_xor_sync(0xffffffffu, other, 1);
        }
      }
#pragma unroll
      for (int jj = 0; jj < JC && j0 + jj < NJ; ++jj) {
        const int j = j0 + jj;
        const int col = col0 + 8 * j + 2 * t;
        const bool col_ok = col < p.N;
        uint32_t bits[2] = {0u, 0u};
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const long long row = row0 + 8 * i;
          const bool ok = col_ok && row < p.M;
          float v0 = acc[4 * j + 2 * i] + bv[jj].x, v1 = acc[4 * j + 2 * i + 1] + bv[jj].y;
          if (F & F_RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
          if (F & F_SCALE) { v0 *= sc[i]; v1 *= sc[i]; }
          if (!ok) continue;
          if (F & F_GATE) {   // backward: pass the gradient only where the forward output was positive
            v0 = gv[jj][i].x > 0.f ? v0 * p.gate_scale : 0.f;
            v1 = gv[jj][i].y > 0.f ? v1 * p.gate_scale : 0.f;
          }
          if (F & F_DROP) {
            v0 *= (keep2[jj][i] & 1u) ? ik : 0.f;
            v1 *= (keep2[jj][i] & 2u) ? ik : 0.f;
            bits[i] = keep2[jj][i];
          }
          if (F & F_RESID) { v0 += rv[jj][i].x; v1 += rv[jj][i].y; }
          if (F & F_ROUND) { v0 = rn_tf32(v0); v1 = rn_tf32(v1); }
          float* dst;
          if (F & F_PERM) {   // row = b*pN + n, col = tt*4 + k  ->  encoder input [T, B, D] (code/models_rd.py:338-341)
            const long long b = row / p.pN, n = row - b * p.pN;
            dst = p.C + ((long long)(col >> 2) * p.pB + b) * p.pD + n * 4 + (col & 3);
          } else {
            dst = p.C + row * p.ldc + col;
          }
          *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
        }
        if ((F & F_DROP) && p.drop_mask) {
          // the backward of the consumer (LayerNorm) reads these bits instead of regenerating the Philox stream.  Columns
          // 8j .. 8j+7 are one byte of the row's bit words (col0 % 8 == 0) and belong to this tile alone, so tiles that
          // share a word never write the same byte.  Bytes past N up to the word's end are written as zeros by the tile
          // holding column N - 1.
          const int cb = col0 + 8 * j;
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            uint32_t b8 = bits[i] << (2 * t);
            b8 |= __shfl_xor_sync(0xffffffffu, b8, 1);
            b8 |= __shfl_xor_sync(0xffffffffu, b8, 2);
            const long long row = row0 + 8 * i;
            if (t == 0 && row < p.M && cb < p.N) {
              uint8_t* w = reinterpret_cast<uint8_t*>(p.drop_mask + row * p.drop_mask_ld);
              w[cb >> 3] = (uint8_t)b8;
              if (cb + 8 >= p.N)
                for (int z = (cb >> 3) + 1; z < 4 * p.drop_mask_ld && z < 4 * ((p.N + 31) >> 5); ++z) w[z] = 0;
            }
          }
        }
      }
    }
    if ((threadIdx.x & 127) == 0) gstamp(p, 3 + wg);
  }
  if (threadIdx.x == 0) gstamp(p, 7);
}

// =================================================================================================
// weight-gradient kernel ("TN"), GROUPED: one launch serves up to WG_MAX independent problems
//   D_k[m, n] = sum_r A_k[r, m] * B_k[r, n]   (A = dY, B = X plus a "ones" column N for the bias gradient)
// over one row split of problem k per work item (problem, m tile, n tile, split).  A training step has ten of these
// (8 encoder weights + 2 lin_value).  Persistent: one CTA per SM walks the items blockIdx.x, + gridDim.x, ...
//   warpgroup 3   issuer: thread 384 alone sends each 32-row k-block's loads into its stage as soon as the MMA
//                 warpgroups release it, all by TMA (32 x 32 boxes, 128B swizzle): the raw X tile [32 x BN] into the
//                 stage's hi | lo region on the stage's xfull mbarrier, the dY tile [32 x 128] into the stage's dY region
//                 on its full mbarrier.  It does nothing else, so waiting for a release delays no transpose.
//   warpgroup 2   transposer, 128 threads.  When a k-block's X has landed, the X tile is read into registers and
//                 TRANSPOSED into the K-major 128B-swizzled images wgmma reads (sw128_offset(n, r)) as hi = top 19 bits
//                 and lo = exact remainder, one 16-byte store per 4 rows of one column, with the ones column written
//                 here (TMA cannot synthesise it).  fence.proxy.async, then arrive.
//   warpgroups    0 and 1: dW rows 0-63 and 64-127 of the tile, one wgmma.m64nBNk8 per k-step and term (lo.hi, hi.lo,
//                 hi.hi) with A = dY^T gathered from the swizzled row-major stage (a transposed gather is addressing) and split in
//                 registers, exactly the tc_nt_kernel pipeline (one group in flight, two A-fragment buffers, a stage is
//                 released only after the group that read it retired).  A warpgroup whose 64 rows lie past M waits and
//                 releases the stages without MMAs.  Partial tiles go to slab [split][M][Nld] (Nld = N + 1 rounded up to 4).
// The tile width BN is a template parameter, one per launch (wgrad_plan picks it for the whole group): with several
// widths dispatched per item inside one kernel, ptxas serialises the wgmma for lack of registers (C7512).
// =================================================================================================
struct WP {
  float* partial;                    // [nsplit][M][Nld]; dY and X arrive through WGroup::tmY / tmX
  int rows, M, N, Nld, n_tiles, m_tiles, nsplit, rows_per_split;
  int item0;                         // first work item of this problem inside the grouped list
};
struct WGroup {
  CUtensorMap tmX[WG_MAX];           // X of problem k: dims {Kin, rows}, boxes of 32 columns x 32 rows, 128B swizzle
  CUtensorMap tmY[WG_MAX];           // dY of problem k: dims {Nout, rows}, boxes of 32 columns x 32 rows, 128B swizzle
  WP it[WG_MAX]; int n, total_items;
  unsigned long long* dbg;           // optional per-CTA phase cycles [CTA][16] (rd_debug_wgrad_timing)
};

// Phase timing of one CTA, clock64 deltas summed in registers and written once at the end when WGroup::dbg is set.
// Slots: 0 / 1 clock64 at the start (after the grid dependency wait) / end of MMA thread 0; 3 / 4 transposing thread
// 256's cycles waiting for its X tile / transposing and storing; 5 / 6 MMA thread 0's cycles waiting for a full stage /
// in the slab-store epilogue; 7 %globaltimer ns from start to end (the clock rate); 8 the k-blocks the CTA transposed;
// 9 clock64 at thread 256's end; 11 / 12 the issuing thread's cycles waiting for an empty stage / issuing the loads of a
// released stage; 13 clock64 at the issuing thread's end.  Slots 2 and 10 are unused: the transposing warps neither
// wait for releases nor issue loads.
__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

constexpr int W_THREADS = 512;            // warpgroups 0, 1: MMA; warpgroup 2: transposer; warpgroup 3: issuer
constexpr int WA_TILE = BK * BM * 4;      // 16 KB: 32 rows of dY x 128 columns
// ring stage: dY tile | X^T hi | X^T lo; as many stages (<= MAX_STAGES) as fit next to the barriers and the alignment slack
__host__ __device__ constexpr int w_stage_bytes(int bn) { return WA_TILE + 2 * bn * 128; }
__host__ __device__ constexpr int w_nstages(int bn) { return (SMEM_LIMIT - 1280) / w_stage_bytes(bn) < MAX_STAGES ? (SMEM_LIMIT - 1280) / w_stage_bytes(bn) : MAX_STAGES; }

// Tile widths the weight-gradient kernel is instantiated for (multiples of 8 up to MAX_BN)
#define RD_WG_WIDTHS(X) X(32) X(64) X(96) X(128) X(144) X(160)

__device__ __forceinline__ void sts_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

struct WItem { int pi, n_t, m_t, split, k_blocks, r_begin, r_end; };
__device__ __forceinline__ WItem wgrad_item(const WGroup& g, int w) {
  WItem it;
  it.pi = 0;
#pragma unroll 1
  for (int k = 1; k < g.n; ++k) if (w >= g.it[k].item0) it.pi = k;
  const WP& p = g.it[it.pi];
  const int item = w - p.item0;
  it.n_t = item % p.n_tiles; it.m_t = (item / p.n_tiles) % p.m_tiles; it.split = item / (p.n_tiles * p.m_tiles);
  it.r_begin = it.split * p.rows_per_split;
  it.r_end = min(p.rows, it.r_begin + p.rows_per_split);
  it.k_blocks = (it.r_end - it.r_begin + BK - 1) / BK;
  return it;
}

struct WRing {
  uint32_t base, stage_bytes, bar_base, phase = 0;
  int nstages, stage = 0, rstage = 0;
  __device__ uint32_t full(int s) const { return bar_base + 8u * s; }
  __device__ uint32_t empty(int s) const { return bar_base + 8u * (MAX_STAGES + s); }
  __device__ uint32_t xfull(int s) const { return bar_base + 8u * (2 * MAX_STAGES + s); }    // the stage's raw X tile
  __device__ uint32_t addr(int s) const { return base + (uint32_t)s * stage_bytes; }
};

// one item on MMA warpgroup `wg`: k-blocks -> accumulators -> this split's slab; adds its cycles waiting for full stages
// to t_full and in the epilogue to t_epi
template <int BN>
__device__ __forceinline__ void wgrad_consume(const WP& p, const WItem& it, WRing& q, int wg, int arow, int t,
                                              long long& t_full, long long& t_epi) {
  constexpr uint32_t b_tile = (uint32_t)BN * 128u;
  auto release = [&]() {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(q.empty(q.rstage));
    if (++q.rstage == q.nstages) q.rstage = 0;
  };
  if (it.m_t * BM + wg * 64 >= p.M) {      // this warpgroup's rows are all padding: pass the stages through
    for (int kb = 0; kb < it.k_blocks; ++kb) {
      mbar_wait(q.full(q.stage), q.phase);
      if (++q.stage == q.nstages) { q.stage = 0; q.phase ^= 1u; }
      release();
    }
    return;
  }
  // The dY stage holds four TMA boxes of 32 rows x 32 columns m, 128B-swizzled: (r, m) at 4096 (m >> 5) +
  // sw128_offset(r, m % 32), bank 4 ((((m % 32) >> 2) ^ r) & 7) + m % 4.  Lane (g, t) gathers m = arow + g (+8) at
  // r = 8 ks + t (+4); arow % 32 = 16 w + g with w = wq % 2, and arow, arow + 8 share a box.  Read in the order
  // (r, r + 4), the chunk index (4w + g/4 (+2)) ^ (t (+4)) would take 4 values over a warp (2-way conflicts).  So the
  // lanes with g >= 4 (h = 1) read row r + 4 first: the chunk of the first load is (4w + h) ^ (t + 4h), whose bits are
  // (h ^ t0, t1, w ^ h), a bijection of (h, t0, t1); with g % 4 as the word inside the chunk, 32 distinct banks.  The
  // other three loads flip bit 1 (m + 8) and / or bit 2 (the other row), also bijections.  Selects put the values back.
  const int h = (arow >> 2) & 1;
  const uint32_t mbox = 4096u * (uint32_t)(arow >> 5);
  const int mm = arow & 31, ra = t + 4 * h, rb = t + 4 - 4 * h;
  const uint32_t o0 = mbox + sw128_offset(ra, mm), o1 = mbox + sw128_offset(ra, mm + 8);
  const uint32_t o2 = mbox + sw128_offset(rb, mm), o3 = mbox + sw128_offset(rb, mm + 8);
  auto acquire = [&](uint32_t (&ah)[BK / 8][4], uint32_t (&al)[BK / 8][4]) {
    const long long c0 = clock64();
    mbar_wait(q.full(q.stage), q.phase);
    t_full += clock64() - c0;
    const uint32_t sa = q.addr(q.stage);
#pragma unroll
    for (int ks = 0; ks < BK / 8; ++ks) {
      const uint32_t sk = sa + 1024u * ks;     // rows + 8 ks: the swizzle depends on r % 8 only
      const float v0 = lds_f32(sk + o0), v1 = lds_f32(sk + o1), v2 = lds_f32(sk + o2), v3 = lds_f32(sk + o3);
      const float x0 = h ? v2 : v0, x1 = h ? v3 : v1, x2 = h ? v0 : v2, x3 = h ? v1 : v3;
      ah[ks][0] = tf32_hi(x0); ah[ks][1] = tf32_hi(x1); ah[ks][2] = tf32_hi(x2); ah[ks][3] = tf32_hi(x3);
      al[ks][0] = tf32_lo(x0); al[ks][1] = tf32_lo(x1); al[ks][2] = tf32_lo(x2); al[ks][3] = tf32_lo(x3);
    }
    if (++q.stage == q.nstages) { q.stage = 0; q.phase ^= 1u; }
    return sa + (uint32_t)WA_TILE;
  };
  float acc[BN / 2];
#pragma unroll
  for (int e = 0; e < BN / 2; ++e) acc[e] = 0.f;
  uint32_t ah0[BK / 8][4], al0[BK / 8][4], ah1[BK / 8][4], al1[BK / 8][4];
  uint32_t sb0 = acquire(ah0, al0), sb1 = 0;
  for (int kb = 0; kb < it.k_blocks; kb += 2) {
    issue_kblock<BN, true>(acc, ah0, al0, sb0, b_tile);
    wgmma_wait<1>();
    if (kb > 0) release();
    if (kb + 1 >= it.k_blocks) break;
    sb1 = acquire(ah1, al1);
    issue_kblock<BN, true>(acc, ah1, al1, sb1, b_tile);
    wgmma_wait<1>();
    release();
    if (kb + 2 < it.k_blocks) sb0 = acquire(ah0, al0);
  }
  wgmma_wait<0>();
#pragma unroll
  for (int e = 0; e < BN / 2; ++e) fence_operand(acc[e]);
  release();

  // element (row0 + 8i, col0 + 8j + {0, 1}); Nld % 4 == 0 and the column even: a pair is all in or all out
  const long long c0 = clock64();
  const int row0 = it.m_t * BM + arow, col0 = it.n_t * BN + 2 * t;
  float* slab = p.partial + (long long)it.split * p.M * p.Nld;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = col0 + 8 * j;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = row0 + 8 * i;
      if (col < p.Nld && row < p.M)
        *reinterpret_cast<float2*>(slab + (long long)row * p.Nld + col) = make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
    }
  }
  t_epi += clock64() - c0;
}

template <int BN>
__global__ void __launch_bounds__(W_THREADS, 1)
tc_wgrad_kernel(const __grid_constant__ WGroup g) {
  constexpr int NU = BN / 16;               // 4-row x 1-column chunks per producer thread and k-block
  constexpr int NBOX = (BN + 31) / 32;      // 32-column TMA boxes of X per k-block
  static_assert(BN % 16 == 0, "the transpose covers the tile in groups of 16 columns");
  static_assert(NBOX * 4096 <= 2 * BN * 128, "the raw X boxes land in the stage's hi | lo images");
  static_assert(w_nstages(BN) >= 3, "the consumers hold two stages; a third lets the producers run ahead");
  extern __shared__ uint8_t smem_raw[];
  pdl_launch_dependents();
  WRing q;
  q.base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  q.stage_bytes = (uint32_t)w_stage_bytes(BN);
  q.nstages = w_nstages(BN);
  q.bar_base = q.base + (uint32_t)(w_nstages(BN) * w_stage_bytes(BN));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 8 && lane == 0) {
    for (int k = 0; k < g.n; ++k) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&g.tmX[k]) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&g.tmY[k]) : "memory");
    }
    // full: the 128 transposing threads + the issuing thread's expect_tx for dY
    for (int s = 0; s < MAX_STAGES; ++s) { mbar_init(q.full(s), 129); mbar_init(q.empty(s), 8); mbar_init(q.xfull(s), 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();          // everything above is private to this CTA; the previous kernel's output is first touched below
  const long long clk0 = clock64();
  const unsigned long long gt0 = gtimer();
  unsigned long long* const dbg = g.dbg ? g.dbg + (size_t)blockIdx.x * 16 : nullptr;

  if (warp >= 12) {
    // ===== issuer warpgroup ========================================================================
    // Thread 384 alone walks the (item, k-block) sequence and sends each k-block's loads into its stage as soon as the
    // MMA warpgroups release it, all by TMA: X (NBOX boxes) on the stage's xfull barrier, then dY (four boxes of 32 rows
    // x 32 columns, 128B swizzle, see wgrad_consume) on its full barrier.  Only the ring bounds how far it runs ahead.
    // The work item is computed once per item: the walk over the group's problems reads kernel parameters at a register
    // index.
    asm volatile("setmaxnreg.dec.sync.aligned.u32 32;" ::: "memory");
    if (warp == 12 && lane == 0) {
      long long t_empty = 0, t_issue = 0;
      int stage = 0;
      uint32_t phase = 0;
      for (int w = blockIdx.x; w < g.total_items; w += gridDim.x) {
        const WItem it = wgrad_item(g, w);
        for (int kb = 0; kb < it.k_blocks; ++kb) {
          const long long c0 = clock64();
          mbar_wait(q.empty(stage), phase ^ 1u);
          const long long c1 = clock64();
          t_empty += c1 - c0;
          const uint32_t sa = q.addr(stage);
          const int r0 = it.r_begin + kb * BK;
          // rows past `rows`, columns past Kin and m past Nout arrive as zeros
          mbar_expect_tx(q.xfull(stage), NBOX * 4096u);
#pragma unroll
          for (int b = 0; b < NBOX; ++b)
            tma_load_2d(&g.tmX[it.pi], q.xfull(stage), sa + (uint32_t)WA_TILE + 4096u * b, it.n_t * BN + 32 * b, r0);
          mbar_expect_tx(q.full(stage), (uint32_t)WA_TILE);
#pragma unroll
          for (int b = 0; b < BM / 32; ++b)
            tma_load_2d(&g.tmY[it.pi], q.full(stage), sa + 4096u * b, it.m_t * BM + 32 * b, r0);
          if (++stage == q.nstages) { stage = 0; phase ^= 1u; }
          t_issue += clock64() - c1;
        }
      }
      if (dbg) { dbg[11] = t_empty; dbg[12] = t_issue; dbg[13] = clock64(); }
    }
    return;
  }

  if (warp >= 8) {
    // ===== transposer warpgroup ====================================================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 112;" ::: "memory");
    const int pt = threadIdx.x - 256, pw = warp - 8;
    const int total = g.total_items;
    long long t_x = 0, t_store = 0, n_kb = 0;
    // The raw X tile (NBOX boxes of 32 rows x 32 columns, 128B-swizzled, at the start of the
    // stage's hi image; (r, n) at 4096 (n >> 5) + sw128_offset(r, n % 32)) -> registers, with the ones column N of the
    // bias gradient set here -> the K-major images, one 16-byte store per chunk of rows 4a .. 4a + 3 of one image row n
    // (sw128_offset(n, 4a)) for hi and one for lo.  Lane = 8c + a, c = lane / 8, a = lane % 8, of warp pw holds, per
    // 16-column group i < BN / 16, column n = 16 i + 4 cq + c with cq = (a >> 1) ^ pw, rows 4a .. 4a + 3: over the four
    // warps every (n, a) of the group once.  It reads them with four scalar loads (no shuffles; as many shared-memory
    // wavefronts as one 16-byte load per row).
    //   load j (row 4a + j): chunk ((n % 32) >> 2) ^ (4a + j) = (4 (i % 2) + cq) ^ (4 (a % 2) + j), bits 0-1
    //     (a >> 1) ^ pw ^ j and bit 2 (i % 2) ^ (a % 2): a bijection of a; word c inside the chunk -> 32 banks.
    //   16-byte store: a quarter warp is one c and a = 0..7; the chunk (a ^ n) % 8 with n % 8 = 4 (cq % 2) + c has bits
    //     0-1 (a ^ c) % 4 and bit 2 a2 ^ a1 ^ pw0 ^ c2 (c2 = 0): a bijection of a -> 8 distinct chunks, conflict-free.
    const int a = lane & 7, c = lane >> 3, cq = (a >> 1) ^ pw;
    uint32_t ld_off[2][4];        // raw X: group i reads box i >> 1 at ld_off[i % 2][j]
#pragma unroll
    for (int e = 0; e < 2; ++e)
#pragma unroll
      for (int j = 0; j < 4; ++j) ld_off[e][j] = sw128_offset(4 * a + j, 16 * e + 4 * cq + c);
    const uint32_t st_off = sw128_offset(4 * cq + c, 4 * a);     // image: + 2048 i (16 rows of 128 bytes per group)
    int w = blockIdx.x, kb = 0;
    WItem it = wgrad_item(g, w);
    while (w < total) {
      const WP& p = g.it[it.pi];
      const long long c0 = clock64();
      mbar_wait(q.xfull(q.stage), q.phase);
      const long long c1 = clock64();
      const uint32_t sb = q.addr(q.stage) + (uint32_t)WA_TILE, sl = sb + (uint32_t)BN * 128u;
      const int r = it.r_begin + kb * BK + 4 * a, ones = p.N - it.n_t * BN - 4 * cq - c;     // ones: 16 i of column N
      float xv[NU][4];
#pragma unroll
      for (int i = 0; i < NU; ++i) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          xv[i][j] = lds_f32(sb + 4096u * (uint32_t)(i >> 1) + ld_off[i & 1][j]);
          if (16 * i == ones && r + j < it.r_end) xv[i][j] = 1.f;
        }
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");        // every raw read is done before the images overwrite it
#pragma unroll
      for (int i = 0; i < NU; ++i) {
        const uint32_t o = st_off + 2048u * i;
        sts_v4(sb + o, tf32_hi(xv[i][0]), tf32_hi(xv[i][1]), tf32_hi(xv[i][2]), tf32_hi(xv[i][3]));
        sts_v4(sl + o, tf32_lo(xv[i][0]), tf32_lo(xv[i][1]), tf32_lo(xv[i][2]), tf32_lo(xv[i][3]));
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy stores -> wgmma's reads
      mbar_arrive(q.full(q.stage));
      if (++q.stage == q.nstages) { q.stage = 0; q.phase ^= 1u; }
      t_x += c1 - c0; t_store += clock64() - c1; ++n_kb;
      if (++kb == it.k_blocks) {
        kb = 0; w += gridDim.x;
        if (w < total) it = wgrad_item(g, w);
      }
    }
    if (dbg && pt == 0) { dbg[3] = t_x; dbg[4] = t_store; dbg[8] = n_kb; dbg[9] = clock64(); }
    return;
  }

  // ===== warpgroups 0, 1: MMA ======================================================================
  // 128 x (2 x 184 + 112 + 32) = 65,536: the whole register file
  asm volatile("setmaxnreg.inc.sync.aligned.u32 184;" ::: "memory");
  const int wg = warp >> 2, wq = warp & 3, gq = lane >> 2, t = lane & 3;
  const int arow = wg * 64 + wq * 16 + gq;
  long long t_full = 0, t_epi = 0;
  for (int w = blockIdx.x; w < g.total_items; w += gridDim.x) {
    const WItem it = wgrad_item(g, w);
    wgrad_consume<BN>(g.it[it.pi], it, q, wg, arow, t, t_full, t_epi);
  }
  if (dbg && threadIdx.x == 0) {
    dbg[0] = clk0; dbg[1] = clock64(); dbg[5] = t_full; dbg[6] = t_epi; dbg[7] = gtimer() - gt0;
  }
}

// dW[m, n] = sum_s partial[s][m][n] (n < N), db[m] = sum_s partial[s][m][N]; fixed order -> deterministic.
// One launch for every problem of a group.
// kind 0: a weight gradient (above).  kind 1: plain column sums out[c] = sum_s partial[s*stride + c], c < N
// (the LayerNorm dgamma / dbeta partial rows ride along in the same launch).
struct RItem { const float* partial; float* dW; float* db; int nsplit, M, N, Mpad, Nld, kind; long long stride; long long start; };
constexpr int RG_MAX = WG_MAX + CS_MAX;
struct RGroup { RItem it[RG_MAX]; long long total; int n; };
__global__ void wgrad_reduce_kernel(const __grid_constant__ RGroup g) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.total) return;
  int k = 0;
#pragma unroll 1
  for (int j = 1; j < g.n; ++j) if (i >= g.it[j].start) k = j;
  const RItem& r = g.it[k];
  const long long e = i - r.start;
  if (r.kind == 1) {      // one warp per output column (item starts are multiples of 32): lanes stride over the chunks
    const long long col = e >> 5;
    const int lane = (int)(e & 31);
    const float* src = r.partial + col;
    float s = 0.f;
#pragma unroll 4
    for (int sp = lane; sp < r.nsplit; sp += 32) s += __ldg(src + sp * r.stride);
    s = warp_sum(s);        // fixed butterfly order: deterministic
    if (lane == 0) r.dW[col] = s;
    return;
  }
  // kind 0: one thread per four consecutive columns of a row (N % 4 == 0, slabs 16-byte aligned), plus one per row for
  // the bias column N
  const int q_per_row = (r.N >> 2) + 1;
  const int m = (int)(e / q_per_row), q = (int)(e - (long long)m * q_per_row);
  if (m >= r.M) return;       // padding between this item and the next (warp-aligned) one
  const long long stride = (long long)r.Mpad * r.Nld;
  if (q == (r.N >> 2)) {
    const float* src = r.partial + (long long)m * r.Nld + r.N;
    float s = 0.f;
#pragma unroll 4
    for (int sp = 0; sp < r.nsplit; ++sp) s += __ldg(src + sp * stride);
    if (r.db) r.db[m] = s;
    return;
  }
  const float* src = r.partial + (long long)m * r.Nld + 4 * q;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int sp0 = 0; sp0 < r.nsplit; sp0 += 8) {      // eight slabs in flight per round trip, summed in slab order
    float4 t[8];
#pragma unroll
    for (int u = 0; u < 8; ++u)
      t[u] = sp0 + u < r.nsplit ? __ldg(reinterpret_cast<const float4*>(src + (sp0 + u) * stride)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int u = 0; u < 8; ++u) { s.x += t[u].x; s.y += t[u].y; s.z += t[u].z; s.w += t[u].w; }
  }
  float* dst = r.dW + (long long)m * r.N + 4 * q;
  if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
    *reinterpret_cast<float4*>(dst) = s;
  } else {
    dst[0] = s.x; dst[1] = s.y; dst[2] = s.z; dst[3] = s.w;
  }
}

static const int kWgWidths[] = {
#define RD_WG_LIST(W) W,
    RD_WG_WIDTHS(RD_WG_LIST)
#undef RD_WG_LIST
};

// Row splits of one problem for a target of `rows_target` rows per split.  They depend on the shapes alone, never on the
// tile width, so every width computes each element of a split as the same product sequence (bitwise equal results).
// ~512 rows (16 k-blocks) per item so the pipeline amortises its fill, but never more than ~2 rounds of items per
// problem in 128 x 160 tiles (bounds the partial buffer for the big configurations).  512 sizes the partial buffers
// (the CAPACITY in row splits); wgrad_rows_target may raise it for a group, which only lowers the split count.
WSplit wgrad_split(int M, int N, long long rows, int rows_target = 512) {
  WSplit w;
  w.Nld = (int)round_up(N + 1, 4);                          // + the ones column
  const long long mn = ceil_div(M, BM) * ceil_div(N + 1, MAX_BN);
  long long ns = ceil_div(rows, rows_target);
  const long long cap = (2 * num_sms()) / mn > 1 ? (2 * num_sms()) / mn : 1;
  if (ns > cap) ns = cap;
  if (ns < 1) ns = 1;
  w.rows_per_split = (int)round_up(ceil_div(rows, ns), BK);
  w.nsplit = (int)ceil_div(rows, w.rows_per_split);
  return w;
}

// Rows per split of a group: the smallest target >= 512 (in steps of 32, up to 1024) for which the group's count of
// 128 x 160 work items fills whole waves of the SMs.  With the same splits (and per split the same k-block and k-step
// order of lo.hi, hi.lo, hi.hi) every weight gradient is bitwise the one the mma.sync kernel this one replaced gave.
int wgrad_rows_target(const WgradItem* items, int n) {
  auto count_items = [&](int target) {
    long long t = 0;
    for (int i = 0; i < n; ++i) {
      const WgradItem& a = items[i];
      t += (long long)wgrad_split(a.Nout, a.Kin, a.rows, target).nsplit * ceil_div(a.Nout, BM) * ceil_div(a.Kin + 1, MAX_BN);
    }
    return t;
  };
  const long long sms = num_sms(), t0 = count_items(512);
  if (t0 > sms && t0 % sms) {
    const long long goal = (t0 / sms) * sms;
    for (int t = 544; t <= 1024; t += 32)
      if (count_items(t) <= goal) return t;
  }
  return 512;
}

// Tile width of a group: the instantiated width that minimises the MMA work of the group's items, sum over items of
// rows x (width + a per-tile overhead of 32 columns: the dY tile is staged and gathered once per n tile), computed and
// padded columns alike; ties go to the wider tile (fewer n tiles).  RD_TC_WGRAD_BN=<width> forces a listed width
// (tests compare widths on the same problems).
int wgrad_width(const WgradItem* items, int n) {
  if (const char* e = getenv("RD_TC_WGRAD_BN")) {
    const int f = atoi(e);
    for (int bn : kWgWidths) if (bn == f) return f;         // not a listed width: ignored
  }
  int best_bn = MAX_BN;
  long long best = -1;
  for (int bn : kWgWidths) {
    long long cost = 0;
    for (int i = 0; i < n; ++i)
      cost += ceil_div(items[i].Nout, BM) * ceil_div(items[i].Kin + 1, bn) * items[i].rows * (bn + 32);
    if (best < 0 || cost <= best) { best = cost; best_bn = bn; }
  }
  return best_bn;
}

struct SplitItems { WeightSplit it[16]; long long start[17]; int n; StepPrologue pro; };

__global__ void split_weights_kernel(const __grid_constant__ SplitItems s) {
  pdl_launch_dependents();
  pdl_wait();
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) {     // step prologue riding along: dropout counter capture (+ advance) and ticket reset
    if (s.pro.rng_state) {
      s.pro.rng_captured[0] = s.pro.rng_state[0];
      s.pro.rng_captured[1] = s.pro.rng_state[1] + s.pro.step_offset;
      if (s.pro.advance) s.pro.rng_state[1] = s.pro.rng_state[1] + 1;
    }
    if (s.pro.zero_counter) *s.pro.zero_counter = 0u;
  }
  if (i >= s.start[s.n]) return;
  int t = 0;
  while (t + 1 < s.n && i >= s.start[t + 1]) ++t;
  const WeightSplit w = s.it[t];
  long long e = i - s.start[t];
  int r = (int)(e / w.cols), c = (int)(e - (long long)r * w.cols);
  float v = w.w[e];
  float lo = v - __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
  if (w.lo) w.lo[e] = lo;
  if (w.t) { w.t[(long long)c * w.rows + r] = v; w.t_lo[(long long)c * w.rows + r] = lo; }
  if (w.rn || w.rn_t) {
    const float rn = rn_tf32(v);
    if (w.rn) w.rn[e] = rn;
    if (w.rn_t) w.rn_t[(long long)c * w.rows + r] = rn;
  }
}

}  // namespace

// Tile widths tc_nt_kernel is instantiated for, each with every epilogue combination of its mode (RD_NT_WIDTHS_* below
// must list the same).  Error-compensated (encoder GEMMs, small ob-prop layers): fine steps around the P19 shapes
// (on 132 SMs tc_nt_plan picks 152 -> 2 x 80, 272 -> 2 x 136, 456 -> 2 x 232 at 7,680 rows, 240 -> 3 x 80 at 4,352);
// it stops at 232, where the accumulators and two A-fragment buffers still fit in registers.  Single pass (the
// HBM-bound ob-prop layers): the multiples of 32 from 64 up and 240, which serves C = 240 in one tile (the roofline
// size); PAM's C = 2400 at 4,352 rows gets 11 x 224.
#define RD_NT_WIDTHS_EXACT(X) X(48) X(80) X(96) X(120) X(136) X(152) X(184) X(232)
#define RD_NT_WIDTHS_FAST(X) X(64) X(96) X(128) X(160) X(192) X(224) X(240) X(256)
#define RD_NT_LIST(W) W,
static const int kNtWidthsExact[] = {RD_NT_WIDTHS_EXACT(RD_NT_LIST)};
static const int kNtWidthsFast[] = {RD_NT_WIDTHS_FAST(RD_NT_LIST)};
#undef RD_NT_LIST
template <typename Fn>
static int nt_first_width(bool exact, Fn&& pred) {
  if (exact) { for (int w : kNtWidthsExact) if (pred(w)) return w; }
  else { for (int w : kNtWidthsFast) if (pred(w)) return w; }
  return 0;
}
static bool nt_width_ok(int bn, bool exact) { return nt_first_width(exact, [&](int w) { return w == bn; }) != 0; }

void tc_nt_plan(long long M, int N, bool exact, int* BN, int* n_tiles) {
  // RD_TC_NT_BN=<width> forces the tile width (a listed one that covers N in at most 64 tiles; tests use it to run
  // every plan on the same problem)
  if (const char* e = getenv("RD_TC_NT_BN")) {
    const int bn = atoi(e);
    if (nt_width_ok(bn, exact) && ceil_div(N, bn) <= 64) { *BN = bn; *n_tiles = (int)ceil_div(N, bn); return; }
  }
  // Per-SM cost of a plan: the tiles of the busiest SM times their width plus a fixed per-tile overhead (pipeline
  // fill and epilogue), in columns.  Smallest cost wins; ties go to fewer n tiles (A is read once per n tile).  The
  // overhead of 32 columns is an estimate, not a measurement; the P19 plans above come out the same for any value
  // from 0 to 256.  BM stays 128: a 64-row tile would need its own producer schedule (or the two MMA warpgroups
  // working on different tiles, "ping-pong"), which this kernel does not have.
  const long long m_tiles = ceil_div(M, BM), sms = num_sms();
  constexpr long long TILE_OVERHEAD = 32;
  long long best = -1;
  for (int nt = 1; nt <= 64; ++nt) {
    const long long need = ceil_div(N, nt);
    const int bn = nt_first_width(exact, [&](int w) { return w >= need; });
    if (bn == 0 || ceil_div(N, bn) < nt) continue;     // too narrow, or a wider plan with empty tiles
    const long long cost = ceil_div(m_tiles * nt, sms) * (bn + TILE_OVERHEAD);
    if (best < 0 || cost < best) { best = cost; *BN = bn; *n_tiles = nt; }
  }
  if (best < 0) {      // wider than 64 of the widest tiles
    *BN = exact ? kNtWidthsExact[sizeof(kNtWidthsExact) / sizeof(int) - 1] : kNtWidthsFast[sizeof(kNtWidthsFast) / sizeof(int) - 1];
    *n_tiles = (int)ceil_div(N, *BN);
  }
}

// the instantiation of tile width `bn` (one of the mode's listed widths; tc_nt checked it)
template <int F, bool EX, typename L>
static int nt_launch(int bn, L&& launch) {
#define RD_NT_WIDTH(W) case W: return launch(tc_nt_kernel<F, EX, W>);
  if constexpr (EX) {
    switch (bn) { RD_NT_WIDTHS_EXACT(RD_NT_WIDTH) default: break; }
  } else {
    switch (bn) { RD_NT_WIDTHS_FAST(RD_NT_WIDTH) default: break; }
  }
#undef RD_NT_WIDTH
  set_error("tc_nt: tile width %d not instantiated", bn);
  return -2;
}

static unsigned long long* g_gemm_dbg = nullptr;
void tc_gemm_set_debug(unsigned long long* buf) { g_gemm_dbg = buf; }

int tc_nt(const TcNtArgs& a, cudaStream_t st) {
  const bool exact = a.B_lo != nullptr;
  if (!nt_width_ok(a.BN, exact) || a.n_tiles < 1 || (long long)a.BN * a.n_tiles < a.N || a.M < 1 || a.M > 0x7fffffffLL ||
      a.K % 4 || a.N % 4 || a.lda % 4) {
    set_error("tc_nt: unsupported tiling / shape (M=%lld N=%d K=%d BN=%d)", a.M, a.N, a.K, a.BN);
    return -2;
  }
  if ((reinterpret_cast<uintptr_t>(a.A) | reinterpret_cast<uintptr_t>(a.B) | reinterpret_cast<uintptr_t>(a.B_lo) |
       reinterpret_cast<uintptr_t>(a.C) | reinterpret_cast<uintptr_t>(a.gate) | reinterpret_cast<uintptr_t>(a.resid)) & 15) {
    set_error("tc_nt: pointers must be 16-byte aligned");
    return -2;
  }
  // the epilogue reads gate and resid as float2, writes keep-bit bytes up to column N - 1 and divides by the perm sizes
  if ((a.gate && a.gate_ld % 2) || (a.resid && a.resid_ld % 2) || (a.drop_p > 0.f && !a.rng) ||
      (a.drop_p > 0.f && a.rep.B && a.rep.Bc < 1) || (a.drop_mask && 32LL * a.drop_mask_ld < a.N) ||
      (a.perm && (a.pB < 1 || a.pN < 1 || a.pD < 1))) {
    set_error("tc_nt: bad epilogue (odd gate_ld / resid_ld, dropout without rng, replicate rows Bc=%d, keep-bit ld %d "
              "for N=%d or perm sizes)", a.rep.Bc, a.drop_mask_ld, a.N);
    return -2;
  }
  NtP p;
  p.M = a.M; p.N = a.N; p.K = a.K; p.n_tiles = a.n_tiles;
  p.m_tiles = (int)ceil_div(a.M, BM);
  p.k_blocks = (int)ceil_div(a.K, BK);
  const int stage_bytes = A_TILE + (exact ? 2 : 1) * a.BN * 128;
  const int fixed = 1024 + 256;
  p.nstages = (SMEM_LIMIT - fixed) / stage_bytes;
  if (p.nstages > MAX_STAGES) p.nstages = MAX_STAGES;
  if (p.nstages < 2) { set_error("tc_nt: not enough shared memory"); return -2; }
  const int smem_bytes = fixed + p.nstages * stage_bytes;
  p.C = a.C; p.ldc = a.N;
  p.bias = a.bias; p.scale = a.scale; p.scale_mod = a.scale_mod > 0 ? a.scale_mod : 1;
  p.gate = a.gate; p.gate_ld = a.gate_ld; p.gate_scale = a.gate_scale;
  p.drop_p = a.drop_p; p.rng = a.rng; p.drop_site = a.drop_site; p.drop_mask = a.drop_mask; p.drop_mask_ld = a.drop_mask_ld;
  p.rep = a.rep;
  p.resid = a.resid; p.resid_ld = a.resid_ld;
  p.pB = a.pB; p.pN = a.pN; p.pD = a.pD;
  p.dbg = g_gemm_dbg;

  const int f = (a.relu ? F_RELU : 0) | (a.scale ? F_SCALE : 0) | (a.gate ? F_GATE : 0) | (a.drop_p > 0.f ? F_DROP : 0) |
                (a.resid ? F_RESID : 0) | (a.round_out ? F_ROUND : 0) | (a.perm ? F_PERM : 0) |
                (a.drop_p > 0.f && a.rep.B ? F_REP : 0);
  // the tensor maps and the device queries come after every argument check (an uninstantiated epilogue included)
  auto launch = [&](auto kern) -> int {
    CUtensorMap tmA, tmB, tmBlo;
    {
      cuuint64_t d[2] = {(cuuint64_t)a.K, (cuuint64_t)a.M};
      cuuint64_t s[1] = {(cuuint64_t)a.lda * 4};
      cuuint32_t b[2] = {BK, BM};
      RD_TRY(encode(&tmA, a.A, 2, d, s, b, CU_TENSOR_MAP_SWIZZLE_128B, "A"));
    }
    {
      cuuint64_t d[2] = {(cuuint64_t)a.K, (cuuint64_t)a.N};
      cuuint64_t s[1] = {(cuuint64_t)a.K * 4};
      cuuint32_t b[2] = {BK, (cuuint32_t)a.BN};
      RD_TRY(encode(&tmB, a.B, 2, d, s, b, CU_TENSOR_MAP_SWIZZLE_128B, "B"));
      if (exact) RD_TRY(encode(&tmBlo, a.B_lo, 2, d, s, b, CU_TENSOR_MAP_SWIZZLE_128B, "B_lo"));
      else tmBlo = tmB;
    }
    const int total = p.m_tiles * p.n_tiles;
    const int grid = total < num_sms() ? total : num_sms();
    RD_TRY(ensure_max_smem((const void*)kern, SMEM_LIMIT));   // once per (instantiation, device)
    launch_pdl(kern, dim3(grid), dim3(NT_THREADS), smem_bytes, st, tmA, tmB, tmBlo, p);
    return 0;
  };
  int rc = -2;
#define RD_NT_CASE(FLAGS, EX) \
  if (f == (FLAGS) && exact == (EX)) rc = nt_launch<(FLAGS), (EX)>(a.BN, launch); else
  // observation propagation: layer 2 -> encoder input, layer 1 (rounded for the next single-pass layer), the plain
  // operator, backward d(input); encoder: bias[,relu][,dropout][,residual] forward, [gate][,residual] backward
  RD_NT_CASE(F_PERM | F_RELU | F_SCALE, false)
  RD_NT_CASE(F_RELU | F_SCALE | F_ROUND, false)
  RD_NT_CASE(F_RELU | F_SCALE, false)
  RD_NT_CASE(F_GATE | F_SCALE, false)
  RD_NT_CASE(F_PERM | F_RELU | F_SCALE, true)
  RD_NT_CASE(F_RELU | F_SCALE, true)
  RD_NT_CASE(F_GATE | F_SCALE, true)
  RD_NT_CASE(0, true)
  RD_NT_CASE(F_RESID, true)
  RD_NT_CASE(F_DROP, true)
  RD_NT_CASE(F_DROP | F_RESID, true)
  RD_NT_CASE(F_GATE, true)
  RD_NT_CASE(F_RELU, true)
  RD_NT_CASE(F_RELU | F_DROP, true)
  RD_NT_CASE(F_DROP | F_RESID | F_REP, true)       // Monte Carlo dropout replicates: dropout1, dropout2, the FFN
  RD_NT_CASE(F_RELU | F_DROP | F_REP, true)
  { set_error("tc_nt: epilogue combination %d (exact=%d) not instantiated", f, (int)exact); return -2; }
#undef RD_NT_CASE
  if (rc != 0) return rc;
  RD_CHECK_LAUNCH("tc_nt_kernel");
  return 0;
}

bool tc_gemm_supported(const TcGemmArgs& a) {
  static int env = -1;
  if (env < 0) { const char* e = getenv("RD_TC_GEMM"); env = (e && e[0] == '0') ? 0 : 1; }
  if (env != 1) return false;
  if (a.K % 4 || a.N % 4 || a.lda % 4 || a.K < 8 || a.N < 16 || a.M < 1 || a.M > 0x7fffffffLL) return false;
  if ((a.gate && a.gate_ld % 4) || (a.resid && a.resid_ld % 4)) return false;
  uintptr_t bits = reinterpret_cast<uintptr_t>(a.A) | reinterpret_cast<uintptr_t>(a.B) | reinterpret_cast<uintptr_t>(a.B_lo) |
                   reinterpret_cast<uintptr_t>(a.C) | reinterpret_cast<uintptr_t>(a.gate) | reinterpret_cast<uintptr_t>(a.resid);
  const int id = (a.relu ? 8 : 0) | (a.gate ? 4 : 0) | (a.drop_p > 0.f ? 2 : 0) | (a.resid ? 1 : 0);
  const bool combo = id == 0 || id == 1 || id == 2 || id == 3 || id == 4 || id == 8 || id == 10;
  return combo && (bits & 15) == 0 && a.B_lo != nullptr;
}

int tc_gemm(const TcGemmArgs& a, cudaStream_t st) {
  if (!tc_gemm_supported(a)) { set_error("tc_gemm: unsupported shape/alignment (M=%lld N=%d K=%d)", a.M, a.N, a.K); return -2; }
  TcNtArgs n;
  n.A = a.A; n.lda = a.lda; n.B = a.B; n.B_lo = a.B_lo; n.M = a.M; n.N = a.N; n.K = a.K; n.C = a.C;
  tc_nt_plan(a.M, a.N, true, &n.BN, &n.n_tiles);
  n.bias = a.bias; n.relu = a.relu; n.gate = a.gate; n.gate_ld = a.gate_ld; n.gate_scale = a.gate_scale;
  n.drop_p = a.drop_p; n.rng = a.rng; n.drop_site = a.drop_site; n.rep = a.rep; n.drop_mask = a.drop_mask; n.drop_mask_ld = a.drop_mask_ld;
  n.resid = a.resid; n.resid_ld = a.resid_ld;
  return tc_nt(n, st);
}

bool tc_wgrad_supported(int Nout, int Kin, long long ldy, long long ldx, const void* dY, const void* X) {
  static int env = -1;
  if (env < 0) { const char* e = getenv("RD_TC_WGRAD"); env = (e && e[0] == '0') ? 0 : 1; }
  if (env != 1) return false;
  if (Nout % 4 || Kin % 4 || ldy % 4 || ldx % 4 || Nout < 16 || Kin < 16) return false;
  return ((reinterpret_cast<uintptr_t>(dY) | reinterpret_cast<uintptr_t>(X)) & 15) == 0;
}

long long tc_wgrad_partial_floats(int Nout, int Kin, long long rows) {
  const WSplit w = wgrad_split(Nout, Kin, rows);
  return round_up((long long)w.nsplit * Nout * w.Nld, 64);
}

static unsigned long long* g_wgrad_dbg = nullptr;
void tc_wgrad_set_debug(unsigned long long* buf) { g_wgrad_dbg = buf; }

// The group's plan: one rows target, each problem's row split under it, one tile width
static WgradPlan wgrad_plan(const WgradItem* items, int n) {
  WgradPlan pl;
  pl.rows_target = n > 0 ? wgrad_rows_target(items, n) : 512;
  pl.BN = n > 0 ? wgrad_width(items, n) : 0;
  for (int i = 0; i < n; ++i) pl.sp[i] = wgrad_split(items[i].Nout, items[i].Kin, items[i].rows, pl.rows_target);
  return pl;
}

int tc_wgrad_group(const WgradItem* items, int n, const ColsumItem* cs, int ncs, cudaStream_t st, WgradPlan* plan) {
  if (n <= 0 && ncs <= 0) return 0;
  if (n > WG_MAX || ncs > CS_MAX) { set_error("tc_wgrad_group: at most %d problems (+ %d column sums) per launch", WG_MAX, CS_MAX); return -2; }
  WGroup g;
  RGroup r;
  g.n = n; r.n = n + (ncs > 0 ? ncs : 0);
  g.dbg = g_wgrad_dbg;
  const WgradPlan pl = wgrad_plan(items, n > 0 ? n : 0);
  const WSplit* sp = pl.sp;
  int order[WG_MAX];
  long long tot = 0;
  for (int i = 0; i < n; ++i) {
    const WgradItem& a = items[i];
    if (!tc_wgrad_supported(a.Nout, a.Kin, a.ldy, a.ldx, a.dY, a.X) || !a.partial || a.rows < 1 ||
        (reinterpret_cast<uintptr_t>(a.partial) & 15)) {
      set_error("tc_wgrad_group: problem %d has an unsupported shape/alignment", i);
      return -2;
    }
    if (a.rows > 0x7fffffffLL) { set_error("tc_wgrad_group: too many rows"); return -2; }
    const WSplit& w = sp[i];
    order[i] = i;
    RItem& q = r.it[i];
    q.partial = a.partial; q.dW = a.dW; q.db = a.db; q.nsplit = w.nsplit; q.M = a.Nout; q.N = a.Kin; q.Mpad = a.Nout; q.Nld = w.Nld;
    q.kind = 0; q.stride = 0;
    q.start = tot;
    tot += (long long)a.Nout * (a.Kin / 4 + 1);
  }
  const int BN = pl.BN;
  // the persistent grid deals the items round robin: problems with the longest items (rows per split) go first
  for (int i = 1; i < n; ++i)
    for (int j = i; j > 0 && sp[order[j]].rows_per_split > sp[order[j - 1]].rows_per_split; --j) {
      const int t = order[j]; order[j] = order[j - 1]; order[j - 1] = t;
    }
  int item = 0;
  for (int k = 0; k < n; ++k) {
    const WgradItem& a = items[order[k]];
    const WSplit& w = sp[order[k]];
    WP& p = g.it[k];
    p.partial = a.partial;
    p.rows = (int)a.rows; p.M = a.Nout; p.N = a.Kin; p.Nld = w.Nld;
    {
      cuuint64_t d[2] = {(cuuint64_t)a.Kin, (cuuint64_t)a.rows};
      cuuint64_t s[1] = {(cuuint64_t)a.ldx * 4};
      cuuint32_t b[2] = {BK, BK};
      RD_TRY(encode(&g.tmX[k], a.X, 2, d, s, b, CU_TENSOR_MAP_SWIZZLE_128B, "X"));
      cuuint64_t dy[2] = {(cuuint64_t)a.Nout, (cuuint64_t)a.rows};
      cuuint64_t sy[1] = {(cuuint64_t)a.ldy * 4};
      RD_TRY(encode(&g.tmY[k], a.dY, 2, dy, sy, b, CU_TENSOR_MAP_SWIZZLE_128B, "dY"));
    }
    p.n_tiles = (int)ceil_div(a.Kin + 1, BN); p.m_tiles = (int)ceil_div(a.Nout, BM);
    p.nsplit = w.nsplit; p.rows_per_split = w.rows_per_split;
    p.item0 = item;
    item += w.nsplit * p.m_tiles * p.n_tiles;
  }
  g.total_items = item;
  for (int i = 0; i < ncs; ++i) {
    RItem& q = r.it[n + i];
    q.partial = cs[i].partial; q.dW = cs[i].out; q.db = nullptr; q.nsplit = cs[i].nsplit; q.M = 1; q.N = cs[i].ncols;
    q.Mpad = 1; q.Nld = 0; q.kind = 1; q.stride = cs[i].stride;
    tot = round_up(tot, 32);                 // warp-aligned: 32 threads per output column
    q.start = tot;
    tot += 32LL * cs[i].ncols;
  }
  r.total = tot;
  if (n > 0) {
    const int smem_bytes = 1280 + w_nstages(BN) * w_stage_bytes(BN);
    const int grid = item < num_sms() ? item : num_sms();
    auto launch = [&](auto kern) -> int {
      RD_TRY(ensure_max_smem((const void*)kern, SMEM_LIMIT));
      launch_pdl(kern, dim3(grid), dim3(W_THREADS), smem_bytes, st, g);
      return 0;
    };
    int rc = -2;
    switch (BN) {
#define RD_WG_CASE(W) case W: rc = launch(tc_wgrad_kernel<W>); break;
      RD_WG_WIDTHS(RD_WG_CASE)
#undef RD_WG_CASE
      default: break;
    }
    if (rc != 0) { set_error("tc_wgrad_group: tile width %d not instantiated", BN); return -2; }
    RD_CHECK_LAUNCH("tc_wgrad_kernel");
  }
  launch_pdl(wgrad_reduce_kernel, dim3((unsigned)ceil_div(tot, 256)), dim3(256), 0, st, r);
  RD_CHECK_LAUNCH("wgrad_reduce_kernel");
  if (plan) *plan = pl;
  return 0;
}

int tc_wgrad(const float* dY, long long ldy, const float* X, long long ldx, long long rows, int Nout, int Kin,
             float* dW, float* db, float* partial, cudaStream_t st) {
  WgradItem it{dY, ldy, X, ldx, rows, Nout, Kin, dW, db, partial};
  return tc_wgrad_group(&it, 1, nullptr, 0, st);
}

int split_weights(const WeightSplit* items, int n, cudaStream_t st, const StepPrologue* pro) {
  if (n <= 0 && !pro) return 0;
  if (n > 16) { set_error("split_weights: at most 16 tensors per launch"); return -2; }
  SplitItems s;
  s.n = n; s.start[0] = 0;
  for (int i = 0; i < n; ++i) { s.it[i] = items[i]; s.start[i + 1] = s.start[i] + (long long)items[i].rows * items[i].cols; }
  s.pro = pro ? *pro : StepPrologue{};
  const long long total = s.start[n] > 0 ? s.start[n] : 1;
  launch_pdl(split_weights_kernel, dim3((unsigned)ceil_div(total, 256)), dim3(256), 0, st, s);
  RD_CHECK_LAUNCH("split_weights_kernel");
  return 0;
}

}  // namespace rd
