// Random projection of per-sample gradient rows (TracIn-RP, rd_grad_projection).
//
// out[r, m] = (1/sqrt(dim)) sum_s sum_{j in seg_s} G[r, j] Omega(seed, j, m), Omega = +-1 drawn from Philox4x32-10 as a
// function of (seed, absolute column j, dimension m) alone (proj_block / proj_sign; the mapping is in the header).  The
// rows go on the wgmma N side and the projection dimensions on M, so a launch of a few rows wastes no M tile:
//   grad_proj_kernel         one CTA per (128 dimensions, 64 rows, segment).  Warp 8: one TMA thread fills a 6-stage ring
//                            with the rows' tile [64 x 32] and the same tile of their remainder image (psg_lo_kernel),
//                            for each 32-column k-block of the segment; k-blocks start at absolute multiples of 32
//                            columns.  Warpgroups 0 and 1: dimensions 0-63 and 64-127.  The A fragments (Omega^T) are drawn
//                            in registers, one Philox block per (dimension, 128 columns) feeding 32 fragment elements, and
//                            are 0 outside the segment.  Two wgmma.m64n64k8 TF32 per k-step (Omega.lo, then Omega.hi):
//                            Omega is exact in TF32, so the split of G alone compensates.  Each k-block goes to fresh
//                            accumulators that the CUDA cores add in order (as psg_dot_kernel does); the segment's fp32
//                            sum goes to partial[seg][r][m].
//   grad_proj_reduce_kernel  out[r, m] = fp32((1/sqrt(dim)) * (the segments' sums added in order in fp64)).
// The instruction shape, the k-block order and the tile of a row's dimensions do not depend on `rows`, and no value
// crosses between the columns of a wgmma's N side, so every output row is bitwise independent of the other rows.
#include <math.h>
#include <stdlib.h>

#include "rd_tc_common.cuh"
#include "rd_influence.cuh"
#include "rd_wgmma_tf32.cuh"

namespace rd {
using namespace tc;
namespace {

constexpr int GP_BM = 128, GP_BN = 64, GP_BK = 32, GP_STAGES = 6, GP_THREADS = 384;
constexpr int GP_TILE = GP_BN * GP_BK * 4;       // 8 KB: the rows' k-block, raw then remainder
constexpr int GP_STAGE = 2 * GP_TILE;
constexpr int GP_SMEM = 1024 + GP_STAGES * GP_STAGE + 256;

// The Philox block of dimension m and columns [128 jb, 128 jb + 128): column j is bit (j & 31) of word (j >> 5) & 3
__device__ __forceinline__ uint4 proj_block(uint32_t k0, uint32_t k1, uint64_t jb, uint32_t m) {
  return philox4(k0, k1, (uint32_t)jb, (uint32_t)(jb >> 32), m, 0u);
}
__device__ __forceinline__ uint32_t proj_word(const uint4& w, int q) {
  return q == 0 ? w.x : (q == 1 ? w.y : (q == 2 ? w.z : w.w));
}
// TF32 / fp32 bits of Omega from bit b of x: 0 -> +1, 1 -> -1
__device__ __forceinline__ uint32_t proj_sign(uint32_t x, int b) { return 0x3F800000u | (((x >> b) & 1u) << 31); }

// A fragments of one k-block: dimension m0 (word x0) and m0 + 8 (word x1), k-block columns b = 8 ks + t (+ 4); columns
// outside [lo, hi) (relative to the k-block) are 0
__device__ __forceinline__ void gp_afrag(uint32_t x0, uint32_t x1, int t, int lo, int hi, uint32_t (&a)[GP_BK / 8][4]) {
#pragma unroll
  for (int ks = 0; ks < GP_BK / 8; ++ks) {
    const int b = ks * 8 + t;
    const bool v0 = b >= lo && b < hi, v1 = b + 4 >= lo && b + 4 < hi;
    a[ks][0] = v0 ? proj_sign(x0, b) : 0u;
    a[ks][1] = v0 ? proj_sign(x1, b) : 0u;
    a[ks][2] = v1 ? proj_sign(x0, b + 4) : 0u;
    a[ks][3] = v1 ? proj_sign(x1, b + 4) : 0u;
  }
}

__device__ __forceinline__ void gp_issue(float (&acc)[GP_BN / 2], const uint32_t (&a)[GP_BK / 8][4], uint32_t sb) {
#pragma unroll
  for (int e = 0; e < GP_BN / 2; ++e) fence_operand(acc[e]);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < GP_BK / 8; ++ks) {
    const uint32_t bo = sb + (uint32_t)ks * 32u;
    wgmma_tf32<GP_BN>(acc, a[ks], wgmma_desc_sw128(bo + GP_TILE));   // small terms first
    wgmma_tf32<GP_BN>(acc, a[ks], wgmma_desc_sw128(bo));
  }
  wgmma_commit();
}

__global__ void __launch_bounds__(GP_THREADS, 1)
grad_proj_kernel(const __grid_constant__ CUtensorMap tmG, const __grid_constant__ CUtensorMap tmGlo,
                 const long long* __restrict__ seg, int rows, int dim, uint32_t k0, uint32_t k1, float* __restrict__ partial) {
  extern __shared__ uint8_t smem_raw[];
  pdl_launch_dependents();
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const TmaRing<GP_STAGES> ring{base + (uint32_t)GP_STAGES * GP_STAGE};
  const int m_t = blockIdx.x, r_t = blockIdx.y, z = blockIdx.z;

  if (warp == 8 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmG) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmGlo) : "memory");
    ring.init(8);
  }
  __syncthreads();
  pdl_wait();
  const long long off = seg[2 * z], end = off + seg[2 * z + 1];
  const long long c_first = off & ~31LL;
  const int k_blocks = (int)((end - c_first + GP_BK - 1) / GP_BK);

  if (warp >= 8) {
    // ===== TMA producer ==========================================================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 8 && lane == 0) {
      RingPos<GP_STAGES> p;
      for (int kb = 0; kb < k_blocks; ++kb) {
        const int stage = ring.produce(p, GP_STAGE);
        const uint32_t sa = base + (uint32_t)stage * GP_STAGE;
        const int col = (int)(c_first + (long long)kb * GP_BK);
        tma_load_2d(&tmG, ring.full(stage), sa, col, r_t * GP_BN);
        tma_load_2d(&tmGlo, ring.full(stage), sa + GP_TILE, col, r_t * GP_BN);
      }
    }
    return;
  }

  // ===== warpgroups 0, 1: Omega, MMA and epilogue ====================================================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  const int wg = warp >> 2, wq = warp & 3, g = lane >> 2, t = lane & 3;
  const uint32_t m0 = (uint32_t)(m_t * GP_BM + wg * 64 + wq * 16 + g);
  RingPos<GP_STAGES> cpos, rpos;
  int next = 0;
  uint4 w0 = make_uint4(0u, 0u, 0u, 0u), w1 = w0;
  // draws the next k-block's A fragments (a new Philox block at every 128-column boundary) while its tiles land
  auto acquire = [&](uint32_t (&a)[GP_BK / 8][4]) {
    const long long c0 = c_first + (long long)next * GP_BK;
    if (next == 0 || (c0 & 127) == 0) {
      w0 = proj_block(k0, k1, (uint64_t)c0 >> 7, m0);
      w1 = proj_block(k0, k1, (uint64_t)c0 >> 7, m0 + 8);
    }
    const int q = (int)(c0 >> 5) & 3;
    gp_afrag(proj_word(w0, q), proj_word(w1, q), t, (int)(off - c0), (int)(end - c0), a);
    ++next;
    return base + (uint32_t)ring.consume(cpos) * GP_STAGE;
  };
  auto release = [&]() { ring.release(rpos, lane); };
  float acc[GP_BN / 2], a0[GP_BN / 2], a1[GP_BN / 2];
#pragma unroll
  for (int e = 0; e < GP_BN / 2; ++e) { acc[e] = 0.f; a0[e] = 0.f; a1[e] = 0.f; }
  auto fold = [&](float (&a)[GP_BN / 2]) {
#pragma unroll
    for (int e = 0; e < GP_BN / 2; ++e) { fence_operand(a[e]); acc[e] += a[e]; a[e] = 0.f; }
  };
  uint32_t f0[GP_BK / 8][4], f1[GP_BK / 8][4];
  uint32_t sb0 = acquire(f0), sb1 = 0;
  for (int kb = 0; kb < k_blocks; kb += 2) {
    gp_issue(a0, f0, sb0);
    wgmma_wait<1>();
    if (kb > 0) { release(); fold(a1); }          // k-block kb - 1 has retired
    if (kb + 1 >= k_blocks) break;
    sb1 = acquire(f1);
    gp_issue(a1, f1, sb1);
    wgmma_wait<1>();
    release();
    fold(a0);                                     // k-block kb has retired
    if (kb + 2 < k_blocks) sb0 = acquire(f0);
  }
  wgmma_wait<0>();
  release();
  if (k_blocks & 1) fold(a0); else fold(a1);

  // element (dimension m0 + 8i, row 8j + 2t + c of the tile)
#pragma unroll
  for (int j = 0; j < GP_BN / 8; ++j)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int r = r_t * GP_BN + 8 * j + 2 * t + c;
        if (r < rows) partial[((long long)z * rows + r) * dim + m0 + 8 * i] = acc[4 * j + 2 * i + c];
      }
}

__global__ void grad_proj_reduce_kernel(const float* __restrict__ partial, int n_seg, int rows, int dim, double scale,
                                        float* __restrict__ out, long long ldo) {
  pdl_launch_dependents();
  pdl_wait();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)rows * dim) return;
  const int r = (int)(idx / dim), m = (int)(idx % dim);
  double s = 0.0;
  for (int z = 0; z < n_seg; ++z) s += (double)partial[((long long)z * rows + r) * dim + m];
  out[(long long)r * ldo + m] = (float)(scale * s);
}

__global__ void proj_signs_kernel(uint32_t k0, uint32_t k1, long long col0, int n_cols, int dim, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)n_cols * dim) return;
  const uint64_t j = (uint64_t)(col0 + idx / dim);
  const uint32_t m = (uint32_t)(idx % dim);
  out[idx] = __uint_as_float(proj_sign(proj_word(proj_block(k0, k1, j >> 7, m), (int)(j >> 5) & 3), (int)(j & 31)));
}

struct ProjLayout { int64_t lo, seg, partial, total; };     // floats
ProjLayout proj_layout(int rows, int64_t ldg, int dim, int n_seg) {
  ProjLayout l;
  l.lo = 0;
  l.seg = round_up((int64_t)rows * ldg, 64);
  l.partial = l.seg + round_up(4LL * n_seg, 64);
  l.total = l.partial + (int64_t)n_seg * rows * dim;
  return l;
}

bool proj_dim_ok(int32_t dim) { return dim >= 128 && dim <= 32768 && dim % GP_BM == 0; }

}  // namespace
}  // namespace rd

using namespace rd;

extern "C" {

size_t rd_grad_projection_scratch_bytes(int32_t rows, int64_t ldg, int32_t dim, int32_t n_seg) {
  if (rows < 1 || ldg < 1 || !proj_dim_ok(dim) || n_seg < 1) return 0;
  return (size_t)proj_layout(rows, ldg, dim, n_seg).total * sizeof(float);
}

int rd_grad_projection(const float* G, int32_t rows, int64_t ldg, const int64_t* seg_off, const int64_t* seg_len,
                       int32_t n_seg, int32_t dim, uint64_t seed, float* out, int64_t ldo, void* scratch, void* stream) {
  const char* fn = "rd_grad_projection";
  if (!G || !seg_off || !seg_len || !out || !scratch) { set_error("%s: NULL argument", fn); return -2; }
  if (rows < 1 || ldg < 4 || (ldg & 3) || ldg > 0x7fffffffLL - 64 || n_seg < 1 || n_seg > 65535 || !proj_dim_ok(dim) ||
      ldo < dim || ceil_div(rows, GP_BN) > 65535) {
    set_error("%s: bad sizes (rows=%d ldg=%lld n_seg=%d dim=%d ldo=%lld; dim must be a multiple of 128 in [128, 32768])",
              fn, rows, (long long)ldg, n_seg, dim, (long long)ldo);
    return -2;
  }
  if ((reinterpret_cast<uintptr_t>(G) | reinterpret_cast<uintptr_t>(scratch)) & 15) {
    set_error("%s: G and scratch must be 16-byte aligned", fn);
    return -2;
  }
  const ProjLayout l = proj_layout(rows, ldg, dim, n_seg);
  float* S = (float*)scratch;
  long long* seg = reinterpret_cast<long long*>(S + l.seg);
  long long* host = (long long*)malloc(sizeof(long long) * 2 * n_seg);
  if (!host) { set_error("%s: out of host memory", fn); return -1; }
  for (int i = 0; i < n_seg; ++i) {
    if ((seg_off[i] & 3) || seg_off[i] < 0 || seg_len[i] < 1 || seg_len[i] > RD_GRAD_DOT_SEGMENT || seg_off[i] + seg_len[i] > ldg) {
      set_error("%s: segment %d [%lld, +%lld) is not 4-aligned, 1..%d columns long and inside the row", fn, i,
                (long long)seg_off[i], (long long)seg_len[i], RD_GRAD_DOT_SEGMENT);
      free(host);
      return -2;
    }
    host[2 * i] = seg_off[i]; host[2 * i + 1] = seg_len[i];
  }
  cudaStream_t st = (cudaStream_t)stream;
  // pageable source: the call returns once the table has been staged, so `host` may be freed right after
  const cudaError_t ce = cudaMemcpyAsync(seg, host, sizeof(long long) * 2 * n_seg, cudaMemcpyHostToDevice, st);
  free(host);
  if (ce != cudaSuccess) { set_error("%s: segment table copy: %s", fn, cudaGetErrorString(ce)); return -1; }

  float* lo = S + l.lo;
  RD_TRY(grad_lo_image(G, (long long)rows * ldg, lo, st));
  CUtensorMap tmG, tmGlo;
  {
    cuuint64_t d[2] = {(cuuint64_t)ldg, (cuuint64_t)rows};
    cuuint64_t s[1] = {(cuuint64_t)ldg * 4};
    cuuint32_t b[2] = {GP_BK, GP_BN};
    RD_TRY(encode(&tmG, G, 2, d, s, b, CU_TENSOR_MAP_SWIZZLE_128B, "G"));
    RD_TRY(encode(&tmGlo, lo, 2, d, s, b, CU_TENSOR_MAP_SWIZZLE_128B, "G_lo"));
  }
  RD_TRY(ensure_max_smem((const void*)grad_proj_kernel, GP_SMEM));
  float* partial = S + l.partial;
  launch_pdl(grad_proj_kernel, dim3((unsigned)(dim / GP_BM), (unsigned)ceil_div(rows, GP_BN), (unsigned)n_seg),
             dim3(GP_THREADS), GP_SMEM, st, tmG, tmGlo, (const long long*)seg, (int)rows, (int)dim, (uint32_t)seed,
             (uint32_t)(seed >> 32), partial);
  RD_CHECK_LAUNCH("grad_proj_kernel");
  const long long n = (long long)rows * dim;
  launch_pdl(grad_proj_reduce_kernel, dim3((unsigned)ceil_div(n, 256)), dim3(256), 0, st, (const float*)partial,
             (int)n_seg, (int)rows, (int)dim, 1.0 / sqrt((double)dim), out, (long long)ldo);
  RD_CHECK_LAUNCH("grad_proj_reduce_kernel");
  return 0;
}

int rd_debug_projection_signs(uint64_t seed, int64_t col0, int32_t n_cols, int32_t dim, float* out, void* stream) {
  if (!out || col0 < 0 || n_cols < 0 || !proj_dim_ok(dim)) {
    set_error("rd_debug_projection_signs: bad arguments (col0=%lld n_cols=%d dim=%d)", (long long)col0, n_cols, dim);
    return -2;
  }
  if (n_cols == 0) return 0;
  const long long n = (long long)n_cols * dim;
  if (ceil_div(n, 256) > 0x7fffffffLL) { set_error("rd_debug_projection_signs: too many columns (%d)", n_cols); return -2; }
  launch_pdl(proj_signs_kernel, dim3((unsigned)ceil_div(n, 256)), dim3(256), 0, (cudaStream_t)stream, (uint32_t)seed,
             (uint32_t)(seed >> 32), (long long)col0, (int)n_cols, (int)dim, out);
  RD_CHECK_LAUNCH("proj_signs_kernel");
  return 0;
}

}  // extern "C"
