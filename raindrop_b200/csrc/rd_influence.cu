// Inner products of per-sample gradient rows (TracIn influence, rd_per_sample_grad_dot).
//
// scores[q, t] += alpha * sum_s < Gq[q, seg_s], Gt[t, seg_s] >, segments of at most RD_GRAD_DOT_SEGMENT columns that
// never cross a field.  Both operands are K-major rows, the tc_nt_kernel case (rd_tc_gemm.cu), with a third grid
// dimension over the segments:
//   psg_lo_kernel        Gq_lo = Gq - (top 19 bits of Gq), the exact remainder of the query rows (the error-compensated
//                        B operand, as split_weights makes it for the encoder weights)
//   psg_dot_kernel       one CTA per (query tile of 64, train tile of 128, segment).  Warpgroup 2: one TMA thread fills
//                        a 4-stage ring with the train tile [128 x 32] and the query tiles hi / lo [64 x 32] (128B swizzle)
//                        of each 32-column k-block of the segment.  Warpgroups 0 and 1: train rows 0-63 and 64-127, A
//                        fragments from shared memory split into hi / lo in registers and zeroed past the segment's end
//                        (a k-block may run into the next field), three wgmma.m64n64k8 TF32 per k-step (lo.hi, hi.lo,
//                        hi.hi), one group in flight while the next A fragments are loaded.  The segment's fp32 sum goes
//                        to partial[seg][q][t].
//   psg_dot_reduce_kernel  scores[q, t] += alpha * (sum over the segments in order, fp64).
// Every score is the same sequence of products and additions whatever the tile plan, the query blocking or the train
// chunking, so results are bitwise reproducible across them.
#include "rd_tc_common.cuh"
#include "rd_influence.cuh"
#include "rd_wgmma_tf32.cuh"

namespace rd {
using namespace tc;
namespace {

constexpr int GD_BM = 128, GD_BN = 64, GD_BK = 32, GD_STAGES = 4, GD_THREADS = 384;
constexpr int GD_A_TILE = GD_BM * GD_BK * 4;     // 16 KB: train rows
constexpr int GD_B_TILE = GD_BN * GD_BK * 4;     // 8 KB: query rows, hi then lo
constexpr int GD_STAGE = GD_A_TILE + 2 * GD_B_TILE;
constexpr int GD_SMEM = 1024 + GD_STAGES * GD_STAGE + 256;

__device__ __forceinline__ float gd_lds(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}

// A fragments of one k-block, columns at or past `rem` (the segment's end) read as 0, split into hi / lo
__device__ __forceinline__ void gd_afrag(uint32_t sa, int arow, int t, int rem, uint32_t (&ah)[GD_BK / 8][4],
                                         uint32_t (&al)[GD_BK / 8][4]) {
#pragma unroll
  for (int ks = 0; ks < GD_BK / 8; ++ks) {
    const int col = ks * 8 + t;
    float x[4] = {gd_lds(sa + sw128_offset(arow, col)), gd_lds(sa + sw128_offset(arow + 8, col)),
                  gd_lds(sa + sw128_offset(arow, col + 4)), gd_lds(sa + sw128_offset(arow + 8, col + 4))};
    if (col >= rem) { x[0] = 0.f; x[1] = 0.f; }
    if (col + 4 >= rem) { x[2] = 0.f; x[3] = 0.f; }
#pragma unroll
    for (int i = 0; i < 4; ++i) { ah[ks][i] = tf32_hi(x[i]); al[ks][i] = tf32_lo(x[i]); }
  }
}

__device__ __forceinline__ void gd_issue(float (&acc)[GD_BN / 2], const uint32_t (&ah)[GD_BK / 8][4],
                                         const uint32_t (&al)[GD_BK / 8][4], uint32_t sb) {
#pragma unroll
  for (int e = 0; e < GD_BN / 2; ++e) fence_operand(acc[e]);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < GD_BK / 8; ++ks) {
    const uint32_t bo = sb + (uint32_t)ks * 32u;
    const uint64_t bh = wgmma_desc_sw128(bo);
    wgmma_tf32<GD_BN>(acc, al[ks], bh);
    wgmma_tf32<GD_BN>(acc, ah[ks], wgmma_desc_sw128(bo + GD_B_TILE));
    wgmma_tf32<GD_BN>(acc, ah[ks], bh);
  }
  wgmma_commit();
}

__global__ void __launch_bounds__(GD_THREADS, 1)
psg_dot_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmBlo, const long long* __restrict__ seg, int Bq, int Bt,
               float* __restrict__ partial) {
  extern __shared__ uint8_t smem_raw[];
  pdl_launch_dependents();
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const TmaRing<GD_STAGES> ring{base + (uint32_t)GD_STAGES * GD_STAGE};
  const int q_t = blockIdx.x, t_t = blockIdx.y, z = blockIdx.z;

  if (warp == 8 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmBlo) : "memory");
    ring.init(8);
  }
  __syncthreads();
  pdl_wait();
  const long long off = seg[2 * z];
  const int len = (int)seg[2 * z + 1];
  const int k_blocks = (len + GD_BK - 1) / GD_BK;

  if (warp >= 8) {
    // ===== TMA producer ==========================================================================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 8 && lane == 0) {
      RingPos<GD_STAGES> p;
      for (int kb = 0; kb < k_blocks; ++kb) {
        const int stage = ring.produce(p, GD_STAGE);
        const uint32_t sa = base + (uint32_t)stage * GD_STAGE;
        const int col = (int)(off + (long long)kb * GD_BK);
        tma_load_2d(&tmA, ring.full(stage), sa, col, t_t * GD_BM);
        tma_load_2d(&tmB, ring.full(stage), sa + GD_A_TILE, col, q_t * GD_BN);
        tma_load_2d(&tmBlo, ring.full(stage), sa + GD_A_TILE + GD_B_TILE, col, q_t * GD_BN);
      }
    }
    return;
  }

  // ===== warpgroups 0, 1: MMA and epilogue ========================================================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  const int wg = warp >> 2, wq = warp & 3, g = lane >> 2, t = lane & 3;
  const int arow = wg * 64 + wq * 16 + g;
  RingPos<GD_STAGES> cpos, rpos;
  int next = 0;
  auto acquire = [&](uint32_t (&ah)[GD_BK / 8][4], uint32_t (&al)[GD_BK / 8][4]) {
    const uint32_t sa = base + (uint32_t)ring.consume(cpos) * GD_STAGE;
    gd_afrag(sa, arow, t, len - next * GD_BK, ah, al);
    ++next;
    return sa + (uint32_t)GD_A_TILE;
  };
  auto release = [&]() { ring.release(rpos, lane); };
  // The tensor cores' fp32 accumulation is not round-to-nearest: summed over thousands of k-steps, same-sign products lose
  // magnitude systematically (measured 4.5e-5 relative at 4,096 columns).  So each k-block's 12 wgmma go to fresh
  // accumulators (k-blocks alternate between a0 and a1), and the k-block sums are added on the CUDA cores, in order.
  float acc[GD_BN / 2], a0[GD_BN / 2], a1[GD_BN / 2];
#pragma unroll
  for (int e = 0; e < GD_BN / 2; ++e) { acc[e] = 0.f; a0[e] = 0.f; a1[e] = 0.f; }
  auto fold = [&](float (&a)[GD_BN / 2]) {
#pragma unroll
    for (int e = 0; e < GD_BN / 2; ++e) { fence_operand(a[e]); acc[e] += a[e]; a[e] = 0.f; }
  };
  uint32_t ah0[GD_BK / 8][4], al0[GD_BK / 8][4], ah1[GD_BK / 8][4], al1[GD_BK / 8][4];
  uint32_t sb0 = acquire(ah0, al0), sb1 = 0;
  for (int kb = 0; kb < k_blocks; kb += 2) {
    gd_issue(a0, ah0, al0, sb0);
    wgmma_wait<1>();
    if (kb > 0) { release(); fold(a1); }          // k-block kb - 1 has retired
    if (kb + 1 >= k_blocks) break;
    sb1 = acquire(ah1, al1);
    gd_issue(a1, ah1, al1, sb1);
    wgmma_wait<1>();
    release();
    fold(a0);                                     // k-block kb has retired
    if (kb + 2 < k_blocks) sb0 = acquire(ah0, al0);
  }
  wgmma_wait<0>();
  release();
  if (k_blocks & 1) fold(a0); else fold(a1);

  // element (train row arow + 8i, query column 8j + 2t + c) of the tile
#pragma unroll
  for (int j = 0; j < GD_BN / 8; ++j)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int tr = t_t * GD_BM + arow + 8 * i, qc = q_t * GD_BN + 8 * j + 2 * t + c;
        if (tr < Bt && qc < Bq) partial[((long long)z * Bq + qc) * Bt + tr] = acc[4 * j + 2 * i + c];
      }
}

__global__ void psg_lo_kernel(const float4* __restrict__ x, float4* __restrict__ lo, long long n4) {
  pdl_launch_dependents();
  pdl_wait();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = x[i];
    lo[i] = make_float4(__uint_as_float(tf32_lo(v.x)), __uint_as_float(tf32_lo(v.y)), __uint_as_float(tf32_lo(v.z)),
                        __uint_as_float(tf32_lo(v.w)));
  }
}

__global__ void psg_dot_reduce_kernel(const float* __restrict__ partial, int n_seg, int Bq, int Bt, double alpha,
                                      double* __restrict__ scores, long long lds) {
  pdl_launch_dependents();
  pdl_wait();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)Bq * Bt) return;
  const int q = (int)(idx / Bt), t = (int)(idx % Bt);
  double s = 0.0;
  for (int z = 0; z < n_seg; ++z) s += (double)partial[((long long)z * Bq + q) * Bt + t];
  scores[(long long)q * lds + t] += alpha * s;
}

struct DotLayout { int64_t lo, seg, partial, total; };     // floats
DotLayout dot_layout(int Bq, int Bt, int64_t ldg, int n_seg) {
  DotLayout l;
  l.lo = 0;
  l.seg = round_up((int64_t)Bq * ldg, 64);
  l.partial = l.seg + round_up(4LL * n_seg, 64);
  l.total = l.partial + (int64_t)n_seg * Bq * Bt;
  return l;
}

}  // namespace

int grad_lo_image(const float* G, long long n, float* lo, cudaStream_t st) {
  const long long n4 = n / 4;
  long long blocks = ceil_div(n4, 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  launch_pdl(psg_lo_kernel, dim3((unsigned)blocks), dim3(256), 0, st, reinterpret_cast<const float4*>(G),
             reinterpret_cast<float4*>(lo), n4);
  RD_CHECK_LAUNCH("psg_lo_kernel");
  return 0;
}

}  // namespace rd

using namespace rd;

extern "C" {

size_t rd_per_sample_grad_dot_scratch_bytes(int32_t Bq, int32_t Bt, int64_t ldg, int32_t n_seg) {
  if (Bq < 1 || Bt < 1 || ldg < 1 || n_seg < 1) return 0;
  return (size_t)dot_layout(Bq, Bt, ldg, n_seg).total * sizeof(float);
}

int rd_per_sample_grad_dot(const float* Gq, int32_t Bq, const float* Gt, int32_t Bt, int64_t ldg, const int64_t* seg_off,
                           const int64_t* seg_len, int32_t n_seg, double alpha, double* scores, int64_t lds, void* scratch,
                           void* stream) {
  const char* fn = "rd_per_sample_grad_dot";
  if (!Gq || !Gt || !seg_off || !seg_len || !scores || !scratch) { set_error("%s: NULL argument", fn); return -2; }
  if (Bq < 1 || Bt < 1 || ldg < 4 || (ldg & 3) || ldg > 0x7fffffffLL || n_seg < 1 || n_seg > 65535 || lds < Bt ||
      ceil_div(Bt, GD_BM) > 65535) {
    set_error("%s: bad sizes (Bq=%d Bt=%d ldg=%lld n_seg=%d lds=%lld)", fn, Bq, Bt, (long long)ldg, n_seg, (long long)lds);
    return -2;
  }
  if ((reinterpret_cast<uintptr_t>(Gq) | reinterpret_cast<uintptr_t>(Gt) | reinterpret_cast<uintptr_t>(scratch)) & 15) {
    set_error("%s: Gq, Gt and scratch must be 16-byte aligned", fn);
    return -2;
  }
  const DotLayout l = dot_layout(Bq, Bt, ldg, n_seg);
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
  RD_TRY(grad_lo_image(Gq, (long long)Bq * ldg, lo, st));

  CUtensorMap tmA, tmB, tmBlo;
  {
    cuuint64_t d[2] = {(cuuint64_t)ldg, (cuuint64_t)Bt};
    cuuint64_t s[1] = {(cuuint64_t)ldg * 4};
    cuuint32_t b[2] = {GD_BK, GD_BM};
    RD_TRY(encode(&tmA, Gt, 2, d, s, b, CU_TENSOR_MAP_SWIZZLE_128B, "Gt"));
  }
  {
    cuuint64_t d[2] = {(cuuint64_t)ldg, (cuuint64_t)Bq};
    cuuint64_t s[1] = {(cuuint64_t)ldg * 4};
    cuuint32_t b[2] = {GD_BK, GD_BN};
    RD_TRY(encode(&tmB, Gq, 2, d, s, b, CU_TENSOR_MAP_SWIZZLE_128B, "Gq"));
    RD_TRY(encode(&tmBlo, lo, 2, d, s, b, CU_TENSOR_MAP_SWIZZLE_128B, "Gq_lo"));
  }
  RD_TRY(ensure_max_smem((const void*)psg_dot_kernel, GD_SMEM));
  float* partial = S + l.partial;
  launch_pdl(psg_dot_kernel, dim3((unsigned)ceil_div(Bq, GD_BN), (unsigned)ceil_div(Bt, GD_BM), (unsigned)n_seg),
             dim3(GD_THREADS), GD_SMEM, st, tmA, tmB, tmBlo, (const long long*)seg, (int)Bq, (int)Bt, partial);
  RD_CHECK_LAUNCH("psg_dot_kernel");
  const long long n = (long long)Bq * Bt;
  launch_pdl(psg_dot_reduce_kernel, dim3((unsigned)ceil_div(n, 256)), dim3(256), 0, st, (const float*)partial, (int)n_seg,
             (int)Bq, (int)Bt, alpha, scores, (long long)lds);
  RD_CHECK_LAUNCH("psg_dot_reduce_kernel");
  return 0;
}

}  // extern "C"
