// Temporal self-attention for short sequences (T <= 64, head_dim <= 96) on the tensor cores (sm_90a).
//
// nn.TransformerEncoder's attention as called at code/models_rd.py:358 for the P19 shape (T = 60, hd = 76):
// per (sample, head) S = scale * Q K^T, key-padding-masked softmax, attention dropout, O = P V -- and the whole
// backward (dV = Pd^T dO, dP = dO V^T, dS = P * (dP - rowsum(dP * P)), dQ = scale * dS K, dK = scale * dS^T Q).
// One CTA of four warps per (sample, head); warp w owns rows 16w .. 16w+15 of every product.  Every contraction is an
// error-compensated mma.sync.m16n8k8 TF32 product (operands split into hi + lo in registers, three MMAs per k-step:
// lo.hi + hi.lo + hi.hi), so the results are fp32-accurate like the CUDA-core kernels in rd_attn_small.cu.  Half of
// these contractions run over the ROWS of a shared-memory tile (O = P V, dV, dQ, dK), which wgmma's TF32 form cannot
// read; mma.sync takes fragments gathered per thread, so one row-major image per operand serves every role and nothing
// is transposed.  Nothing T x T reaches HBM; the backward RECOMPUTES the probabilities from Q, K and the counter-based
// dropout stream.
//
// Shared memory: head slices [64][LD] with LD = round_up(hd, 8) + 4 (a row stride of 4 mod 8 floats keeps the
// row-wise fragment gathers free of bank conflicts), probability / score-gradient tiles [64][68].  At P19 (hd = 76,
// LD = 84) the forward takes 80 KB and the backward 101 KB (Pd reuses the V slice), so two CTAs share an SM.
#include <stdlib.h>

#include "rd_kernels.cuh"
#include "rd_tc_common.cuh"

namespace rd {
using namespace tc;
namespace {

constexpr int TR = 64;                    // rows (timestamps) per head slice
constexpr int HD_MAX = 96;
constexpr int LDP = TR + 4;               // probability / score-gradient tiles
constexpr int NTHR = 128;

struct AttnTcP {
  float* ctx; float* dqkv;
  const int64_t* lengths;
  int B, H, T, hd, D, ld;
  float scale, drop_p;
  const uint64_t* rng; uint32_t site;
  DropRep rep;                  // forward only: replicate-major samples (rep_remap)
  unsigned long long* dbg;      // optional start / end timestamps (rd_debug_attention_timing): [CTA][16] of clock64
};

__device__ __forceinline__ void stamp(const AttnTcP& p, int slot) {
  if (p.dbg && threadIdx.x == 0) p.dbg[(size_t)blockIdx.x * 16 + slot] = (unsigned long long)clock64();
}
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// rows t < T, columns d < hd of one head slice (row r of the slice at src + r * row_stride) -> s[64][ld], zero padded to
// 64 rows and round_up(hd, 8) columns
__device__ __forceinline__ void load_slice(float* s, const float* src, long long row_stride, const AttnTcP& p) {
  const int q = ((p.hd + 7) & ~7) >> 2;          // float4 per padded row
  for (int v = threadIdx.x; v < TR * q; v += NTHR) {
    const int r = v / q, c = 4 * (v - r * q);
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < p.T && c < p.hd) x = __ldg(reinterpret_cast<const float4*>(src + r * row_stride + c));
    *reinterpret_cast<float4*>(s + r * p.ld + c) = x;
  }
}

// acc[j] (16 rows from r0) += A . B over `ksteps` k-steps of 8, n8 tiles j < nt.
//   A_T:  A[m][k] = sa[k * lda + m]  (else sa[m * lda + k])
//   B_KN: B[k][n] = sb[k * ldb + n]  (else sb[n * ldb + k])
template <int NTMAX, bool A_T, bool B_KN>
__device__ __forceinline__ void mma_rows16(float (&acc)[NTMAX][4], const float* sa, int lda, int r0, const float* sb, int ldb,
                                           int nt, int ksteps) {
  const int g = (threadIdx.x & 31) >> 2, t = threadIdx.x & 3;
#pragma unroll 1
  for (int ks = 0; ks < ksteps; ++ks) {
    const int k0 = ks * 8;
    float x0, x1, x2, x3;
    if (A_T) {
      x0 = sa[(k0 + t) * lda + r0 + g]; x1 = sa[(k0 + t) * lda + r0 + g + 8];
      x2 = sa[(k0 + t + 4) * lda + r0 + g]; x3 = sa[(k0 + t + 4) * lda + r0 + g + 8];
    } else {
      x0 = sa[(r0 + g) * lda + k0 + t]; x1 = sa[(r0 + g + 8) * lda + k0 + t];
      x2 = sa[(r0 + g) * lda + k0 + t + 4]; x3 = sa[(r0 + g + 8) * lda + k0 + t + 4];
    }
    const uint32_t ah[4] = {tf32_hi(x0), tf32_hi(x1), tf32_hi(x2), tf32_hi(x3)};
    const uint32_t al[4] = {tf32_lo(x0), tf32_lo(x1), tf32_lo(x2), tf32_lo(x3)};
#pragma unroll
    for (int j = 0; j < NTMAX; ++j) {
      if (j < nt) {
        const int n = j * 8 + g;
        const float y0 = B_KN ? sb[(k0 + t) * ldb + n] : sb[n * ldb + k0 + t];
        const float y1 = B_KN ? sb[(k0 + t + 4) * ldb + n] : sb[n * ldb + k0 + t + 4];
        mma_tf32x3(acc[j], ah, al, tf32_hi(y0), tf32_hi(y1), tf32_lo(y0), tf32_lo(y1));
      }
    }
  }
}

template <int NTMAX>
__device__ __forceinline__ void zero(float (&acc)[NTMAX][4]) {
#pragma unroll
  for (int j = 0; j < NTMAX; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
}

// keep factor (0 or ik) of attention-dropout element (i, j): index space [B, H, T, T]
__device__ __forceinline__ float keep_at(const AttnTcP& p, const RngKey& key, int b, int h, int i, int j, float ik) {
  if (p.drop_p <= 0.f) return 1.f;
  if (i >= p.T || j >= p.T) return 0.f;
  return dropout_scale(key, p.site, ((uint64_t)(b * p.H + h) * p.T + i) * p.T + j, p.drop_p, ik);
}

// accumulator rows 16w + g (+8) of an [64 x hd] product -> dst row r at dst + r * row_stride, r < T, d < hd
__device__ __forceinline__ void store_rows(const float (&acc)[HD_MAX / 8][4], float* dst, long long row_stride, int r0,
                                           const AttnTcP& p) {
  const int g = (threadIdx.x & 31) >> 2, t = threadIdx.x & 3;
#pragma unroll
  for (int j = 0; j < HD_MAX / 8; ++j) {
    const int d = j * 8 + 2 * t;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = r0 + g + 8 * i;
      if (r < p.T && d < p.hd)
        *reinterpret_cast<float2*>(dst + r * row_stride + d) = make_float2(acc[j][2 * i], acc[j][2 * i + 1]);
    }
  }
}

// row statistics of the masked softmax over the two rows (16w + g, +8) this thread holds a quarter of
struct RowStat { float mxs[2], sum[2]; };
__device__ __forceinline__ RowStat row_stats(const float (&s)[TR / 8][4], int nv, float sl2) {
  const int t = threadIdx.x & 3;
  RowStat r;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < TR / 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) if (j * 8 + 2 * t + e < nv) mx = fmaxf(mx, s[j][2 * i + e]);
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    r.mxs[i] = mx * sl2;
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < TR / 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) if (j * 8 + 2 * t + e < nv) sum += ex2_approx(fmaf(s[j][2 * i + e], sl2, -r.mxs[i]));
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    r.sum[i] = sum;
  }
  return r;
}

// =================================================================================================
// forward: ctx[t, b, h*hd + d] = sum_j dropout(softmax(scale * Q K^T))[t, j] V[j, d]
// =================================================================================================
// REP: attention dropout of replicate-major samples (rep_remap); a separate instance, so the training step's is unchanged
template <bool REP>
__global__ void __launch_bounds__(NTHR) attn_tc_fwd_kernel(const float* __restrict__ qkv, const AttnTcP p) {
  extern __shared__ float sm[];
  pdl_launch_dependents();
  pdl_wait();
  stamp(p, 0);
  const int b = blockIdx.x / p.H, h = blockIdx.x - b * p.H;
  const int w = threadIdx.x >> 5, g = (threadIdx.x & 31) >> 2, t = threadIdx.x & 3;
  float* sQ = sm; float* sK = sQ + TR * p.ld; float* sV = sK + TR * p.ld; float* sP = sV + TR * p.ld;
  const long long rs = (long long)p.B * 3 * p.D;
  const float* base = qkv + (long long)b * 3 * p.D + h * p.hd;
  load_slice(sQ, base, rs, p);
  load_slice(sK, base + p.D, rs, p);
  load_slice(sV, base + 2 * p.D, rs, p);
  RngKey key = load_rng_key(p.drop_p > 0.f ? p.rng : nullptr);
  int bd = b;             // the sample whose dropout words this CTA draws
  if (REP) bd = (int)(rep_remap(p.rng, p.rep, (uint32_t)b, 1, 0, &key));
  const long long len = p.lengths[b];
  const int nv = (int)(len < p.T ? (len < 0 ? 0 : len) : p.T);
  const int ksd = (p.hd + 7) >> 3;
  __syncthreads();

  float s[TR / 8][4];
  zero(s);
  mma_rows16<TR / 8, false, false>(s, sQ, p.ld, 16 * w, sK, p.ld, TR / 8, ksd);
  const float sl2 = p.scale * 1.4426950408889634f;
  const RowStat st = row_stats(s, nv, sl2);
  const float ik = p.drop_p > 0.f ? 1.f / (1.f - p.drop_p) : 1.f;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int r = 16 * w + g + 8 * i;
    const float invk = ((r < p.T && nv > 0) ? 1.f / st.sum[i] : 0.f);
#pragma unroll
    for (int j = 0; j < TR / 8; ++j) {
      float o[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int c = j * 8 + 2 * t + e;
        const float ex = c < nv ? ex2_approx(fmaf(s[j][2 * i + e], sl2, -st.mxs[i])) : 0.f;
        o[e] = (ex != 0.f && invk != 0.f) ? ex * invk * keep_at(p, key, bd, h, r, c, ik) : 0.f;
      }
      *reinterpret_cast<float2*>(sP + r * LDP + j * 8 + 2 * t) = make_float2(o[0], o[1]);
    }
  }
  __syncwarp();           // O rows 16w.. read only this warp's probability rows (V is complete since the barrier)
  float o[HD_MAX / 8][4];
  zero(o);
  mma_rows16<HD_MAX / 8, false, true>(o, sP, LDP, 16 * w, sV, p.ld, ksd, TR / 8);
  store_rows(o, p.ctx + (long long)b * p.D + h * p.hd, (long long)p.B * p.D, 16 * w, p);
  stamp(p, 12);
}

// =================================================================================================
// backward
// =================================================================================================
__global__ void __launch_bounds__(NTHR) attn_tc_bwd_kernel(const float* __restrict__ qkv, const float* __restrict__ dctx,
                                                           const AttnTcP p) {
  extern __shared__ float sm[];
  pdl_launch_dependents();
  pdl_wait();
  stamp(p, 0);
  const int b = blockIdx.x / p.H, h = blockIdx.x - b * p.H;
  const int w = threadIdx.x >> 5, g = (threadIdx.x & 31) >> 2, t = threadIdx.x & 3;
  float* sQ = sm; float* sK = sQ + TR * p.ld; float* sV = sK + TR * p.ld; float* sG = sV + TR * p.ld;
  // V is dead once dP = dO V^T is formed: the masked probabilities Pd take its place when they fit there
  float* sS = sG + TR * p.ld; float* sPd = p.ld >= LDP ? sV : sS + TR * LDP;
  const long long rs = (long long)p.B * 3 * p.D;
  const float* base = qkv + (long long)b * 3 * p.D + h * p.hd;
  load_slice(sQ, base, rs, p);
  load_slice(sK, base + p.D, rs, p);
  load_slice(sV, base + 2 * p.D, rs, p);
  load_slice(sG, dctx + (long long)b * p.D + h * p.hd, (long long)p.B * p.D, p);
  const RngKey key = load_rng_key(p.drop_p > 0.f ? p.rng : nullptr);
  const long long len = p.lengths[b];
  const int nv = (int)(len < p.T ? (len < 0 ? 0 : len) : p.T);
  const int ksd = (p.hd + 7) >> 3;
  __syncthreads();

  {
    float s[TR / 8][4], dp[TR / 8][4];
    zero(s); zero(dp);
    mma_rows16<TR / 8, false, false>(s, sQ, p.ld, 16 * w, sK, p.ld, TR / 8, ksd);     // recompute the scores
    mma_rows16<TR / 8, false, false>(dp, sG, p.ld, 16 * w, sV, p.ld, TR / 8, ksd);    // dPd[i, j] = sum_d dO[i, d] V[j, d]
    __syncthreads();      // every warp has read V (Pd may overwrite it below)
    const float sl2 = p.scale * 1.4426950408889634f;
    const RowStat st = row_stats(s, nv, sl2);
    const float ik = p.drop_p > 0.f ? 1.f / (1.f - p.drop_p) : 1.f;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = 16 * w + g + 8 * i;
      const float inv = (r < p.T && nv > 0) ? 1.f / st.sum[i] : 0.f;
      float pr[TR / 8][2], m[TR / 8][2];
      float dot = 0.f;                 // rowsum(dP * P) with dP = dPd * mask
#pragma unroll
      for (int j = 0; j < TR / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = j * 8 + 2 * t + e;
          pr[j][e] = c < nv ? ex2_approx(fmaf(s[j][2 * i + e], sl2, -st.mxs[i])) * inv : 0.f;
          m[j][e] = pr[j][e] != 0.f ? keep_at(p, key, b, h, r, c, ik) : 0.f;
          dot += dp[j][2 * i + e] * m[j][e] * pr[j][e];
        }
      dot += __shfl_xor_sync(0xffffffffu, dot, 1);
      dot += __shfl_xor_sync(0xffffffffu, dot, 2);
#pragma unroll
      for (int j = 0; j < TR / 8; ++j) {
        const int c = j * 8 + 2 * t;
        *reinterpret_cast<float2*>(sPd + r * LDP + c) = make_float2(pr[j][0] * m[j][0], pr[j][1] * m[j][1]);   // Pd = P * mask
        *reinterpret_cast<float2*>(sS + r * LDP + c) =                                                       // scale * dS
            make_float2(pr[j][0] * (dp[j][2 * i] * m[j][0] - dot) * p.scale, pr[j][1] * (dp[j][2 * i + 1] * m[j][1] - dot) * p.scale);
      }
    }
  }
  __syncthreads();        // dV and dK contract over all rows i of Pd / dS
  float acc[HD_MAX / 8][4];
  float* out = p.dqkv + (long long)b * 3 * p.D + h * p.hd;
  // dV[j, d] = sum_i Pd[i, j] dO[i, d]
  zero(acc);
  mma_rows16<HD_MAX / 8, true, true>(acc, sPd, LDP, 16 * w, sG, p.ld, ksd, TR / 8);
  store_rows(acc, out + 2 * p.D, rs, 16 * w, p);
  // dQ[i, d] = sum_j (scale dS)[i, j] K[j, d]
  zero(acc);
  mma_rows16<HD_MAX / 8, false, true>(acc, sS, LDP, 16 * w, sK, p.ld, ksd, TR / 8);
  store_rows(acc, out, rs, 16 * w, p);
  // dK[j, d] = sum_i (scale dS)[i, j] Q[i, d]
  zero(acc);
  mma_rows16<HD_MAX / 8, true, true>(acc, sS, LDP, 16 * w, sQ, p.ld, ksd, TR / 8);
  store_rows(acc, out + p.D, rs, 16 * w, p);
  stamp(p, 12);
}

int slice_ld(int hd) { return ((hd + 7) & ~7) + 4; }
int fwd_smem(int hd) { return (3 * TR * slice_ld(hd) + TR * LDP) * (int)sizeof(float); }
int bwd_smem(int hd) { return (4 * TR * slice_ld(hd) + (slice_ld(hd) >= LDP ? 1 : 2) * TR * LDP) * (int)sizeof(float); }

}  // namespace

static unsigned long long* g_attn_dbg = nullptr;
void attn_tc_set_debug(unsigned long long* buf) { g_attn_dbg = buf; }

bool attn_tc_supported(int T, int hd) {
  static int env = -1;
  if (env < 0) { const char* e = getenv("RD_ATTN_TC"); env = (e && e[0] == '0') ? 0 : 1; }
  return env == 1 && T <= TR && hd <= HD_MAX && hd % 4 == 0 && hd >= 4;
}

int attn_tc_fwd(const float* qkv, const int64_t* lengths, int B, int H, int T, int hd, float drop_p, const uint64_t* rng,
                uint32_t site, float* ctx, cudaStream_t st, DropRep rep) {
  if (!attn_tc_supported(T, hd) || ((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(ctx)) & 15)) {
    set_error("attn_tc_fwd: unsupported shape / alignment (T=%d hd=%d)", T, hd);
    return -2;
  }
  AttnTcP p{};
  p.ctx = ctx; p.lengths = lengths; p.B = B; p.H = H; p.T = T; p.hd = hd; p.D = H * hd; p.ld = slice_ld(hd);
  p.scale = 1.f / sqrtf((float)hd); p.drop_p = drop_p; p.rng = rng; p.site = site; p.rep = rep; p.dbg = g_attn_dbg;
  auto kern = drop_p > 0.f && rep.B ? attn_tc_fwd_kernel<true> : attn_tc_fwd_kernel<false>;
  RD_TRY(ensure_max_smem((const void*)kern, fwd_smem(HD_MAX)));
  launch_pdl(kern, dim3(B * H), dim3(NTHR), fwd_smem(hd), st, qkv, p);
  RD_CHECK_LAUNCH("attn_tc_fwd_kernel");
  return 0;
}

int attn_tc_bwd(const float* qkv, const float* dctx, const int64_t* lengths, int B, int H, int T, int hd, float drop_p,
                const uint64_t* rng, uint32_t site, float* dqkv, cudaStream_t st) {
  if (!attn_tc_supported(T, hd) ||
      ((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(dctx) | reinterpret_cast<uintptr_t>(dqkv)) & 15)) {
    set_error("attn_tc_bwd: unsupported shape / alignment (T=%d hd=%d)", T, hd);
    return -2;
  }
  AttnTcP p{};
  p.dqkv = dqkv; p.lengths = lengths; p.B = B; p.H = H; p.T = T; p.hd = hd; p.D = H * hd; p.ld = slice_ld(hd);
  p.scale = 1.f / sqrtf((float)hd); p.drop_p = drop_p; p.rng = rng; p.site = site; p.dbg = g_attn_dbg;
  RD_TRY(ensure_max_smem((const void*)attn_tc_bwd_kernel, bwd_smem(HD_MAX)));
  launch_pdl(attn_tc_bwd_kernel, dim3(B * H), dim3(NTHR), bwd_smem(hd), st, qkv, dctx, p);
  RD_CHECK_LAUNCH("attn_tc_bwd_kernel");
  return 0;
}

}  // namespace rd
