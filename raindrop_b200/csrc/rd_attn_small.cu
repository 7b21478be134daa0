// Fused temporal self-attention for short sequences (T <= 64, head_dim <= 96): one CTA per (sample, head)
// keeps Q, K, V [T x hd] and the T x T score tile in shared memory, so QK^T, the key-padding-masked
// softmax, attention dropout and PV are one launch (forward) and the whole backward is one launch
// (probabilities are RECOMPUTED from Q, K and the counter-based dropout mask: nothing T x T is stored).
// This is the temporal-attention stage of nn.TransformerEncoder as called at code/models_rd.py:358 for
// the P19 shape (T = 60, hd = 76), in fp32 on the CUDA cores with 4x4 / 4x5 register tiles (implementation 2 of
// rd_temporal_attention_*; the tensor-core kernels in rd_attn_tc.cu are the default); longer sequences take the
// batched-GEMM path (rd_model.cu).
#include <stdlib.h>

#include "rd_kernels.cuh"
#include "rd_tc_common.cuh"

namespace rd {
namespace {

constexpr int TM = 64;      // max sequence length
constexpr int HDM = 96;     // max head dim (6 columns per thread x 16 threads)
constexpr int LDR = 100;    // row-major [t][d] stride (d < 96 zero padded; even -> float2 reads of 6 contiguous columns)
constexpr int LDT = 68;     // transposed [d][t] / [j][i] stride (multiple of 4 -> float4 reads of 4 contiguous rows)

struct AttnP {
  const float* qkv; float* ctx;            // forward
  const float* dctx; float* dqkv;          // backward
  const int64_t* lengths;
  int B, H, T, hd, D;
  float scale, drop_p;
  const uint64_t* rng; uint32_t site;
  DropRep rep;                             // forward only
};

// One [T x hd] head slice -> shared memory, row-major (rm[t*LDR + d], zero padded to 64 x 96) and/or
// transposed (tr[d*LDT + t], t zero padded to 64).  All global loads of a thread are issued before the
// first store (6 independent 128-bit loads in flight per thread: the slice is latency-, not bandwidth-bound).
__device__ __forceinline__ void load_head(const float* __restrict__ src, long long row_stride, int T, int hd, bool vec,
                                          float* rm, float* tr) {
  if (vec) {
    const int nvec = hd >> 2;
    float4 v[6];
    int tt[6], cc[6];
    const int nthr = blockDim.x;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const int idx = threadIdx.x + k * nthr;     // 6 x blockDim >= 64 * 24 float4 for both CTA sizes
      tt[k] = idx / nvec; cc[k] = idx - tt[k] * nvec;
      v[k] = (tt[k] < T) ? __ldg(reinterpret_cast<const float4*>(src + (long long)tt[k] * row_stride + 4 * cc[k]))
                         : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      if (tt[k] >= TM) continue;
      if (rm) *reinterpret_cast<float4*>(rm + tt[k] * LDR + 4 * cc[k]) = v[k];
      if (tr) {
        float* o = tr + (4 * cc[k]) * LDT + tt[k];
        o[0] = v[k].x; o[LDT] = v[k].y; o[2 * LDT] = v[k].z; o[3 * LDT] = v[k].w;
      }
    }
  } else {
    for (int idx = threadIdx.x; idx < TM * hd; idx += blockDim.x) {
      const int t = idx / hd, d = idx - t * hd;
      const float x = t < T ? __ldg(src + (long long)t * row_stride + d) : 0.f;
      if (rm) rm[t * LDR + d] = x;
      if (tr) tr[d * LDT + t] = x;
    }
  }
  if (rm) {   // zero the padding columns hd..95 (read by the 6-column register tiles)
    const int npad = HDM - hd;
    for (int idx = threadIdx.x; idx < TM * npad; idx += blockDim.x) {
      const int t = idx / npad, d = hd + idx - t * npad;
      rm[t * LDR + d] = 0.f;
    }
  }
}

// out[i][j] = alpha * sum_d At[d][i] * Bt[d][j]   (both operands transposed in smem: 2 LDS.128 per 16 FMA)
// With 512 threads the reduction range is split between the two 256-thread groups (group 1 adds its
// partial into `out` after a barrier): twice the warps per SM to hide shared-memory latency.
__device__ __forceinline__ void gemm_tt(const float* At, const float* Bt, int hd, float alpha, float* out) {
  const int t256 = threadIdx.x & 255, grp = threadIdx.x >> 8, ngrp = blockDim.x >> 8;
  const int tx = t256 & 15, ty = t256 >> 4;
  float acc[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
  const int d0 = grp * ((hd + ngrp - 1) / ngrp), d1 = min(hd, d0 + (hd + ngrp - 1) / ngrp);
  for (int d = d0; d < d1; ++d) {
    const float4 a = *reinterpret_cast<const float4*>(At + d * LDT + 4 * ty);
    const float4 b = *reinterpret_cast<const float4*>(Bt + d * LDT + 4 * tx);
    const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[r][c] = fmaf(av[r], bv[c], acc[r][c]);
  }
  if (grp == 0) {
#pragma unroll
    for (int r = 0; r < 4; ++r)
      *reinterpret_cast<float4*>(out + (4 * ty + r) * LDT + 4 * tx) =
          make_float4(acc[r][0] * alpha, acc[r][1] * alpha, acc[r][2] * alpha, acc[r][3] * alpha);
  }
  if (ngrp > 1) {
    __syncthreads();
    if (grp == 1) {
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        float4* o = reinterpret_cast<float4*>(out + (4 * ty + r) * LDT + 4 * tx);
        float4 v = *o;
        v.x += acc[r][0] * alpha; v.y += acc[r][1] * alpha; v.z += acc[r][2] * alpha; v.w += acc[r][3] * alpha;
        *o = v;
      }
    }
  }
}

// key-padding-masked softmax of the rows of Ps (in place -> probabilities); the dropped copy goes to
// Pd[i*pd_si + j*pd_sj] (row-major or transposed, whatever the consumer wants)
__device__ __forceinline__ void softmax_rows(const AttnP& p, int b, int h, float* Ps, float* Pd, int pd_si, int pd_sj) {
  const int T = p.T;
  const long long len = p.lengths[b];
  const int nv = (int)(len < T ? (len < 0 ? 0 : len) : T);
  const float ik = p.drop_p > 0.f ? 1.f / (1.f - p.drop_p) : 1.f;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = warp; i < TM; i += (int)(blockDim.x >> 5)) {
    float* row = Ps + i * LDT;
    float v0 = (i < T && lane < nv) ? row[lane] : -INFINITY, v1 = (i < T && lane + 32 < nv) ? row[lane + 32] : -INFINITY;
    float mx = warp_max(fmaxf(v0, v1));
    float e0 = (i < T && lane < nv) ? expf(v0 - mx) : 0.f, e1 = (i < T && lane + 32 < nv) ? expf(v1 - mx) : 0.f;
    float sum = warp_sum(e0 + e1);
    float inv = (i < T && nv > 0) ? 1.f / sum : 0.f;
    uint64_t base = ((uint64_t)(b * p.H + h) * T + i) * T;     // index space [B, H, T, T]
    RngKey key;
    if (p.rep.B && p.drop_p > 0.f) base = rep_remap(p.rng, p.rep, (uint32_t)b, (uint64_t)p.H * T * T, ((uint64_t)h * T + i) * T, &key);
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int j = lane + 32 * half;
      const float pr = (half ? e1 : e0) * inv;
      row[j] = pr;
      float m = 1.f;
      if (p.drop_p > 0.f && i < T && j < T)
        m = p.rep.B ? dropout_scale(key, p.site, base + j, p.drop_p, ik) : dropout_scale(p.rng, p.site, base + j, p.drop_p, ik);
      Pd[i * pd_si + j * pd_sj] = pr * m;
    }
  }
}

__global__ void __launch_bounds__(512) attn_small_fwd_kernel(AttnP p) {
  extern __shared__ __align__(16) float sm[];
  const int b = blockIdx.x / p.H, h = blockIdx.x - b * p.H;
  float* Qt = sm; float* Kt = Qt + HDM * LDT; float* Vs = Kt + HDM * LDT;
  float* Ps = Vs + TM * LDR; float* PdT = Ps + TM * LDT;
  const long long rs = (long long)p.B * 3 * p.D;
  const float* base = p.qkv + (long long)b * 3 * p.D + h * p.hd;
  const bool vec = (p.hd % 4 == 0) && (p.D % 4 == 0);
  load_head(base, rs, p.T, p.hd, vec, nullptr, Qt);
  load_head(base + p.D, rs, p.T, p.hd, vec, nullptr, Kt);
  load_head(base + 2 * p.D, rs, p.T, p.hd, vec, Vs, nullptr);
  __syncthreads();
  gemm_tt(Qt, Kt, p.hd, p.scale, Ps);
  __syncthreads();
  softmax_rows(p, b, h, Ps, PdT, 1, LDT);      // dropped probabilities transposed: PdT[j][i]
  __syncthreads();
  // ctx[i, d] = sum_j Pd[i, j] V[j, d]; thread tile 4 rows x 6 contiguous columns; the two 256-thread groups
  // each reduce over half of the keys, group 1 parks its partial in shared memory, group 0 adds and stores
  const int t256 = threadIdx.x & 255, grp = threadIdx.x >> 8;
  const int tx = t256 & 15, ty = t256 >> 4;
  float acc[4][6];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 6; ++c) acc[r][c] = 0.f;
  const int jh = (p.T + 1) >> 1;
  const int j0 = grp * jh, j1 = min(p.T, j0 + jh);
  for (int j = j0; j < j1; ++j) {
    const float4 p4 = *reinterpret_cast<const float4*>(PdT + j * LDT + 4 * ty);
    const float pv[4] = {p4.x, p4.y, p4.z, p4.w};
    float vv[6];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float2 v2 = *reinterpret_cast<const float2*>(Vs + j * LDR + 6 * tx + 2 * c);
      vv[2 * c] = v2.x; vv[2 * c + 1] = v2.y;
    }
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 6; ++c) acc[r][c] = fmaf(pv[r], vv[c], acc[r][c]);
  }
  float* park = Qt;                       // Q^T / K^T are dead after the scores: 64 x LDR floats fit in Q^T + K^T
  if (grp == 1) {
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 6; ++c) park[(4 * ty + r) * LDR + 6 * tx + c] = acc[r][c];
  }
  __syncthreads();
  if (grp == 0) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int i = 4 * ty + r;
      if (i >= p.T) continue;
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        const int d = 6 * tx + c;
        if (d < p.hd) p.ctx[((long long)i * p.B + b) * p.D + h * p.hd + d] = acc[r][c] + park[i * LDR + d];
      }
    }
  }
}

constexpr int NTB = 512;   // backward: two 256-thread groups split every reduction
__global__ void __launch_bounds__(NTB) attn_small_bwd_kernel(AttnP p) {
  extern __shared__ __align__(16) float sm[];
  const int b = blockIdx.x / p.H, h = blockIdx.x - b * p.H;
  float* Qs = sm; float* Ks = Qs + TM * LDR; float* Gs = Ks + TM * LDR;             // row-major Q, K, d(ctx)
  float* At = Gs + TM * LDR; float* Bt = At + HDM * LDT;                             // transposed scratch pair
  float* Ps = Bt + HDM * LDT; float* Pd = Ps + TM * LDT; float* dS = Pd + TM * LDT; float* dST = dS + TM * LDT;
  const long long rs = (long long)p.B * 3 * p.D;
  const float* base = p.qkv + (long long)b * 3 * p.D + h * p.hd;
  const float* gsrc = p.dctx + (long long)b * p.D + h * p.hd;
  const long long grs = (long long)p.B * p.D;
  const bool vec = (p.hd % 4 == 0) && (p.D % 4 == 0);
  load_head(base, rs, p.T, p.hd, vec, Qs, At);            // Q: row-major for dK, transposed for the scores
  load_head(base + p.D, rs, p.T, p.hd, vec, Ks, Bt);      // K
  load_head(gsrc, grs, p.T, p.hd, vec, Gs, nullptr);      // d(ctx)
  __syncthreads();
  gemm_tt(At, Bt, p.hd, p.scale, Ps);                     // recompute the scores ...
  __syncthreads();
  load_head(gsrc, grs, p.T, p.hd, vec, nullptr, At);      // scratch pair now holds G^T and V^T
  load_head(base + 2 * p.D, rs, p.T, p.hd, vec, nullptr, Bt);
  softmax_rows(p, b, h, Ps, Pd, LDT, 1);                  // ... and the probabilities (row-major dropped copy)
  __syncthreads();
  gemm_tt(At, Bt, p.hd, 1.f, dS);                         // dPd[i, j] = sum_d G[i, d] V[j, d]
  __syncthreads();
  {  // dS = P * (dP - rowsum(dP * P)), dP = dPd * mask/(1-p); written row-major and transposed
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float ik = p.drop_p > 0.f ? 1.f / (1.f - p.drop_p) : 1.f;
    for (int i = warp; i < TM; i += NTB / 32) {
      const uint64_t ibase = ((uint64_t)(b * p.H + h) * p.T + i) * p.T;
      float dp[2], pr[2];
      float dot = 0.f;
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int j = lane + 32 * half;
        const bool ok = i < p.T && j < p.T;
        pr[half] = ok ? Ps[i * LDT + j] : 0.f;
        const float m = (p.drop_p > 0.f && ok) ? dropout_scale(p.rng, p.site, ibase + j, p.drop_p, ik) : 1.f;
        dp[half] = ok ? dS[i * LDT + j] * m : 0.f;
        dot += dp[half] * pr[half];
      }
      dot = warp_sum(dot);
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int j = lane + 32 * half;
        const float v = pr[half] * (dp[half] - dot);
        dS[i * LDT + j] = v;
        dST[j * LDT + i] = v;
      }
    }
  }
  __syncthreads();
  // dQ[i, d] = scale * sum_j dS[i, j] K[j, d];  dK[j', d] = scale * sum_i dS[i, j'] Q[i, d];  dV[j', d] = sum_i Pd[i, j'] G[i, d]
  const int t256 = threadIdx.x & 255, grp = threadIdx.x >> 8;
  const int tx = t256 & 15, ty = t256 >> 4;
  float aq[4][6], ak[4][6], av[4][6];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 6; ++c) { aq[r][c] = 0.f; ak[r][c] = 0.f; av[r][c] = 0.f; }
  const int jh = (p.T + 1) >> 1;
  const int j0 = grp * jh, j1 = min(p.T, j0 + jh);        // each group reduces over half of the sequence
  for (int j = j0; j < j1; ++j) {
    const float4 s4 = *reinterpret_cast<const float4*>(dST + j * LDT + 4 * ty);   // dS[i = 4ty.., j]
    const float4 t4 = *reinterpret_cast<const float4*>(dS + j * LDT + 4 * ty);    // dS[i = j, j' = 4ty..]
    const float4 q4 = *reinterpret_cast<const float4*>(Pd + j * LDT + 4 * ty);    // Pd[i = j, j' = 4ty..]
    const float s_row[4] = {s4.x, s4.y, s4.z, s4.w}, s_col[4] = {t4.x, t4.y, t4.z, t4.w}, p_col[4] = {q4.x, q4.y, q4.z, q4.w};
    float kk[6], qq[6], gg[6];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float2 k2 = *reinterpret_cast<const float2*>(Ks + j * LDR + 6 * tx + 2 * c);
      const float2 q2 = *reinterpret_cast<const float2*>(Qs + j * LDR + 6 * tx + 2 * c);
      const float2 g2 = *reinterpret_cast<const float2*>(Gs + j * LDR + 6 * tx + 2 * c);
      kk[2 * c] = k2.x; kk[2 * c + 1] = k2.y; qq[2 * c] = q2.x; qq[2 * c + 1] = q2.y; gg[2 * c] = g2.x; gg[2 * c + 1] = g2.y;
    }
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        aq[r][c] = fmaf(s_row[r], kk[c], aq[r][c]);
        ak[r][c] = fmaf(s_col[r], qq[c], ak[r][c]);
        av[r][c] = fmaf(p_col[r], gg[c], av[r][c]);
      }
  }
  __syncthreads();                                          // all reads of Qs / Ks / Gs are done: reuse them
  if (grp == 1) {                                           // group 1 parks its partial sums in shared memory ...
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        const int o = (4 * ty + r) * LDR + 6 * tx + c;
        Qs[o] = aq[r][c]; Ks[o] = ak[r][c]; Gs[o] = av[r][c];
      }
  }
  __syncthreads();
  if (grp == 0) {                                           // ... group 0 adds them (fixed order) and writes dqkv
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int i = 4 * ty + r;
      if (i >= p.T) continue;
      float* o = p.dqkv + ((long long)i * p.B + b) * 3 * p.D + h * p.hd;
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        const int d = 6 * tx + c;
        const int so = i * LDR + d;
        if (d < p.hd) {
          o[d] = (aq[r][c] + Qs[so]) * p.scale; o[p.D + d] = (ak[r][c] + Ks[so]) * p.scale; o[2 * p.D + d] = av[r][c] + Gs[so];
        }
      }
    }
  }
}

size_t fwd_smem(int) { return sizeof(float) * (2 * HDM * LDT + TM * LDR + 2 * TM * LDT); }
size_t bwd_smem(int) { return sizeof(float) * (3 * TM * LDR + 2 * HDM * LDT + 4 * TM * LDT); }

}  // namespace

bool attn_small_supported(int T, int hd) {
  static int env = -1;
  if (env < 0) { const char* e = getenv("RD_ATTN_SMALL"); env = (e && e[0] == '0') ? 0 : 1; }
  return env == 1 && T <= TM && hd <= HDM;
}

static int ensure_smem_attrs() {
  RD_TRY(tc::ensure_max_smem((const void*)attn_small_fwd_kernel, (int)fwd_smem(HDM)));
  RD_TRY(tc::ensure_max_smem((const void*)attn_small_bwd_kernel, (int)bwd_smem(HDM)));
  return 0;
}

int attn_small_fwd(const float* qkv, const int64_t* lengths, int B, int H, int T, int hd, float drop_p,
                   const uint64_t* rng, uint32_t site, float* ctx, cudaStream_t st, DropRep rep) {
  AttnP p{};
  p.qkv = qkv; p.ctx = ctx; p.lengths = lengths; p.B = B; p.H = H; p.T = T; p.hd = hd; p.D = H * hd;
  p.scale = 1.f / sqrtf((float)hd); p.drop_p = drop_p; p.rng = rng; p.site = site; p.rep = rep;
  RD_TRY(ensure_smem_attrs());
  attn_small_fwd_kernel<<<B * H, 512, fwd_smem(hd), st>>>(p);
  RD_CHECK_LAUNCH("attn_small_fwd_kernel");
  return 0;
}

int attn_small_bwd(const float* qkv, const float* dctx, const int64_t* lengths, int B, int H, int T, int hd, float drop_p,
                   const uint64_t* rng, uint32_t site, float* dqkv, cudaStream_t st) {
  AttnP p{};
  p.qkv = qkv; p.dctx = dctx; p.dqkv = dqkv; p.lengths = lengths; p.B = B; p.H = H; p.T = T; p.hd = hd; p.D = H * hd;
  p.scale = 1.f / sqrtf((float)hd); p.drop_p = drop_p; p.rng = rng; p.site = site;
  RD_TRY(ensure_smem_attrs());
  attn_small_bwd_kernel<<<B * H, NTB, bwd_smem(hd), st>>>(p);
  RD_CHECK_LAUNCH("attn_small_bwd_kernel");
  return 0;
}

}  // namespace rd
