// Batch active learning over an unlabelled pool (rd_batch_bald, rd_badge).
//
// BatchBALD (Kirsch, van Amersfoort & Gal 2019).  p[m, n, c] = softmax(logits[m, n, :]) of replicate m < M.  Step i
// holds the chosen set A as rows of P_A [R, M]: row r is prod_{a in A} p[m, a, y_a^r] for one configuration y^r of A's
// labels, scaled so that its largest entry is 1, with its log-scale ls[r] (fp64) kept apart: products of up to k
// probabilities leave the fp32 range long before k = 200.  Exact mode (C^|A| <= n_configs) enumerates every
// configuration as a mixed-radix row (row j*C + c of A u {n} is row j of A times p[:, n, c]); sampled mode holds
// S = n_configs configurations drawn from the mixture.  Both reduce to one form:
//   H(y_A, y_n) ~= -sum_r w_r sum_c Q[r, (n, c)] (ls_r - log M + log Q[r, (n, c)]),   Q = P_A . p[:, n, :]
// with w_r = exp(ls_r) / M (exact: the joint probability is exp(ls_r) Q / M) or w_r = 1 / (S rowsum_r) (sampled:
// Kirsch's importance-weighted estimate, whose weight p(y^r, c) / p(y^r) is Q / rowsum, free of the scale).
//   ba_softmax_kernel   pT[(n C + c), m] = fp32(p) (rows padded to a multiple of 32 replicates with zeros) and the
//                       expected entropy E_m H(y_n | theta_m) in fp64, one thread per point, m in order.
//   ba_joint_kernel     the hot path.  One warpgroup per (64 configurations, 128 / C candidates) tile computes Q on
//                       the tensor cores in error-compensated 3xTF32 (wgmma m64n128k8; A = P_A rows from registers,
//                       B = pT rows written to shared memory in the 128-byte swizzle), and the epilogue turns Q into
//                       the tile's fp64 partial of the sum above: Q never leaves the SM.  Each entropy term uses the
//                       fp32 logarithm and is accumulated in fp64, over the tile's rows in a fixed order.
//   ba_reduce_kernel    score[n] = -(partials over configuration tiles, in order) - (sum of the chosen points' and n's
//                       expected entropies); chosen points score -inf.
//   ba_argmax_kernel    one CTA: the largest score, ties to the lowest index; records the pick on the device.
//   ba_expand_kernel / ba_sample_init_kernel / ba_sample_update_kernel  the rows of A u {pick}.
// Every sum has one order fixed by (N, M, C, n_configs) alone, so the result is bitwise independent of the candidate
// chunk; the host loop is launches only (no synchronisation), so a call can be captured in a CUDA graph.
//
// Sampled configurations: configuration s draws its replicate m_s = floor(U(s, 0) M) and, for the pick of step j, its
// label y = min{c : U(s, j + 1) < fp32 cumsum_c p[m_s, a_j, c]} (the largest class with p > 0 if rounding leaves none).
// U(s, j) is word 0 of the Philox block with key (seed lo, seed hi ^ step hi) and counter (s, j, SITE_BATCHBALD, step
// lo): U = (word >> 8) 2^-24 (labels), m_s = (word M) >> 32.  Nothing is redrawn when a point joins A.
//
// BADGE (Ash et al. 2020).  g_n = (p_n - e_{yhat_n}) (x) [h_n; 1]; the embedding is never formed:
//   |g_i - g_c|^2 = |a_i|^2 |h~_i|^2 + |a_c|^2 |h~_c|^2 - 2 (a_i . a_c)(h~_i . h~_c)   (a = p - e_yhat, h~ = [h; 1])
// with fp32 products taken in fp64, sums in fp64, clamped at 0.  The first centre has the largest norm; each later one is
// drawn with probability D^2 / sum D^2 by one fp64 uniform (key as above, counter (pick, 0, SITE_BADGE, step lo),
// U = ((w0 >> 5) 2^26 + (w1 >> 6)) 2^-53) against the CDF summed in tiles of BG_TILE points in index order.
#include <math.h>

#include "rd_tc_common.cuh"
#include "rd_wgmma_tf32.cuh"

namespace rd {
using namespace tc;
namespace {

constexpr uint32_t SITE_BATCHBALD = 105;   // Philox site of the sampled configurations (key {seed, step})
constexpr uint32_t SITE_BADGE = 106;       // Philox site of the D^2 draws (key {seed, step})

constexpr int BJ_BM = 64, BJ_BN = 128, BJ_BK = 32, BJ_THREADS = 128;
constexpr int BJ_B_TILE = BJ_BN * BJ_BK * 4;                 // 16 KB: the candidate rows, hi then lo
constexpr int BJ_QLD = BJ_BN + 4;                            // row stride of the staged Q tile (floats)
constexpr int BJ_SMEM = 1024 + 2 * BJ_B_TILE + BJ_BM * BJ_QLD * 4 + BJ_BM * 16 + 128 * 8;
constexpr int ROW_WARPS = 8;
constexpr int BG_TILE = 256;                                 // points per tile of the BADGE CDF

__device__ __forceinline__ uint4 active_block(uint64_t seed, uint64_t step, uint32_t c0, uint32_t c1, uint32_t site) {
  return philox4((uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(step >> 32), c0, c1, site, (uint32_t)step);
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- BatchBALD ---------------------------------------------------------------------------------------------------------
__global__ void ba_softmax_kernel(const float* __restrict__ logits, long long N, int M, int C, int Mp,
                                  float* __restrict__ pT, double* __restrict__ condent) {
  pdl_launch_dependents();
  pdl_wait();
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  double hsum = 0.0;
  for (int m = 0; m < M; ++m) {
    const float* l = logits + ((long long)m * N + n) * C;
    double mx = -INFINITY;
    for (int c = 0; c < C; ++c) mx = fmax(mx, (double)l[c]);
    double s = 0.0;
    for (int c = 0; c < C; ++c) s += exp((double)l[c] - mx);
    const double ls = log(s);
    double h = 0.0;
    for (int c = 0; c < C; ++c) {
      const double lp = ((double)l[c] - mx) - ls, p = exp(lp);
      h -= p * lp;
      pT[(n * C + c) * Mp + m] = (float)p;
    }
    hsum += h;
  }
  for (int m = M; m < Mp; ++m)
    for (int c = 0; c < C; ++c) pT[(n * C + c) * Mp + m] = 0.f;
  condent[n] = hsum / (double)M;
}

// The one configuration of the empty set: a row of ones, ls = 0, w = 1 / M.
__global__ void ba_init_kernel(int M, int Mp, float* __restrict__ rows, double* __restrict__ ls, double* __restrict__ w,
                               double* __restrict__ condA, long long N, uint8_t* __restrict__ chosen) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < Mp) rows[i] = i < M ? 1.f : 0.f;
  if (i == 0) { ls[0] = 0.0; w[0] = 1.0 / (double)M; condA[0] = 0.0; }
  if (i < N) chosen[i] = 0;
}

// partial[ct, j] = sum over the tile's rows r of w_r sum_c Q[r, (n, c)] (ls_r - log M + log Q), n = n_base + j.
// grid (configuration tiles, candidate tiles of the chunk).
__global__ void __launch_bounds__(BJ_THREADS, 3)
ba_joint_kernel(const float* __restrict__ rows, const double* __restrict__ ls, const double* __restrict__ w, int R,
                const float* __restrict__ pT, long long N, int M, int C, int Mp, long long n_base, int n_chunk,
                double* __restrict__ partial, long long partial_ld) {
  extern __shared__ uint8_t smem_raw[];
  pdl_launch_dependents();
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* sbase = smem_raw + (base - smem_u32(smem_raw));
  float* Qs = reinterpret_cast<float*>(sbase + 2 * BJ_B_TILE);
  double* sL = reinterpret_cast<double*>(sbase + 2 * BJ_B_TILE + BJ_BM * BJ_QLD * 4);
  double* sW = sL + BJ_BM;
  double* red = sW + BJ_BM;                                 // [128]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int NT = BJ_BN / C;                                 // candidates per tile
  const int r0 = blockIdx.x * BJ_BM;
  const long long c0 = (long long)blockIdx.y * NT;          // first candidate of the tile, within the chunk
  pdl_wait();
  const double logM = log((double)M);
  if (tid < BJ_BM) {
    const int r = r0 + tid;
    sL[tid] = r < R ? ls[r] - logM : 0.0;
    sW[tid] = r < R ? w[r] : 0.0;
  }
  float acc[BJ_BN / 2];
#pragma unroll
  for (int e = 0; e < BJ_BN / 2; ++e) acc[e] = 0.f;
  const int ra = r0 + 16 * warp + g, rb = ra + 8;
  const float* rowa = rows + (long long)ra * Mp;
  const float* rowb = rows + (long long)rb * Mp;
  for (int kb = 0; kb < Mp / BJ_BK; ++kb) {
    __syncthreads();                                        // the previous k-block's MMAs have retired (wait<0>)
    for (int e = tid; e < BJ_BN * BJ_BK; e += BJ_THREADS) {
      const int row = e >> 5, col = e & 31;
      const long long cand = c0 + row / C;
      float x = 0.f;
      if (row < NT * C && cand < n_chunk)
        x = __ldg(pT + ((n_base + cand) * C + row % C) * (long long)Mp + kb * BJ_BK + col);
      const uint32_t off = sw128_offset(row, col);
      *reinterpret_cast<uint32_t*>(sbase + off) = tf32_hi(x);
      *reinterpret_cast<uint32_t*>(sbase + BJ_B_TILE + off) = tf32_lo(x);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    uint32_t ah[BJ_BK / 8][4], al[BJ_BK / 8][4];
#pragma unroll
    for (int ks = 0; ks < BJ_BK / 8; ++ks) {
      const int col = kb * BJ_BK + ks * 8 + t;
      float x[4] = {0.f, 0.f, 0.f, 0.f};
      if (ra < R) { x[0] = __ldg(rowa + col); x[2] = __ldg(rowa + col + 4); }
      if (rb < R) { x[1] = __ldg(rowb + col); x[3] = __ldg(rowb + col + 4); }
#pragma unroll
      for (int i = 0; i < 4; ++i) { ah[ks][i] = tf32_hi(x[i]); al[ks][i] = tf32_lo(x[i]); }
    }
#pragma unroll
    for (int e = 0; e < BJ_BN / 2; ++e) fence_operand(acc[e]);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < BJ_BK / 8; ++ks) {
      const uint64_t bh = wgmma_desc_sw128(base + (uint32_t)ks * 32u);
      wgmma_tf32<BJ_BN>(acc, al[ks], bh);                   // small terms first
      wgmma_tf32<BJ_BN>(acc, ah[ks], wgmma_desc_sw128(base + BJ_B_TILE + (uint32_t)ks * 32u));
      wgmma_tf32<BJ_BN>(acc, ah[ks], bh);
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int e = 0; e < BJ_BN / 2; ++e) fence_operand(acc[e]);
  }
  // ---- epilogue: Q to shared memory, then (candidate, row part) per thread --------------------------------------------
#pragma unroll
  for (int j = 0; j < BJ_BN / 8; ++j) {
    const int col = 8 * j + 2 * t, row = 16 * warp + g;
    Qs[row * BJ_QLD + col] = acc[4 * j];
    Qs[row * BJ_QLD + col + 1] = acc[4 * j + 1];
    Qs[(row + 8) * BJ_QLD + col] = acc[4 * j + 2];
    Qs[(row + 8) * BJ_QLD + col + 1] = acc[4 * j + 3];
  }
  __syncthreads();
  int parts = 1;
  while (2 * parts * NT <= BJ_THREADS) parts *= 2;           // a power of two: rows per part = 64 / parts
  const int cand = tid % NT, part = tid / NT, rpp = BJ_BM / parts;
  double s = 0.0;
  if (part < parts && c0 + cand < n_chunk) {
    for (int rr = part * rpp; rr < (part + 1) * rpp; ++rr) {
      if (r0 + rr >= R) break;
      const double Lr = sL[rr];
      double v = 0.0;
      for (int c = 0; c < C; ++c) {
        const float q = Qs[rr * BJ_QLD + cand * C + c];
        if (q > 0.f) v += (double)q * (Lr + (double)logf(q));
      }
      s += sW[rr] * v;
    }
  }
  red[tid] = s;
  __syncthreads();
  if (part == 0 && cand < NT && c0 + cand < n_chunk) {
    double tot = 0.0;
    for (int p = 0; p < parts; ++p) tot += red[p * NT + cand];
    partial[(long long)blockIdx.x * partial_ld + c0 + cand] = tot;
  }
}

__global__ void ba_reduce_kernel(const double* __restrict__ partial, long long partial_ld, int n_tiles, long long n_base,
                                 int n_chunk, const double* __restrict__ condent, const double* __restrict__ condA,
                                 const uint8_t* __restrict__ chosen, double* __restrict__ score,
                                 double* __restrict__ bald) {
  pdl_launch_dependents();
  pdl_wait();
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_chunk) return;
  const long long n = n_base + j;
  double h = 0.0;
  for (int tt = 0; tt < n_tiles; ++tt) h += partial[(long long)tt * partial_ld + j];
  const double sc = -h - (condA[0] + condent[n]);
  score[n] = chosen[n] ? -INFINITY : sc;
  if (bald) bald[n] = sc;
}

// The largest vals[n] over the unchosen n, ties to the lowest index: out_idx[0] = n, chosen[n] = 1; with out_val,
// out_val[0] = vals[n];
// with cond, condA[0] += cond[n]; with exact_out, exact_out[0] = exact.  One CTA of 1024 threads.
__global__ void __launch_bounds__(1024) ba_argmax_kernel(const double* __restrict__ vals, long long N,
                                                          uint8_t* __restrict__ chosen, int64_t* __restrict__ out_idx,
                                                          double* __restrict__ out_val, const double* __restrict__ cond,
                                                          double* __restrict__ condA, uint8_t* __restrict__ exact_out,
                                                          int exact) {
  __shared__ double sv[32];
  __shared__ long long si[32];
  pdl_launch_dependents();
  pdl_wait();
  double bv = -INFINITY;
  long long bi = -1;
  for (long long n = threadIdx.x; n < N; n += blockDim.x) {
    if (chosen[n]) continue;
    const double v = vals[n];
    if (bi < 0 || v > bv) { bv = v; bi = n; }
  }
  auto better = [](double v1, long long i1, double v2, long long i2) {
    if (i2 < 0) return true;
    if (i1 < 0) return false;
    return v1 > v2 || (v1 == v2 && i1 < i2);
  };
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const long long oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (!better(bv, bi, ov, oi)) { bv = ov; bi = oi; }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { sv[warp] = bv; si[warp] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w2 = 1; w2 < (int)(blockDim.x >> 5); ++w2)
      if (!better(bv, bi, sv[w2], si[w2])) { bv = sv[w2]; bi = si[w2]; }
    if (bi < 0) bi = 0;                                     // k <= N on the host: not reached
    out_idx[0] = bi;
    if (out_val) out_val[0] = vals[bi];
    chosen[bi] = 1;
    if (cond) condA[0] += cond[bi];
    if (exact_out) exact_out[0] = (uint8_t)exact;
  }
}

// Row j*C + c of the new set = row j of the old one times p[:, a, c], rescaled to max 1.  One warp per new row.
__global__ void __launch_bounds__(32 * ROW_WARPS) ba_expand_kernel(const float* __restrict__ rows, const double* __restrict__ ls,
                                                                    int R, const float* __restrict__ pT, int M, int C,
                                                                    int Mp, const int64_t* __restrict__ pick,
                                                                    float* __restrict__ out, double* __restrict__ ls_out,
                                                                    double* __restrict__ w_out) {
  pdl_launch_dependents();
  pdl_wait();
  const long long r = (long long)blockIdx.x * ROW_WARPS + threadIdx.x / 32;
  const int lane = threadIdx.x & 31;
  if (r >= (long long)R * C) return;
  const long long j = r / C;
  const int c = (int)(r % C);
  const long long a = pick[0];
  const float* src = rows + j * Mp;
  const float* p = pT + (a * C + c) * (long long)Mp;
  double mx = 0.0;
  for (int m = lane; m < M; m += 32) mx = fmax(mx, (double)src[m] * (double)p[m]);
  mx = warp_max_d(mx);
  float* dst = out + r * Mp;
  for (int m = lane; m < Mp; m += 32) dst[m] = (m < M && mx > 0.0) ? (float)((double)src[m] * (double)p[m] / mx) : 0.f;
  if (lane == 0) {
    const double l = mx > 0.0 ? ls[j] + log(mx) : -INFINITY;
    ls_out[r] = l;
    w_out[r] = mx > 0.0 ? exp(l) / (double)M : 0.0;
  }
}

// The sampled configurations' replicates m_s and rows of ones.
__global__ void ba_sample_init_kernel(int S, int M, int Mp, uint64_t seed, uint64_t step, int32_t* __restrict__ msamp,
                                      float* __restrict__ rows, double* __restrict__ ls) {
  pdl_launch_dependents();
  pdl_wait();
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)S * Mp) return;
  const int s = (int)(e / Mp), m = (int)(e % Mp);
  rows[e] = m < M ? 1.f : 0.f;
  if (m == 0) {
    const uint32_t wd = active_block(seed, step, (uint32_t)s, 0u, SITE_BATCHBALD).x;
    msamp[s] = (int32_t)(((uint64_t)wd * (uint64_t)M) >> 32);
    ls[s] = 0.0;
  }
}

// Configuration s draws its label for the pick of step j from its own replicate and multiplies its row by p[:, a, y].
// One warp per configuration.
__global__ void __launch_bounds__(32 * ROW_WARPS) ba_sample_update_kernel(float* __restrict__ rows, double* __restrict__ ls,
                                                                           double* __restrict__ w, int S,
                                                                           const int32_t* __restrict__ msamp,
                                                                           const float* __restrict__ pT, int M, int C,
                                                                           int Mp, const int64_t* __restrict__ picks,
                                                                           int j, uint64_t seed, uint64_t step) {
  pdl_launch_dependents();
  pdl_wait();
  const int s = blockIdx.x * ROW_WARPS + threadIdx.x / 32;
  const int lane = threadIdx.x & 31;
  if (s >= S) return;
  const long long a = picks[j];
  const int ms = msamp[s];
  const uint32_t wd = active_block(seed, step, (uint32_t)s, (uint32_t)(j + 1), SITE_BATCHBALD).x;
  const float u = (float)(wd >> 8) * (1.0f / 16777216.0f);
  int y = -1, last = 0;
  float cum = 0.f;
  for (int c = 0; c < C; ++c) {
    const float pc = pT[(a * C + c) * (long long)Mp + ms];
    if (pc > 0.f) last = c;
    cum += pc;
    if (y < 0 && u < cum) y = c;
  }
  if (y < 0) y = last;
  const float* p = pT + (a * C + y) * (long long)Mp;
  float* row = rows + (long long)s * Mp;
  double mx = 0.0;
  for (int m = lane; m < M; m += 32) mx = fmax(mx, (double)row[m] * (double)p[m]);
  mx = warp_max_d(mx);
  double sum = 0.0;
  for (int m = lane; m < M; m += 32) {
    const float v = mx > 0.0 ? (float)((double)row[m] * (double)p[m] / mx) : 0.f;
    row[m] = v;
    sum += (double)v;
  }
  sum = warp_sum_d(sum);
  if (lane == 0) {
    ls[s] = mx > 0.0 ? ls[s] + log(mx) : -INFINITY;
    w[s] = mx > 0.0 ? 1.0 / ((double)S * sum) : 0.0;
  }
}

// ---- BADGE -------------------------------------------------------------------------------------------------------------
// a = p - e_yhat (fp64), na = |a|^2, nh = |h|^2 + 1, norm = na nh, D2 = +inf; d2_first = +inf (the first pick, by
// norm, has no D^2).  One warp per point.
__global__ void __launch_bounds__(32 * ROW_WARPS) bg_prep_kernel(const float* __restrict__ hidden,
                                                                  const float* __restrict__ logits, long long N, int F,
                                                                  int C, double* __restrict__ a, double* __restrict__ na,
                                                                  double* __restrict__ nh, double* __restrict__ norm,
                                                                  double* __restrict__ d2, uint8_t* __restrict__ chosen,
                                                                  double* __restrict__ d2_first) {
  pdl_launch_dependents();
  pdl_wait();
  const long long n = (long long)blockIdx.x * ROW_WARPS + threadIdx.x / 32;
  const int lane = threadIdx.x & 31;
  if (n >= N) return;
  const float* h = hidden + n * F;
  double hh = 0.0;
  for (int f = lane; f < F; f += 32) { const double v = h[f]; hh = fma(v, v, hh); }
  hh = warp_sum_d(hh) + 1.0;
  if (lane == 0) {
    const float* l = logits + n * C;
    int yhat = 0;
    for (int c = 1; c < C; ++c)
      if (l[c] > l[yhat]) yhat = c;
    double mx = -INFINITY;
    for (int c = 0; c < C; ++c) mx = fmax(mx, (double)l[c]);
    double s = 0.0;
    for (int c = 0; c < C; ++c) s += exp((double)l[c] - mx);
    double aa = 0.0;
    for (int c = 0; c < C; ++c) {
      const double v = exp((double)l[c] - mx) / s - (c == yhat ? 1.0 : 0.0);
      a[n * C + c] = v;
      aa = fma(v, v, aa);
    }
    na[n] = aa;
    nh[n] = hh;
    norm[n] = aa * hh;
    d2[n] = INFINITY;
    chosen[n] = 0;
    if (n == 0) d2_first[0] = INFINITY;
  }
}

// D2[i] = min(D2[i], max(0, norm_i + norm_c - 2 (a_i . a_c)(h_i . h_c + 1))), 0 for chosen points.  One warp per point.
__global__ void __launch_bounds__(32 * ROW_WARPS) bg_update_kernel(const float* __restrict__ hidden, long long N, int F,
                                                                    int C, const double* __restrict__ a,
                                                                    const double* __restrict__ norm,
                                                                    const int64_t* __restrict__ pick,
                                                                    const uint8_t* __restrict__ chosen,
                                                                    double* __restrict__ d2) {
  pdl_launch_dependents();
  pdl_wait();
  const long long i = (long long)blockIdx.x * ROW_WARPS + threadIdx.x / 32;
  const int lane = threadIdx.x & 31;
  if (i >= N) return;
  const long long c = pick[0];
  const float* hi = hidden + i * F;
  const float* hc = hidden + c * F;
  double dot = 0.0;
  for (int f = lane; f < F; f += 32) dot = fma((double)hi[f], (double)hc[f], dot);
  dot = warp_sum_d(dot) + 1.0;
  if (lane == 0) {
    if (chosen[i]) { d2[i] = 0.0; return; }
    double ac = 0.0;
    for (int k = 0; k < C; ++k) ac = fma(a[i * C + k], a[c * C + k], ac);
    const double d = fmax(0.0, norm[i] + norm[c] - 2.0 * (ac * dot));
    d2[i] = fmin(d2[i], d);
  }
}

// One draw of the D^2 sampling for pick `pick_no`: tile sums (BG_TILE points each, in index order), the target
// U * total, the tile and then the point where the running sum first exceeds it.  out_idx / out_d2 / chosen as
// ba_argmax_kernel.  One CTA of 1024 threads.
__global__ void __launch_bounds__(1024) bg_sample_kernel(const double* __restrict__ d2, long long N,
                                                          uint8_t* __restrict__ chosen, uint64_t seed, uint64_t step,
                                                          int pick_no, double* __restrict__ tile_sum,
                                                          int64_t* __restrict__ out_idx, double* __restrict__ out_d2) {
  __shared__ long long s_pick;
  pdl_launch_dependents();
  pdl_wait();
  const long long n_tiles = (N + BG_TILE - 1) / BG_TILE;
  for (long long tt = threadIdx.x; tt < n_tiles; tt += blockDim.x) {
    double s = 0.0;
    const long long e = min(N, (tt + 1) * BG_TILE);
    for (long long n = tt * BG_TILE; n < e; ++n) s += d2[n];
    tile_sum[tt] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double total = 0.0;
    for (long long tt = 0; tt < n_tiles; ++tt) total += tile_sum[tt];
    long long pick = -1;
    if (total > 0.0) {
      const uint4 w = active_block(seed, step, (uint32_t)pick_no, 0u, SITE_BADGE);
      const double u = (double)(((uint64_t)(w.x >> 5) << 26) | (uint64_t)(w.y >> 6)) * (1.0 / 9007199254740992.0);
      const double target = u * total;
      double cum = 0.0;
      long long tt = 0;
      for (; tt < n_tiles; ++tt) {
        if (cum + tile_sum[tt] > target) break;
        cum += tile_sum[tt];
      }
      if (tt < n_tiles) {
        const long long e = min(N, (tt + 1) * BG_TILE);
        for (long long n = tt * BG_TILE; n < e; ++n) {
          cum += d2[n];
          if (cum > target) { pick = n; break; }
        }
      }
      if (pick < 0)                                         // rounding at the top of the CDF: the last point with D^2 > 0
        for (long long n = N - 1; n >= 0; --n)
          if (d2[n] > 0.0) { pick = n; break; }
    }
    if (pick < 0)                                           // every unchosen D^2 is 0: the lowest unchosen index
      for (long long n = 0; n < N; ++n)
        if (!chosen[n]) { pick = n; break; }
    s_pick = pick;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const long long p = s_pick < 0 ? 0 : s_pick;
    out_idx[0] = p;
    out_d2[0] = d2[p];
    chosen[p] = 1;
  }
}

// ---- host --------------------------------------------------------------------------------------------------------------
struct BaLayout {
  int Mp, S, n_ctiles;
  size_t pT, condent, rows0, rows1, ls0, ls1, w0, w1, msamp, partial, score, chosen, condA, total;
};

bool ba_args_ok(int64_t N, int32_t M, int32_t C, int32_t n_configs, int64_t chunk) {
  return N >= 1 && N <= (1ll << 31) / RD_ACTIVE_MAX_CLASSES && M >= 1 && M <= RD_ACTIVE_MAX_REPLICATES && C >= 2 &&
         C <= RD_ACTIVE_MAX_CLASSES && n_configs >= 1 && n_configs <= RD_ACTIVE_MAX_CONFIGS && chunk >= 1;
}

BaLayout ba_layout(int64_t N, int32_t M, int32_t C, int32_t n_configs, int64_t chunk) {
  BaLayout l{};
  l.Mp = (int)round_up(M, BJ_BK);
  l.S = n_configs;
  const int64_t Sp = round_up(n_configs, BJ_BM);
  l.n_ctiles = (int)(Sp / BJ_BM);
  const int64_t ch = chunk < N ? chunk : N;
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += (bytes + 255) / 256 * 256; return o; };
  l.pT = take((size_t)N * C * l.Mp * 4);
  l.condent = take((size_t)N * 8);
  l.rows0 = take((size_t)Sp * l.Mp * 4);
  l.rows1 = take((size_t)Sp * l.Mp * 4);
  l.ls0 = take((size_t)Sp * 8);
  l.ls1 = take((size_t)Sp * 8);
  l.w0 = take((size_t)Sp * 8);
  l.w1 = take((size_t)Sp * 8);
  l.msamp = take((size_t)Sp * 4);
  l.partial = take((size_t)l.n_ctiles * ch * 8);
  l.score = take((size_t)N * 8);
  l.chosen = take((size_t)N);
  l.condA = take(8);
  l.total = off;
  return l;
}

struct BgLayout { size_t a, na, nh, norm, d2, chosen, tiles, total; };

BgLayout bg_layout(int64_t N, int32_t C) {
  BgLayout l{};
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += (bytes + 255) / 256 * 256; return o; };
  l.a = take((size_t)N * C * 8);
  l.na = take((size_t)N * 8);
  l.nh = take((size_t)N * 8);
  l.norm = take((size_t)N * 8);
  l.d2 = take((size_t)N * 8);
  l.chosen = take((size_t)N);
  l.tiles = take((size_t)ceil_div(N, BG_TILE) * 8);
  l.total = off;
  return l;
}

bool bg_args_ok(int64_t N, int32_t F, int32_t C) {
  return N >= 1 && N <= (1ll << 31) && F >= 1 && C >= 2 && C <= RD_ACTIVE_MAX_CLASSES;
}

}  // namespace
}  // namespace rd

using namespace rd;

extern "C" {

size_t rd_batch_bald_scratch_bytes(int64_t N, int32_t M, int32_t C, int32_t n_configs, int64_t chunk) {
  if (!ba_args_ok(N, M, C, n_configs, chunk)) return 0;
  return ba_layout(N, M, C, n_configs, chunk).total;
}

int rd_batch_bald(const float* logits, int64_t N, int32_t M, int32_t C, int32_t k, int32_t n_configs, uint64_t seed,
                  uint64_t step, int64_t chunk, void* scratch, int64_t* indices, double* scores, uint8_t* exact,
                  double* bald, void* stream) {
  const char* fn = "rd_batch_bald";
  if (!logits || !scratch || !indices || !scores || !exact || !bald) { set_error("%s: NULL argument", fn); return -2; }
  if (!ba_args_ok(N, M, C, n_configs, chunk) || k < 1 || k > N) {
    set_error("%s: bad sizes (N=%lld M=%d C=%d k=%d n_configs=%d chunk=%lld; 2 <= C <= %d, M <= %d, n_configs <= %d, "
              "1 <= k <= N)", fn, (long long)N, M, C, k, n_configs, (long long)chunk, RD_ACTIVE_MAX_CLASSES,
              RD_ACTIVE_MAX_REPLICATES, RD_ACTIVE_MAX_CONFIGS);
    return -2;
  }
  if (reinterpret_cast<uintptr_t>(scratch) & 255) { set_error("%s: scratch must be 256-byte aligned", fn); return -2; }
  const BaLayout l = ba_layout(N, M, C, n_configs, chunk);
  uint8_t* sb = static_cast<uint8_t*>(scratch);
  float* pT = reinterpret_cast<float*>(sb + l.pT);
  double* condent = reinterpret_cast<double*>(sb + l.condent);
  float* rows[2] = {reinterpret_cast<float*>(sb + l.rows0), reinterpret_cast<float*>(sb + l.rows1)};
  double* ls[2] = {reinterpret_cast<double*>(sb + l.ls0), reinterpret_cast<double*>(sb + l.ls1)};
  double* w[2] = {reinterpret_cast<double*>(sb + l.w0), reinterpret_cast<double*>(sb + l.w1)};
  int32_t* msamp = reinterpret_cast<int32_t*>(sb + l.msamp);
  double* partial = reinterpret_cast<double*>(sb + l.partial);
  double* score = reinterpret_cast<double*>(sb + l.score);
  uint8_t* chosen = sb + l.chosen;
  double* condA = reinterpret_cast<double*>(sb + l.condA);
  const cudaStream_t st = (cudaStream_t)stream;
  const int64_t ch = chunk < N ? chunk : N;
  const int NT = BJ_BN / C;
  RD_TRY(ensure_max_smem((const void*)ba_joint_kernel, BJ_SMEM));

  launch_pdl(ba_softmax_kernel, dim3((unsigned)ceil_div(N, 128)), dim3(128), 0, st, logits, (long long)N, (int)M, (int)C,
             l.Mp, pT, condent);
  RD_CHECK_LAUNCH("ba_softmax_kernel");
  const int64_t init_n = N > l.Mp ? N : l.Mp;
  launch_pdl(ba_init_kernel, dim3((unsigned)ceil_div(init_n, 256)), dim3(256), 0, st, (int)M, l.Mp, rows[0], ls[0], w[0],
             condA, (long long)N, chosen);
  RD_CHECK_LAUNCH("ba_init_kernel");

  int cur = 0;
  int64_t R = 1;                                            // C^i while exact
  bool ex = true;
  for (int i = 0; i < k; ++i) {
    const int n_tiles = (int)ceil_div(R, BJ_BM);
    for (int64_t n0 = 0; n0 < N; n0 += ch) {
      const int nc = (int)((N - n0) < ch ? (N - n0) : ch);
      launch_pdl(ba_joint_kernel, dim3((unsigned)n_tiles, (unsigned)ceil_div(nc, NT)), dim3(BJ_THREADS), BJ_SMEM, st,
                 (const float*)rows[cur], (const double*)ls[cur], (const double*)w[cur], (int)R, (const float*)pT,
                 (long long)N, (int)M, (int)C, l.Mp, (long long)n0, nc, partial, (long long)ch);
      RD_CHECK_LAUNCH("ba_joint_kernel");
      launch_pdl(ba_reduce_kernel, dim3((unsigned)ceil_div(nc, 256)), dim3(256), 0, st, (const double*)partial,
                 (long long)ch, n_tiles, (long long)n0, nc, (const double*)condent, (const double*)condA,
                 (const uint8_t*)chosen, score, i == 0 ? bald : (double*)nullptr);
      RD_CHECK_LAUNCH("ba_reduce_kernel");
    }
    launch_pdl(ba_argmax_kernel, dim3(1), dim3(1024), 0, st, (const double*)score, (long long)N, chosen, indices + i,
               scores + i, (const double*)condent, condA, exact + i, (int)ex);
    RD_CHECK_LAUNCH("ba_argmax_kernel");
    if (i + 1 == k) break;
    if (ex && R * C <= n_configs) {                         // stays exact: expand by C
      launch_pdl(ba_expand_kernel, dim3((unsigned)ceil_div(R * C, ROW_WARPS)), dim3(32 * ROW_WARPS), 0, st,
                 (const float*)rows[cur], (const double*)ls[cur], (int)R, (const float*)pT, (int)M, (int)C, l.Mp,
                 (const int64_t*)(indices + i), rows[1 - cur], ls[1 - cur], w[1 - cur]);
      RD_CHECK_LAUNCH("ba_expand_kernel");
      cur = 1 - cur;
      R *= C;
      continue;
    }
    const int first = ex ? 0 : i;                           // at the switch, replay every pick so far
    if (ex) {
      cur = 1 - cur;
      launch_pdl(ba_sample_init_kernel, dim3((unsigned)ceil_div((int64_t)n_configs * l.Mp, 256)), dim3(256), 0, st,
                 (int)n_configs, (int)M, l.Mp, seed, step, msamp, rows[cur], ls[cur]);
      RD_CHECK_LAUNCH("ba_sample_init_kernel");
      ex = false;
      R = n_configs;
    }
    for (int j = first; j <= i; ++j) {
      launch_pdl(ba_sample_update_kernel, dim3((unsigned)ceil_div(n_configs, ROW_WARPS)), dim3(32 * ROW_WARPS), 0, st,
                 rows[cur], ls[cur], w[cur], (int)n_configs, (const int32_t*)msamp, (const float*)pT, (int)M, (int)C,
                 l.Mp, (const int64_t*)indices, j, seed, step);
      RD_CHECK_LAUNCH("ba_sample_update_kernel");
    }
  }
  return 0;
}

size_t rd_badge_scratch_bytes(int64_t N, int32_t F, int32_t C) {
  if (!bg_args_ok(N, F, C)) return 0;
  return bg_layout(N, C).total;
}

int rd_badge(const float* hidden, const float* logits, int64_t N, int32_t F, int32_t C, int32_t k, uint64_t seed,
             uint64_t step, void* scratch, int64_t* indices, double* d2_out, void* stream) {
  const char* fn = "rd_badge";
  if (!hidden || !logits || !scratch || !indices || !d2_out) { set_error("%s: NULL argument", fn); return -2; }
  if (!bg_args_ok(N, F, C) || k < 1 || k > N) {
    set_error("%s: bad sizes (N=%lld F=%d C=%d k=%d; 2 <= C <= %d, 1 <= k <= N)", fn, (long long)N, F, C, k,
              RD_ACTIVE_MAX_CLASSES);
    return -2;
  }
  if (reinterpret_cast<uintptr_t>(scratch) & 255) { set_error("%s: scratch must be 256-byte aligned", fn); return -2; }
  const BgLayout l = bg_layout(N, C);
  uint8_t* sb = static_cast<uint8_t*>(scratch);
  double* a = reinterpret_cast<double*>(sb + l.a);
  double* na = reinterpret_cast<double*>(sb + l.na);
  double* nh = reinterpret_cast<double*>(sb + l.nh);
  double* norm = reinterpret_cast<double*>(sb + l.norm);
  double* d2 = reinterpret_cast<double*>(sb + l.d2);
  uint8_t* chosen = sb + l.chosen;
  double* tiles = reinterpret_cast<double*>(sb + l.tiles);
  const cudaStream_t st = (cudaStream_t)stream;
  const dim3 rgrid((unsigned)ceil_div(N, ROW_WARPS)), rblock(32 * ROW_WARPS);
  launch_pdl(bg_prep_kernel, rgrid, rblock, 0, st, hidden, logits, (long long)N, (int)F, (int)C, a, na, nh, norm, d2,
             chosen, d2_out);
  RD_CHECK_LAUNCH("bg_prep_kernel");
  launch_pdl(ba_argmax_kernel, dim3(1), dim3(1024), 0, st, (const double*)norm, (long long)N, chosen, indices, (double*)nullptr,
             (const double*)nullptr, (double*)nullptr, (uint8_t*)nullptr, 0);
  RD_CHECK_LAUNCH("ba_argmax_kernel");
  for (int i = 1; i < k; ++i) {
    launch_pdl(bg_update_kernel, rgrid, rblock, 0, st, hidden, (long long)N, (int)F, (int)C, (const double*)a,
               (const double*)norm, (const int64_t*)(indices + i - 1), (const uint8_t*)chosen, d2);
    RD_CHECK_LAUNCH("bg_update_kernel");
    launch_pdl(bg_sample_kernel, dim3(1), dim3(1024), 0, st, (const double*)d2, (long long)N, chosen, seed, step, i,
               tiles, indices + i, d2_out + i);
    RD_CHECK_LAUNCH("bg_sample_kernel");
  }
  return 0;
}

}  // extern "C"
