// Faithfulness of attributions by removal (rd_raindrop_v2_removal_curves, rd_raindrop_v2_removal_infidelity,
// rd_debug_removal_inputs; rd_model.cu orchestrates them).  The players, their removal and the expansion of a chunk's
// rows are those of the coalition calls: coalition_expand (rd_kernels.cu) with COALITION_ROWS reads the per-row keep
// tables written here.
//   removal_rank_kernel          one CTA per sample: 64-bit keys (order key << 32 | player) sorted in shared memory by a
//                                bitonic network, rank[b, g] = the position of player g.  Ties go to the lower index,
//                                -0 equals +0 and NaN sorts after every number.
//   removal_curve_keep_kernel    one thread per (row, player) of a chunk of (curve, count) pairs: deletion row (k, b)
//                                keeps the players with rank >= counts[k], insertion row (k, b) those with rank < counts[k].
//   removal_sample_keep_kernel   one thread per (row, player) of a chunk of replicates: player g of sample b is removed
//                                in replicate m iff Philox word b*P + g at site SITE_REMOVAL, key {seed, step + m}, is
//                                below floor(p_remove 2^32).
//   removal_curve_summary_kernel one thread per sample: F at the target of every curve point, the trapezoid AUCs and
//                                AOPC of logits and of fp64 softmax probabilities, each a serial fp64 sum in point order.
//   removal_moments_kernel       one CTA per sample: per replicate, in replicate order, a = sum of the removed players'
//                                attributions (a fixed tree: strided per-thread sums, then block_sum_fixed) and
//                                d = F(x) - F(row), added to the fp64 moments [1, a, d, a^2, ad, d^2] by one thread.
// Every sum has one order fixed by the shapes: the results are bitwise independent of the chunking.
#include <math.h>

#include "rd_kernels.cuh"
#include "rd_tc_common.cuh"

namespace rd {
namespace {

constexpr int TPB = 256, RANK_TPB = 1024, MOMENT_TPB = 256;
inline unsigned blocks_for(int64_t n) { return (unsigned)ceil_div(n, TPB); }

// Ascending order of the key is the order asked for; NaN (any payload) last, -0 as +0.
__device__ __forceinline__ uint32_t removal_order_key(float v, int order) {
  if (isnan(v)) return 0xffffffffu;
  const float w = order == RD_REMOVAL_ASCENDING ? v : (order == RD_REMOVAL_DESCENDING ? -v : -fabsf(v));
  const uint32_t u = w == 0.f ? 0u : __float_as_uint(w);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

struct RankArgs {
  const float* attr; int32_t* rank;
  int B, P, n, order;
};
__global__ void __launch_bounds__(RANK_TPB) removal_rank_kernel(const __grid_constant__ RankArgs a) {
  extern __shared__ unsigned long long keys[];
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  const float* phi = a.attr + (long long)b * a.P;
  for (int i = threadIdx.x; i < a.n; i += blockDim.x)
    keys[i] = i < a.P ? ((unsigned long long)removal_order_key(__ldg(phi + i), a.order) << 32) | (unsigned)i : ~0ull;
  __syncthreads();
  for (int k = 2; k <= a.n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < a.n; i += blockDim.x) {
        const int l = i ^ j;
        if (l > i) {
          const unsigned long long x = keys[i], y = keys[l];
          if ((x > y) == ((i & k) == 0)) { keys[i] = y; keys[l] = x; }
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < a.P; i += blockDim.x) a.rank[(long long)b * a.P + (unsigned)keys[i]] = i;
}

struct CurveKeepArgs {
  const int32_t* rank; const int32_t* counts; uint8_t* keep;
  long long q0;
  int K, nc, B, P;
};
__global__ void removal_curve_keep_kernel(const __grid_constant__ CurveKeepArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= (long long)a.nc * a.B * a.P) return;
  const long long j = o / a.P;
  const int g = (int)(o - j * a.P), pi = (int)(j / a.B), b = (int)(j - (long long)pi * a.B);
  const long long q = a.q0 + pi;
  const int insertion = q >= a.K, k = (int)(q - (insertion ? a.K : 0));
  const bool top = __ldg(a.rank + (long long)b * a.P + g) < __ldg(a.counts + k);
  a.keep[o] = insertion ? top : !top;
}

struct SampleKeepArgs {
  const uint64_t* rng; uint8_t* keep;
  unsigned long long below;      // floor(p_remove 2^32), 2^32 for p_remove = 1
  long long m0;
  int nc, B, P;
};
__global__ void removal_sample_keep_kernel(const __grid_constant__ SampleKeepArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= (long long)a.nc * a.B * a.P) return;
  const long long j = o / a.P;
  const int g = (int)(o - j * a.P), mi = (int)(j / a.B), b = (int)(j - (long long)mi * a.B);
  const uint64_t seed = __ldg(a.rng), step = __ldg(a.rng + 1) + (uint64_t)(a.m0 + mi);
  const RngKey key{(uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(step >> 32), (uint32_t)step};
  const uint64_t idx = (uint64_t)b * a.P + g;
  const uint4 w = dropout_block(key, SITE_REMOVAL, idx);
  const uint32_t s = (uint32_t)idx & 3u;
  const uint32_t word = s == 0 ? w.x : (s == 1 ? w.y : (s == 2 ? w.z : w.w));
  a.keep[o] = (unsigned long long)word >= a.below;
}

// p(target) of one logit row, softmax in fp64
__device__ double target_prob(const float* __restrict__ l, int ncls, int tgt) {
  double mx = __ldg(l);
  for (int c = 1; c < ncls; ++c) mx = fmax(mx, (double)__ldg(l + c));
  double s = 0.0;
  for (int c = 0; c < ncls; ++c) s += exp((double)__ldg(l + c) - mx);
  return exp((double)__ldg(l + tgt) - mx) / s;
}

struct SummaryArgs {
  const float* curve_logits; const float* ends; const int64_t* target; const int32_t* counts;
  float* values; double* summaries; int64_t* target_out;
  int K, B, P, ncls;
};
__global__ void removal_curve_summary_kernel(const __grid_constant__ SummaryArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.B) return;
  const int C = a.ncls;
  const float* x_row = a.ends + ((long long)a.B + b) * C;
  const int tgt = target_class(a.target, a.ends + (long long)a.B * C, b, C);
  a.target_out[b] = tgt;
  const double fx[2] = {(double)__ldg(x_row + tgt), target_prob(x_row, C, tgt)};
  double* out = a.summaries + (long long)b * RD_REMOVAL_SUMMARIES;
  for (int kind = 0; kind < 2; ++kind) {                 // logit, probability
    for (int curve = 0; curve < 2; ++curve) {            // deletion, insertion
      double auc = 0.0, aopc = 0.0, x_prev = 0.0, y_prev = 0.0;
      for (int k = 0; k < a.K; ++k) {
        const float* row = a.curve_logits + (((long long)curve * a.K + k) * a.B + b) * C;
        const double y = kind == 0 ? (double)__ldg(row + tgt) : target_prob(row, C, tgt);
        const double x = (double)__ldg(a.counts + k) / (double)a.P;
        if (kind == 0) a.values[((long long)curve * a.B + b) * a.K + k] = __ldg(row + tgt);
        if (k > 0) auc += (x - x_prev) * (y + y_prev) * 0.5;
        if (curve == 0) aopc += fx[kind] - y;
        x_prev = x;
        y_prev = y;
      }
      out[3 * kind + curve] = auc;
      if (curve == 0) out[3 * kind + 2] = aopc / a.K;
    }
  }
}

struct MomentArgs {
  const float* logits; const float* clean; const int64_t* target; const float* attr; const uint8_t* keep;
  double* moments; int64_t* target_out;
  int nc, B, P, ncls, first;
};
__global__ void __launch_bounds__(MOMENT_TPB) removal_moments_kernel(const __grid_constant__ MomentArgs a) {
  __shared__ double red[MOMENT_TPB / 32];
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x, C = a.ncls;
  const int tgt = target_class(a.target, a.clean, b, C);
  const double fx = __ldg(a.clean + (long long)b * C + tgt);
  const float* phi = a.attr + (long long)b * a.P;
  double* mom = a.moments + (long long)b * RD_REMOVAL_MOMENTS;
  double s[RD_REMOVAL_MOMENTS];
  if (threadIdx.x == 0) {
    if (a.first && a.target_out) a.target_out[b] = tgt;
    for (int i = 0; i < RD_REMOVAL_MOMENTS; ++i) s[i] = a.first ? 0.0 : mom[i];
  }
  for (int mi = 0; mi < a.nc; ++mi) {
    const long long row = (long long)mi * a.B + b;
    const uint8_t* keep = a.keep + row * a.P;
    double part = 0.0;
    for (int g = threadIdx.x; g < a.P; g += blockDim.x)
      if (!__ldg(keep + g)) part += (double)__ldg(phi + g);
    const double sa = block_sum_fixed(part, red);
    if (threadIdx.x == 0) {
      const double d = fx - (double)__ldg(a.logits + row * C + tgt);
      s[0] += 1.0; s[1] += sa; s[2] += d; s[3] += sa * sa; s[4] += sa * d; s[5] += d * d;
    }
  }
  if (threadIdx.x == 0)
    for (int i = 0; i < RD_REMOVAL_MOMENTS; ++i) mom[i] = s[i];
}

}  // namespace

int removal_rank(const float* attr, int B, int P, int order, int32_t* rank, cudaStream_t st) {
  RankArgs a;
  a.attr = attr; a.rank = rank; a.B = B; a.P = P; a.order = order;
  a.n = 1;
  while (a.n < P) a.n <<= 1;
  const int smem = a.n * (int)sizeof(unsigned long long);
  RD_TRY(tc::ensure_max_smem((const void*)removal_rank_kernel, RD_REMOVAL_MAX_PLAYERS * (int)sizeof(unsigned long long)));
  launch_pdl(removal_rank_kernel, dim3(B), dim3(RANK_TPB), smem, st, a);
  RD_CHECK_LAUNCH("removal_rank_kernel");
  return 0;
}

int removal_curve_keep(const int32_t* rank, const int32_t* counts, int K, int64_t q0, int nc, int B, int P, uint8_t* keep,
                       cudaStream_t st) {
  CurveKeepArgs a;
  a.rank = rank; a.counts = counts; a.keep = keep; a.q0 = q0; a.K = K; a.nc = nc; a.B = B; a.P = P;
  launch_pdl(removal_curve_keep_kernel, dim3(blocks_for((int64_t)nc * B * P)), dim3(TPB), 0, st, a);
  RD_CHECK_LAUNCH("removal_curve_keep_kernel");
  return 0;
}

int removal_sample_keep(const uint64_t* rng, uint64_t below, int64_t m0, int nc, int B, int P, uint8_t* keep,
                        cudaStream_t st) {
  SampleKeepArgs a;
  a.rng = rng; a.keep = keep; a.below = below; a.m0 = m0; a.nc = nc; a.B = B; a.P = P;
  launch_pdl(removal_sample_keep_kernel, dim3(blocks_for((int64_t)nc * B * P)), dim3(TPB), 0, st, a);
  RD_CHECK_LAUNCH("removal_sample_keep_kernel");
  return 0;
}

int removal_curve_summary(const float* curve_logits, const float* ends, const int64_t* target, const int32_t* counts,
                          int K, int B, int P, int ncls, float* values, double* summaries, int64_t* target_out,
                          cudaStream_t st) {
  SummaryArgs a;
  a.curve_logits = curve_logits; a.ends = ends; a.target = target; a.counts = counts; a.values = values;
  a.summaries = summaries; a.target_out = target_out; a.K = K; a.B = B; a.P = P; a.ncls = ncls;
  launch_pdl(removal_curve_summary_kernel, dim3(blocks_for(B)), dim3(TPB), 0, st, a);
  RD_CHECK_LAUNCH("removal_curve_summary_kernel");
  return 0;
}

int removal_moments(const float* logits, const float* clean, const int64_t* target, const float* attr,
                    const uint8_t* keep, int nc, int B, int P, int ncls, int first, double* moments, int64_t* target_out,
                    cudaStream_t st) {
  MomentArgs a;
  a.logits = logits; a.clean = clean; a.target = target; a.attr = attr; a.keep = keep; a.moments = moments;
  a.target_out = target_out; a.nc = nc; a.B = B; a.P = P; a.ncls = ncls; a.first = first;
  launch_pdl(removal_moments_kernel, dim3(B), dim3(MOMENT_TPB), 0, st, a);
  RD_CHECK_LAUNCH("removal_moments_kernel");
  return 0;
}

}  // namespace rd
