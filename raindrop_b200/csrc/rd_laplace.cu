// Laplace approximation of Raindrop_v2 (MacKay 1992; Ritter et al. 2018; Daxberger et al. 2021): the kernels behind the
// per-sample logit covariance of rd_model.cu and the Monte Carlo predictive.
//   laplace_seed_kernel      d_logits = e_c / B, the one-hot seed of logit c for the rows path.
//   laplace_gram_kernel<NC>  one CTA per (column slab, sample): the slab's fp64 partial sums of
//                            w_j J~_{c,j} J~_{c',j} (c <= c') over the sample's NC rows; float4 loads, products in fp32.
//   laplace_fold_kernel      per (sample, pair) the slab partials added in slab order, written to cov[b, c, c'] and
//                            cov[b, c', c].  No atomics: bitwise reproducible, and a sample's result depends on its own
//                            rows only.
//   laplace_chol_kernel      per sample the lower Cholesky factor of Sigma_b in fp64, safe for semi-definite input.
//   laplace_draw_kernel      per (replicate, sample) f = mu_b + L_b eps, eps from Philox4x32-10 at site 99.
#include "rd_kernels.cuh"

namespace rd {
namespace {

constexpr uint32_t SITE_LAPLACE = 99;    // Philox site of the predictive draws (96-98: DP noise, Fisher labels, PGD start)
constexpr int GRAM_THREADS = 256;
constexpr int GRAM_SLAB = 16384;         // columns per CTA: 16 float4 per thread, 64 KiB of each row

__global__ void laplace_seed_kernel(float* __restrict__ d, int B, int ncls, int c) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B * ncls) d[i] = (i % ncls == c) ? 1.0f / (float)B : 0.0f;
}

template <int NC>
__global__ void __launch_bounds__(GRAM_THREADS) laplace_gram_kernel(const float* __restrict__ G, int B, long long ldg,
                                                                   const float* __restrict__ w, double* __restrict__ partial) {
  constexpr int NP = NC * (NC + 1) / 2;
  __shared__ double red[GRAM_THREADS / 32][NP];
  pdl_launch_dependents();
  pdl_wait();
  const int slab = blockIdx.x, b = blockIdx.y;
  const long long c0 = (long long)slab * GRAM_SLAB;
  const long long n4 = (ldg - c0 < GRAM_SLAB ? ldg - c0 : GRAM_SLAB) >> 2;
  const float4* w4 = reinterpret_cast<const float4*>(w + c0);
  const float4* row[NC];
#pragma unroll
  for (int c = 0; c < NC; ++c) row[c] = reinterpret_cast<const float4*>(G + ((long long)c * B + b) * ldg + c0);
  double acc[NP];
#pragma unroll
  for (int p = 0; p < NP; ++p) acc[p] = 0.0;
#pragma unroll 2
  for (long long i = threadIdx.x; i < n4; i += GRAM_THREADS) {
    const float4 wv = __ldg(w4 + i);
    float4 t[NC];
#pragma unroll
    for (int c = 0; c < NC; ++c) t[c] = __ldcs(row[c] + i);        // read once: do not keep the rows in L2
    int p = 0;
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const float ux = wv.x * t[c].x, uy = wv.y * t[c].y, uz = wv.z * t[c].z, uw = wv.w * t[c].w;
#pragma unroll
      for (int d = c; d < NC; ++d, ++p) {
        acc[p] += (double)(ux * t[d].x);
        acc[p] += (double)(uy * t[d].y);
        acc[p] += (double)(uz * t[d].z);
        acc[p] += (double)(uw * t[d].w);
      }
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int p = 0; p < NP; ++p) {
    double v = acc[p];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[warp][p] = v;
  }
  __syncthreads();
  if (threadIdx.x < NP) {
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < GRAM_THREADS / 32; ++k) s += red[k][threadIdx.x];
    partial[((long long)b * gridDim.x + slab) * NP + threadIdx.x] = s;
  }
}

__global__ void laplace_fold_kernel(const double* __restrict__ partial, int B, int ncls, int nslab,
                                    double* __restrict__ cov) {
  pdl_launch_dependents();
  pdl_wait();
  const int np = ncls * (ncls + 1) / 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * np) return;
  const int b = i / np, p = i - b * np;
  int c = 0, q = p;
  while (q >= ncls - c) { q -= ncls - c; ++c; }
  const int d = c + q;
  const double* src = partial + (long long)b * nslab * np + p;
  double s = 0.0;
  for (int k = 0; k < nslab; ++k) s += src[(long long)k * np];
  cov[((long long)b * ncls + c) * ncls + d] = s;
  cov[((long long)b * ncls + d) * ncls + c] = s;
}

// L [B, C, C] (row-major, upper triangle 0): for k in order, the pivot d = S_kk - sum_{j<k} L_kj^2; d <= tol (tol =
// RD_LAPLACE_PIVOT_TOL * trace(S)) zeroes column k, else L_kk = sqrt(d), L_ik = (S_ik - sum_{j<k} L_ij L_kj) / L_kk.
__global__ void laplace_chol_kernel(const double* __restrict__ cov, int B, int C, double* __restrict__ Lo) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const double* S = cov + (long long)b * C * C;
  double* L = Lo + (long long)b * C * C;
  double tr = 0.0;
  for (int k = 0; k < C; ++k) tr += S[k * C + k];
  const double tol = RD_LAPLACE_PIVOT_TOL * tr;
  for (int i = 0; i < C * C; ++i) L[i] = 0.0;
  for (int k = 0; k < C; ++k) {
    double dk = S[k * C + k];
    for (int j = 0; j < k; ++j) dk -= L[k * C + j] * L[k * C + j];
    if (!(dk > tol)) continue;                 // the column stays 0
    const double lkk = sqrt(dk);
    L[k * C + k] = lkk;
    for (int i = k + 1; i < C; ++i) {
      double v = S[i * C + k];
      for (int j = 0; j < k; ++j) v -= L[i * C + j] * L[k * C + j];
      L[i * C + k] = v / lkk;
    }
  }
}

// standard normal of element e = b*C + k of replicate m (key {seed, step + m}): Box-Muller on the pair (x, y) of the
// block at counter e >> 2 for e & 3 in {0, 1}, (z, w) for {2, 3}, as rd_dp_add_noise draws them
__device__ __forceinline__ double laplace_normal(const RngKey& k, uint64_t e) {
  return (double)philox_normal(k, SITE_LAPLACE, e);
}

// logits [nc*B, C] replicate-major (row j = m*B + b, replicate m0 + m): f_c = mu_c + sum_{k <= c} L_ck eps_k in fp64,
// rounded to fp32 once
__global__ void laplace_draw_kernel(const float* __restrict__ mu, const double* __restrict__ Lo, int B, int C,
                                    const uint64_t* __restrict__ rng, long long m0, int nc, float* __restrict__ logits) {
  pdl_launch_dependents();
  pdl_wait();
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nc * B) return;
  const int m = j / B, b = j - m * B;
  const uint64_t seed = rng[0], step = rng[1] + (uint64_t)(m0 + m);
  const RngKey key{(uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(step >> 32), (uint32_t)step};
  double eps[RD_LAPLACE_MAX_CLASSES];
  for (int k = 0; k < C; ++k) eps[k] = laplace_normal(key, (uint64_t)b * C + k);
  const double* L = Lo + (long long)b * C * C;
  for (int c = 0; c < C; ++c) {
    double f = (double)mu[(long long)b * C + c];
    for (int k = 0; k <= c; ++k) f += L[c * C + k] * eps[k];
    logits[(long long)j * C + c] = (float)f;
  }
}

int64_t gram_slabs(int64_t ldg) { return (ldg + GRAM_SLAB - 1) / GRAM_SLAB; }

struct SampleLayout { int64_t L, acc, logits, total; };     // in doubles
SampleLayout sample_layout(int B, int C, int spc) {
  SampleLayout l;
  l.L = 0;
  l.acc = round_up((int64_t)B * C * C, 8);
  l.logits = l.acc + round_up((int64_t)B * (2 * C + 1), 8);
  l.total = l.logits + round_up(((int64_t)spc * B * C + 1) / 2, 8);
  return l;
}

}  // namespace

int64_t laplace_gram_partial_doubles(int B, int ncls, int64_t ldg) {
  return (int64_t)B * gram_slabs(ldg) * (ncls * (ncls + 1) / 2);
}

int laplace_seed(float* d_logits, int B, int ncls, int c, cudaStream_t st) {
  launch_pdl(laplace_seed_kernel, dim3((unsigned)ceil_div((int64_t)B * ncls, 256)), dim3(256), 0, st, d_logits, B, ncls, c);
  RD_CHECK_LAUNCH("laplace_seed_kernel");
  return 0;
}

int laplace_gram(const float* G, int B, int ncls, int64_t ldg, const float* w, double* partial, double* cov,
                 cudaStream_t st) {
  const int64_t nslab = gram_slabs(ldg);
  const dim3 grid((unsigned)nslab, (unsigned)B);
  switch (ncls) {
#define RD_GRAM_CASE(NC) \
    case NC: launch_pdl(laplace_gram_kernel<NC>, grid, dim3(GRAM_THREADS), 0, st, G, B, (long long)ldg, w, partial); break;
    RD_GRAM_CASE(1) RD_GRAM_CASE(2) RD_GRAM_CASE(3) RD_GRAM_CASE(4)
    RD_GRAM_CASE(5) RD_GRAM_CASE(6) RD_GRAM_CASE(7) RD_GRAM_CASE(8)
#undef RD_GRAM_CASE
    default: set_error("laplace_gram: n_classes = %d, at most %d", ncls, RD_LAPLACE_MAX_CLASSES); return -2;
  }
  RD_CHECK_LAUNCH("laplace_gram_kernel");
  const int64_t n = (int64_t)B * (ncls * (ncls + 1) / 2);
  launch_pdl(laplace_fold_kernel, dim3((unsigned)ceil_div(n, 128)), dim3(128), 0, st, (const double*)partial, B, ncls,
             (int)nslab, cov);
  RD_CHECK_LAUNCH("laplace_fold_kernel");
  return 0;
}

}  // namespace rd

using namespace rd;

extern "C" {

size_t rd_laplace_sample_scratch_bytes(int32_t B, int32_t n_classes, int32_t samples_per_chunk) {
  if (B < 1 || n_classes < 1 || n_classes > RD_LAPLACE_MAX_CLASSES || samples_per_chunk < 1) return 0;
  if ((int64_t)B * samples_per_chunk > INT32_MAX) return 0;
  return (size_t)sample_layout(B, n_classes, samples_per_chunk).total * sizeof(double);
}

// One Cholesky launch, then per chunk of spc replicates one draw launch and mc_accumulate (the reduction of
// rd_raindrop_v2_mc_dropout).
int rd_laplace_predictive_mc(const float* mean_logits, const double* cov, int32_t B, int32_t n_classes, const uint64_t* rng,
                             int32_t n_samples, int32_t samples_per_chunk, void* scratch, float* mean_probs,
                             float* variance, float* entropies, float* samples, void* stream) {
  const char* fn = "rd_laplace_predictive_mc";
  if (!mean_logits || !cov || !rng || !scratch || !mean_probs || !variance || !entropies) {
    set_error("%s: NULL argument", fn);
    return -2;
  }
  if (B < 1 || n_classes < 1 || n_classes > RD_LAPLACE_MAX_CLASSES || n_samples < 1 || samples_per_chunk < 1 ||
      (int64_t)B * samples_per_chunk > INT32_MAX) {
    set_error("%s: bad sizes (B=%d n_classes=%d (at most %d) n_samples=%d samples_per_chunk=%d)", fn, B, n_classes,
              RD_LAPLACE_MAX_CLASSES, n_samples, samples_per_chunk);
    return -2;
  }
  if (reinterpret_cast<uintptr_t>(scratch) & 15) { set_error("%s: scratch must be 16-byte aligned", fn); return -2; }
  cudaStream_t st = (cudaStream_t)stream;
  const int C = n_classes, spc = samples_per_chunk;
  const SampleLayout l = sample_layout(B, C, spc);
  double* S = (double*)scratch;
  double* Lo = S + l.L;
  double* acc = S + l.acc;
  float* logits = reinterpret_cast<float*>(S + l.logits);
  launch_pdl(laplace_chol_kernel, dim3((unsigned)ceil_div(B, 128)), dim3(128), 0, st, cov, (int)B, C, Lo);
  RD_CHECK_LAUNCH("laplace_chol_kernel");
  const int64_t M = n_samples;
  for (int64_t m0 = 0; m0 < M; m0 += spc) {
    const int nc = (int)(M - m0 < spc ? M - m0 : spc);
    launch_pdl(laplace_draw_kernel, dim3((unsigned)ceil_div((int64_t)nc * B, 128)), dim3(128), 0, st, mean_logits,
               (const double*)Lo, (int)B, C, rng, (long long)m0, nc, logits);
    RD_CHECK_LAUNCH("laplace_draw_kernel");
    RD_TRY(mc_accumulate(logits, nc, B, C, m0, M, acc, samples, mean_probs, variance, entropies, m0 == 0, m0 + nc >= M, st));
  }
  return 0;
}

}  // extern "C"
