// SWA / SWAG of Raindrop_v2 (Izmailov et al. 2018; Maddox et al. 2019): the two memory-bound kernels over the flat
// parameter bucket that rd_swag_collect / rd_swag_sample launch and rd_raindrop_v2_swag_predictive runs per replicate.
//   swag_collect_kernel  one thread per 4 elements: the fp64 running moments updated with theta and the deviation column
//                        of slot c % K written; 128-bit loads of theta, mean and sq_mean.
//   swag_sample_kernel   one thread per 4 elements: theta_s = mean + sqrt(scale) (sd z1 + D z2 / sqrt(k - 1)), the k
//                        normals z2 drawn once per CTA into shared memory, the slot rows streamed with 128-bit loads.
// Every fp64 operation is an explicitly rounded intrinsic, so nvcc contracts nothing into an FMA and a float64 numpy
// restatement (raindrop_b200/swag.py) reproduces the moments bit for bit.
#include <math.h>

#include "rd_kernels.cuh"

namespace rd {
namespace {

constexpr int SWAG_THREADS = 256;

__global__ void __launch_bounds__(SWAG_THREADS) swag_collect_kernel(const float4* __restrict__ theta, long long n4,
                                                                     double c, int slot, double2* __restrict__ mean,
                                                                     double2* __restrict__ sq, float4* __restrict__ dev) {
  pdl_launch_dependents();
  pdl_wait();
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n4) return;
  const double c1 = __dadd_rn(c, 1.0);
  const float4 t = __ldg(theta + q);
  const double th[4] = {(double)t.x, (double)t.y, (double)t.z, (double)t.w};
  const double2 m0 = mean[2 * q], m1 = mean[2 * q + 1], s0 = sq[2 * q], s1 = sq[2 * q + 1];
  const double mo[4] = {m0.x, m0.y, m1.x, m1.y}, so[4] = {s0.x, s0.y, s1.x, s1.y};
  double mn[4], sn[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    mn[e] = __ddiv_rn(__dadd_rn(__dmul_rn(c, mo[e]), th[e]), c1);
    sn[e] = __ddiv_rn(__dadd_rn(__dmul_rn(c, so[e]), __dmul_rn(th[e], th[e])), c1);
  }
  mean[2 * q] = make_double2(mn[0], mn[1]);
  mean[2 * q + 1] = make_double2(mn[2], mn[3]);
  sq[2 * q] = make_double2(sn[0], sn[1]);
  sq[2 * q + 1] = make_double2(sn[2], sn[3]);
  if (dev)
    dev[(long long)slot * n4 + q] = make_float4((float)__dsub_rn(th[0], mn[0]), (float)__dsub_rn(th[1], mn[1]),
                                                (float)__dsub_rn(th[2], mn[2]), (float)__dsub_rn(th[3], mn[3]));
}

__global__ void __launch_bounds__(SWAG_THREADS) swag_sample_kernel(const double2* __restrict__ mean,
                                                                    const double2* __restrict__ sq,
                                                                    const float4* __restrict__ dev, long long n4, int k,
                                                                    double root_scale, const uint64_t* __restrict__ rng,
                                                                    long long replicate, float4* __restrict__ out) {
  extern __shared__ double z2[];
  pdl_launch_dependents();
  pdl_wait();
  const uint64_t seed = rng[0], step = rng[1] + (uint64_t)replicate;
  const RngKey key{(uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(step >> 32), (uint32_t)step};
  const uint64_t n = 4ull * (uint64_t)n4;
  const int lowrank = k >= 2;
  if (lowrank)
    for (int j = threadIdx.x; j < k; j += blockDim.x) z2[j] = (double)philox_normal(key, SITE_SWAG, n + (uint64_t)j);
  __syncthreads();
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n4) return;
  const uint4 w = dropout_block(key, SITE_SWAG, 4ull * (uint64_t)q);
  float z1[4];
  box_muller(w.x, w.y, &z1[0], &z1[1]);
  box_muller(w.z, w.w, &z1[2], &z1[3]);
  const double2 m0 = mean[2 * q], m1 = mean[2 * q + 1], s0 = sq[2 * q], s1 = sq[2 * q + 1];
  const double mu[4] = {m0.x, m0.y, m1.x, m1.y}, sm[4] = {s0.x, s0.y, s1.x, s1.y};
  double a[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const double var = __dsub_rn(sm[e], __dmul_rn(mu[e], mu[e]));
    a[e] = __dmul_rn(__dsqrt_rn(var > 0.0 ? var : 0.0), (double)z1[e]);
  }
  if (lowrank) {
    double s[4] = {0.0, 0.0, 0.0, 0.0};
    for (int j = 0; j < k; ++j) {
      const float4 d = __ldcs(dev + (long long)j * n4 + q);
      const double zj = z2[j];
      s[0] = __dadd_rn(s[0], __dmul_rn((double)d.x, zj));
      s[1] = __dadd_rn(s[1], __dmul_rn((double)d.y, zj));
      s[2] = __dadd_rn(s[2], __dmul_rn((double)d.z, zj));
      s[3] = __dadd_rn(s[3], __dmul_rn((double)d.w, zj));
    }
    const double root_k1 = __dsqrt_rn((double)(k - 1));
#pragma unroll
    for (int e = 0; e < 4; ++e) a[e] = __dadd_rn(a[e], __ddiv_rn(s[e], root_k1));
  }
  float r[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) r[e] = (float)__dadd_rn(mu[e], __dmul_rn(root_scale, a[e]));
  out[q] = make_float4(r[0], r[1], r[2], r[3]);
}

}  // namespace

int swag_collect(const float* theta, int64_t n, int64_t c, int rank, double* mean, double* sq, float* dev,
                 cudaStream_t st) {
  const long long n4 = n / 4;
  const int slot = rank > 0 ? (int)(c % rank) : 0;
  launch_pdl(swag_collect_kernel, dim3((unsigned)ceil_div(n4, SWAG_THREADS)), dim3(SWAG_THREADS), 0, st,
             reinterpret_cast<const float4*>(theta), n4, (double)c, slot, reinterpret_cast<double2*>(mean),
             reinterpret_cast<double2*>(sq), rank > 0 ? reinterpret_cast<float4*>(dev) : nullptr);
  RD_CHECK_LAUNCH("swag_collect_kernel");
  return 0;
}

int swag_sample(const double* mean, const double* sq, const float* dev, int64_t n, int k, double scale,
                const uint64_t* rng, int64_t replicate, float* out, cudaStream_t st) {
  const long long n4 = n / 4;
  const size_t smem = k >= 2 ? (size_t)k * sizeof(double) : 0;
  launch_pdl(swag_sample_kernel, dim3((unsigned)ceil_div(n4, SWAG_THREADS)), dim3(SWAG_THREADS), smem, st,
             reinterpret_cast<const double2*>(mean), reinterpret_cast<const double2*>(sq),
             reinterpret_cast<const float4*>(dev), n4, k, sqrt(scale), rng, (long long)replicate,
             reinterpret_cast<float4*>(out));
  RD_CHECK_LAUNCH("swag_sample_kernel");
  return 0;
}

// The checks rd_swag_sample and every member of rd_raindrop_v2_swag_predictive share.
int swag_sample_check(const char* fn, const double* mean, const double* sq, const float* dev, int64_t n, int k,
                      double scale) {
  if (!mean || !sq || (k >= 2 && !dev)) { set_error("%s: NULL argument", fn); return -2; }
  if (n < 4 || n % 4 || n / 4 > 0x7fffffffLL * SWAG_THREADS) { set_error("%s: n = %lld must be a positive multiple of 4", fn, (long long)n); return -2; }
  if (k < 0 || k > RD_SWAG_MAX_RANK) { set_error("%s: k = %d must be in [0, %d]", fn, k, RD_SWAG_MAX_RANK); return -2; }
  if (!(scale >= 0.0) || isinf(scale)) { set_error("%s: scale must be finite and >= 0, got %g", fn, scale); return -2; }
  if ((reinterpret_cast<uintptr_t>(mean) | reinterpret_cast<uintptr_t>(sq) | reinterpret_cast<uintptr_t>(dev)) & 15) {
    set_error("%s: mean, sq_mean and dev must be 16-byte aligned", fn);
    return -2;
  }
  return 0;
}

}  // namespace rd

using namespace rd;

extern "C" {

int rd_swag_collect(const float* theta, int64_t n, int64_t n_collected, int32_t rank, double* mean, double* sq_mean,
                    float* dev, void* stream) {
  const char* fn = "rd_swag_collect";
  if (!theta || !mean || !sq_mean || (rank > 0 && !dev)) { set_error("%s: NULL argument", fn); return -2; }
  if (n < 4 || n % 4) { set_error("%s: n = %lld must be a positive multiple of 4", fn, (long long)n); return -2; }
  if (rank < 0 || rank > RD_SWAG_MAX_RANK || n_collected < 0 || n_collected >= (1LL << 53)) {
    set_error("%s: rank = %d must be in [0, %d] and n_collected = %lld in [0, 2^53)", fn, rank, RD_SWAG_MAX_RANK,
              (long long)n_collected);
    return -2;
  }
  if ((reinterpret_cast<uintptr_t>(theta) | reinterpret_cast<uintptr_t>(mean) | reinterpret_cast<uintptr_t>(sq_mean) |
       reinterpret_cast<uintptr_t>(dev)) & 15) {
    set_error("%s: theta, mean, sq_mean and dev must be 16-byte aligned", fn);
    return -2;
  }
  return swag_collect(theta, n, n_collected, rank, mean, sq_mean, dev, (cudaStream_t)stream);
}

int rd_swag_sample(const double* mean, const double* sq_mean, const float* dev, int64_t n, int32_t k, double scale,
                   const uint64_t* rng, int64_t replicate, float* theta_out, void* stream) {
  const char* fn = "rd_swag_sample";
  RD_TRY(swag_sample_check(fn, mean, sq_mean, dev, n, k, scale));
  if (!rng || !theta_out) { set_error("%s: NULL argument", fn); return -2; }
  if (reinterpret_cast<uintptr_t>(theta_out) & 15) { set_error("%s: theta_out must be 16-byte aligned", fn); return -2; }
  if (replicate < 0) { set_error("%s: replicate must be >= 0", fn); return -2; }
  return swag_sample(mean, sq_mean, dev, n, k, scale, rng, replicate, theta_out, (cudaStream_t)stream);
}

}  // extern "C"
