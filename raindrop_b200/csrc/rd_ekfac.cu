// EK-FAC influence functions (George et al. 2018; Grosse et al. 2023): the small kernels around the factor pass and the
// rotated rows of rd_model.cu.
//   kfac_accumulate_kernel   one block's fp32 factor sums (X^T X with its column sums, dY^T dY) added into the caller's
//                            fp64 factors: A = [[X^T X, x], [x^T, rows]] over [X | 1], S scaled by B^2.  One thread per
//                            element, no atomics.
//   ekfac_sq_kernel          lam[j] += sum_r G[r, j]^2 in fp64, rows in order, one thread per column.
//   ekfac_scale_kernel       G[r, j] *= w[j].
//   fisher_label_kernel      one label per sample drawn from softmax(logits) by inverse CDF in fp64, the uniform from
//                            Philox4x32-10 keyed by (seed, global sample index) (the mapping is in the header).
#include "rd_kernels.cuh"

namespace rd {
namespace {

constexpr uint32_t SITE_FISHER_LABEL = 97;     // Philox site of the sampled Fisher labels (the dropout sites are 1-96)

__global__ void kfac_accumulate_kernel(const float* __restrict__ Aw, const float* __restrict__ Ab,
                                       const float* __restrict__ Sw, int Kin, int Nout, double rows, double sscale,
                                       double* __restrict__ A, double* __restrict__ S) {
  pdl_launch_dependents();
  pdl_wait();
  const long long na = (long long)(Kin + 1) * (Kin + 1), ns = (long long)Nout * Nout;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < na) {
    const int i = (int)(idx / (Kin + 1)), j = (int)(idx % (Kin + 1));
    double v;
    if (i < Kin && j < Kin) v = (double)Aw[(long long)i * Kin + j];
    else if (i < Kin) v = (double)Ab[i];
    else if (j < Kin) v = (double)Ab[j];
    else v = rows;
    A[idx] += v;
  } else if (idx < na + ns) {
    S[idx - na] += sscale * (double)Sw[idx - na];
  }
}

__global__ void ekfac_sq_kernel(const float* __restrict__ G, int rows, long long ldg, long long c0, long long n,
                                double* __restrict__ lam) {
  pdl_launch_dependents();
  pdl_wait();
  const long long j = c0 + (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= c0 + n) return;
  double s = 0.0;
  for (int r = 0; r < rows; ++r) {
    const double g = (double)G[(long long)r * ldg + j];
    s += g * g;
  }
  lam[j] += s;
}

__global__ void ekfac_scale_kernel(float* __restrict__ G, int rows, long long ldg, long long c0, long long n,
                                   const float* __restrict__ w) {
  pdl_launch_dependents();
  pdl_wait();
  const long long j = c0 + (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= c0 + n) return;
  const float wj = w[j];
  for (int r = blockIdx.y; r < rows; r += gridDim.y) G[(long long)r * ldg + j] *= wj;
}

// the uniform of global sample index i: 53 bits of the first two words of Philox block (i, site), in [0, 1)
__device__ __forceinline__ double fisher_uniform(uint64_t seed, uint64_t i) {
  const uint4 w = philox4((uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)i, (uint32_t)(i >> 32), SITE_FISHER_LABEL, 0u);
  return ((double)(w.x >> 5) * 67108864.0 + (double)(w.y >> 6)) * (1.0 / 9007199254740992.0);
}

__global__ void fisher_label_kernel(const float* __restrict__ logits, int B, int ncls, uint64_t seed, uint64_t index0,
                                    int64_t* __restrict__ y) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float* l = logits + (long long)b * ncls;
  double m = (double)l[0];
  for (int c = 1; c < ncls; ++c) m = fmax(m, (double)l[c]);
  double total = 0.0;
  for (int c = 0; c < ncls; ++c) total += exp((double)l[c] - m);
  const double target = fisher_uniform(seed, index0 + (uint64_t)b) * total;
  double cum = 0.0;
  int64_t label = ncls - 1;
  for (int c = 0; c < ncls; ++c) {
    cum += exp((double)l[c] - m);
    if (target < cum) { label = c; break; }
  }
  y[b] = label;
}

__global__ void fisher_uniform_kernel(uint64_t seed, uint64_t index0, int n, double* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = fisher_uniform(seed, index0 + (uint64_t)i);
}

// Maximal column runs of the segments: a segment joins the previous run when it starts at that run's end rounded up to
// 4 columns (only bucket padding, whose columns are 0 in every row, lies between them).  f(c0, n) per run.
template <typename F>
int for_runs(const int64_t* seg_off, const int64_t* seg_len, int n_seg, int64_t ldg, const char* fn, F f) {
  long long r0 = -1, r1 = -1;
  for (int i = 0; i < n_seg; ++i) {
    if (seg_off[i] < 0 || seg_len[i] < 1 || seg_off[i] + seg_len[i] > ldg) {
      set_error("%s: segment %d [%lld, +%lld) is not inside the row", fn, i, (long long)seg_off[i], (long long)seg_len[i]);
      return -2;
    }
    if (r0 >= 0 && seg_off[i] == round_up(r1, 4)) { r1 = seg_off[i] + seg_len[i]; continue; }
    if (r0 >= 0) RD_TRY(f(r0, r1 - r0));
    r0 = seg_off[i]; r1 = seg_off[i] + seg_len[i];
  }
  if (r0 >= 0) RD_TRY(f(r0, r1 - r0));
  return 0;
}

}  // namespace

int kfac_accumulate(const float* Aw, const float* Ab, const float* Sw, int Kin, int Nout, long long rows, double sscale,
                    double* A, double* S, cudaStream_t st) {
  const long long n = (long long)(Kin + 1) * (Kin + 1) + (long long)Nout * Nout;
  launch_pdl(kfac_accumulate_kernel, dim3((unsigned)ceil_div(n, 256)), dim3(256), 0, st, Aw, Ab, Sw, Kin, Nout,
             (double)rows, sscale, A, S);
  RD_CHECK_LAUNCH("kfac_accumulate_kernel");
  return 0;
}

}  // namespace rd

using namespace rd;

extern "C" {

int rd_ekfac_accumulate_sq(const float* G, int32_t rows, int64_t ldg, const int64_t* seg_off, const int64_t* seg_len,
                           int32_t n_seg, double* lam, void* stream) {
  const char* fn = "rd_ekfac_accumulate_sq";
  if (!G || !seg_off || !seg_len || !lam) { set_error("%s: NULL argument", fn); return -2; }
  if (rows < 0 || ldg < 1 || n_seg < 0) { set_error("%s: bad sizes (rows=%d ldg=%lld n_seg=%d)", fn, rows, (long long)ldg, n_seg); return -2; }
  if (rows == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  return for_runs(seg_off, seg_len, n_seg, ldg, fn, [&](long long c0, long long n) {
    launch_pdl(ekfac_sq_kernel, dim3((unsigned)ceil_div(n, 128)), dim3(128), 0, st, G, (int)rows, (long long)ldg, c0, n, lam);
    RD_CHECK_LAUNCH("ekfac_sq_kernel");
    return 0;
  });
}

int rd_ekfac_scale_rows(float* G, int32_t rows, int64_t ldg, const int64_t* seg_off, const int64_t* seg_len,
                        int32_t n_seg, const float* w, void* stream) {
  const char* fn = "rd_ekfac_scale_rows";
  if (!G || !seg_off || !seg_len || !w) { set_error("%s: NULL argument", fn); return -2; }
  if (rows < 0 || ldg < 1 || n_seg < 0) { set_error("%s: bad sizes (rows=%d ldg=%lld n_seg=%d)", fn, rows, (long long)ldg, n_seg); return -2; }
  if (rows == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned gy = (unsigned)(rows < 64 ? rows : 64);
  return for_runs(seg_off, seg_len, n_seg, ldg, fn, [&](long long c0, long long n) {
    launch_pdl(ekfac_scale_kernel, dim3((unsigned)ceil_div(n, 128), gy), dim3(128), 0, st, G, (int)rows, (long long)ldg, c0,
               n, w);
    RD_CHECK_LAUNCH("ekfac_scale_kernel");
    return 0;
  });
}

int rd_fisher_labels(const float* logits, int32_t B, int32_t n_classes, uint64_t seed, uint64_t index0, int64_t* y,
                     void* stream) {
  if (!logits || !y || B < 0 || n_classes < 1) { set_error("rd_fisher_labels: bad arguments"); return -2; }
  if (B == 0) return 0;
  launch_pdl(fisher_label_kernel, dim3((unsigned)ceil_div(B, 128)), dim3(128), 0, (cudaStream_t)stream, logits, (int)B,
             (int)n_classes, seed, index0, y);
  RD_CHECK_LAUNCH("fisher_label_kernel");
  return 0;
}

int rd_debug_fisher_uniforms(uint64_t seed, uint64_t index0, int32_t n, double* out, void* stream) {
  if (!out || n < 0) { set_error("rd_debug_fisher_uniforms: bad arguments"); return -2; }
  if (n == 0) return 0;
  fisher_uniform_kernel<<<(unsigned)ceil_div(n, 128), 128, 0, (cudaStream_t)stream>>>(seed, index0, (int)n, out);
  RD_CHECK_LAUNCH("fisher_uniform_kernel");
  return 0;
}

}  // extern "C"
