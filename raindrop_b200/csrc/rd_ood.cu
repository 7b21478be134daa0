// Out-of-distribution scores of Raindrop_v2 (rd_feature_moments, rd_ood_prepare_bank, rd_raindrop_v2_ood_scores): the
// feature moments of a training set, row normalisation and centring, the logit scores, the per-class Mahalanobis
// distances and the running top-k of the nearest-neighbour search.  rd_model.cu runs the forward and the tensor-core
// GEMMs (tc_nt) between these launches.
//
// Determinism: every reduction here has one fixed order per output element.  The moments add the samples one by one in
// index order into the value already stored (accumulate), so the float64 sums are bitwise the same whatever the launch
// shape and however the set is split across calls; products of two fp32 values are exact in fp64, so each step rounds
// once.  Row norms and class distances reduce a row inside one warp in a fixed shuffle tree.  The kNN selection keeps
// the ks largest 64-bit keys (similarity, then bank index) of every candidate, and keys are distinct, so the result is
// one set whatever order the candidates arrive in; the final ranking of those ks is by fp64 values and index alone.
#include <math.h>

#include "rd_kernels.cuh"

namespace rd {
namespace {

constexpr int MOM_TILE = 16, MOM_SLAB = 64, MOM_CLASS_TPB = 128;
constexpr int ROW_WARPS = 8;                 // rows (one warp each) per CTA of the row kernels
constexpr int TOPK_TPB = 256, TOPK_CAP = 2048;
constexpr int TOPK_MAX_SEL = RD_OOD_MAX_K + RD_OOD_SEL_EXTRA;   // the longest running list

// gram[i, j] (+)= sum_s f[s, i] f[s, j]: one thread per entry of a 16 x 16 tile, samples staged in slabs of 64.
__global__ void __launch_bounds__(MOM_TILE * MOM_TILE) ood_gram_kernel(const float* __restrict__ f, long long n, int F,
                                                                      int accumulate, double* __restrict__ gram) {
  __shared__ float a[MOM_SLAB][MOM_TILE], b[MOM_SLAB][MOM_TILE];
  pdl_launch_dependents();
  pdl_wait();
  const int i0 = blockIdx.y * MOM_TILE, j0 = blockIdx.x * MOM_TILE;
  const int tx = threadIdx.x % MOM_TILE, ty = threadIdx.x / MOM_TILE;
  const int i = i0 + ty, j = j0 + tx;
  const bool in = i < F && j < F;
  double acc = accumulate && in ? gram[(long long)i * F + j] : 0.0;
  for (long long s0 = 0; s0 < n; s0 += MOM_SLAB) {
    for (int e = threadIdx.x; e < MOM_SLAB * MOM_TILE; e += MOM_TILE * MOM_TILE) {
      const int r = e / MOM_TILE, c = e % MOM_TILE;
      const long long s = s0 + r;
      a[r][c] = s < n && i0 + c < F ? __ldg(f + s * F + i0 + c) : 0.f;
      b[r][c] = s < n && j0 + c < F ? __ldg(f + s * F + j0 + c) : 0.f;
    }
    __syncthreads();
    const int m = n - s0 < MOM_SLAB ? (int)(n - s0) : MOM_SLAB;
    for (int r = 0; r < m; ++r) acc = fma((double)a[r][ty], (double)b[r][tx], acc);
    __syncthreads();
  }
  if (in) gram[(long long)i * F + j] = acc;
}

// sums[c, j] (+)= sum_{s: y[s] = c} f[s, j] (one thread per (c, j)) and counts[c] (+)= #{s: y[s] = c} (thread 0 of the
// first CTA of row c).  Labels outside [0, C) count nowhere.
__global__ void __launch_bounds__(MOM_CLASS_TPB) ood_class_sums_kernel(const float* __restrict__ f,
                                                                       const int64_t* __restrict__ y, long long n, int F,
                                                                       int accumulate, double* __restrict__ sums,
                                                                       long long* __restrict__ counts) {
  __shared__ long long ys[MOM_SLAB];
  pdl_launch_dependents();
  pdl_wait();
  const int c = blockIdx.y, j = blockIdx.x * MOM_CLASS_TPB + threadIdx.x;
  const bool counter = blockIdx.x == 0 && threadIdx.x == 0;
  double acc = accumulate && j < F ? sums[(long long)c * F + j] : 0.0;
  long long cnt = accumulate && counter ? counts[c] : 0;
  for (long long s0 = 0; s0 < n; s0 += MOM_SLAB) {
    const int m = n - s0 < MOM_SLAB ? (int)(n - s0) : MOM_SLAB;
    for (int r = threadIdx.x; r < m; r += MOM_CLASS_TPB) ys[r] = __ldg(reinterpret_cast<const long long*>(y) + s0 + r);
    __syncthreads();
    for (int r = 0; r < m; ++r) {
      if (ys[r] != c) continue;
      if (j < F) acc += (double)__ldg(f + (s0 + r) * F + j);
      cnt += 1;
    }
    __syncthreads();
  }
  if (j < F) sums[(long long)c * F + j] = acc;
  if (counter) counts[c] = cnt;
}

// Sum of v over a warp, in a fixed tree.
__device__ __forceinline__ double warp_sum(double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// out[r, :] = f[r, :F] / max(||f[r, :F]||_2, 1e-12) (norm in fp64, rounded to fp32, as F.normalize divides), zero in
// columns F .. ld-1; or, with mu, out[r, j] = fp32(f[r, j] - mu[j]) for j < F.  One warp per row.
__global__ void __launch_bounds__(32 * ROW_WARPS) ood_rows_kernel(const float* __restrict__ f, long long ldf, long long n,
                                                                  int F, const double* __restrict__ mu, int ld,
                                                                  float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const long long r = (long long)blockIdx.x * ROW_WARPS + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  if (r >= n) return;
  const float* x = f + r * ldf;
  float* o = out + r * ld;
  if (mu) {
    for (int j = lane; j < ld; j += 32) o[j] = j < F ? (float)((double)__ldg(x + j) - mu[j]) : 0.f;
    return;
  }
  double ss = 0.0;
  for (int j = lane; j < F; j += 32) { const double v = __ldg(x + j); ss = fma(v, v, ss); }
  const float nrm = fmaxf((float)sqrt(warp_sum(ss)), 1e-12f);
  for (int j = lane; j < ld; j += 32) o[j] = j < F ? __ldg(x + j) / nrm : 0.f;
}

// msp = -max_c softmax(l)_c and energy = -T logsumexp(l / T), in fp64 from the fp32 logits; one thread per row.
__global__ void ood_logit_kernel(const float* __restrict__ logits, int n, int C, float temperature, float* __restrict__ msp,
                                 float* __restrict__ energy) {
  pdl_launch_dependents();
  pdl_wait();
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const float* l = logits + (long long)r * C;
  const double T = temperature;
  double m = -INFINITY;
  for (int c = 0; c < C; ++c) m = fmax(m, (double)l[c]);
  double se = 0.0, st = 0.0;
  for (int c = 0; c < C; ++c) { se += exp((double)l[c] - m); st += exp(((double)l[c] - m) / T); }
  if (msp) msp[r] = (float)(-1.0 / se);
  if (energy) energy[r] = (float)(-(m + T * log(st)));
}

// d[r, c] = sum_j (Z[r, j] - M[c, j])^2 in fp64 over j < rp; the minimum over the classes whose d is a number and its
// first argmin (NaN and class 0 when there is none).  One warp per row.
__global__ void __launch_bounds__(32 * ROW_WARPS) ood_class_dist_kernel(const float* __restrict__ Z,
                                                                        const float* __restrict__ M, int n, int C, int rp,
                                                                        float* __restrict__ dist, float* __restrict__ dmin,
                                                                        long long* __restrict__ cls) {
  pdl_launch_dependents();
  pdl_wait();
  const long long r = (long long)blockIdx.x * ROW_WARPS + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  if (r >= n) return;
  const float* z = Z + r * rp;
  double best = INFINITY;
  int arg = 0;
  bool nan_row = true;           // NaN when no class gives a number (non-finite features)
  for (int c = 0; c < C; ++c) {
    double acc = 0.0;
    for (int j = lane; j < rp; j += 32) { const double d = (double)z[j] - (double)__ldg(M + (long long)c * rp + j); acc = fma(d, d, acc); }
    acc = warp_sum(acc);
    if (dist && lane == 0) dist[r * C + c] = (float)acc;
    if (!isnan(acc)) nan_row = false;
    if (acc < best) { best = acc; arg = c; }
  }
  if (lane == 0) {
    if (dmin) dmin[r] = nan_row ? __int_as_float(0x7fc00000) : (float)best;
    if (cls) cls[r] = arg;
  }
}

// The top-k order as one unsigned key: similarity (larger first; -0 counts as +0, NaN below every number), then bank
// index (lower first).  Key 0 is an empty slot: no candidate has it (indices are < 2^31).
__device__ __forceinline__ unsigned long long topk_key(float s, long long idx) {
  uint32_t u = __float_as_uint(s + 0.f);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  if (isnan(s)) u = 0;
  return ((unsigned long long)u << 32) | (uint32_t)~(uint32_t)idx;
}

// Bitonic sort of buf[0, P) in descending order, P a power of two.
__device__ void topk_sort(unsigned long long* buf, int P) {
  for (int size = 2; size <= P; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = threadIdx.x; t < P / 2; t += TOPK_TPB) {
        const int i = 2 * stride * (t / stride) + t % stride, j = i + stride;
        const unsigned long long a = buf[i], b = buf[j];
        if ((i & size) == 0 ? a < b : a > b) { buf[i] = b; buf[j] = a; }
      }
      __syncthreads();
    }
  }
}

// One CTA per query row: merges the row's similarities to bank rows col0 .. col0 + ncols - 1 (sim[row * ld + c]) into
// its running list run[row, :ks] of the ks largest keys (sorted; `first`: the list starts empty).  Candidates above the
// current ks-th key are appended to shared memory; when the buffer could overflow, and at the end, the list and the
// candidates are sorted together and cut to ks.  `last`: instead of the running list, the ks candidates' similarities
// are recomputed as fp64 dots of the fp32 rows (one warp per candidate, a fixed shuffle tree; NaN ranks below every
// number) and the k largest of those are written: idx[row, :k] in (similarity descending, index ascending) order and
// knn[row] = 2 - 2 s_(k).  ks > k keeps the rows the 3xTF32 similarities could have ranked just below the k-th.
__global__ void __launch_bounds__(TOPK_TPB) ood_topk_kernel(const float* __restrict__ sim, long long ld, int ncols,
                                                            long long col0, int k, int ks, int first, int last,
                                                            unsigned long long* __restrict__ run,
                                                            const float* __restrict__ q, const float* __restrict__ bank,
                                                            int Fp, float* __restrict__ knn, long long* __restrict__ idx) {
  __shared__ unsigned long long buf[TOPK_CAP];
  __shared__ double exact[TOPK_MAX_SEL], rankv[TOPK_MAX_SEL];
  __shared__ int cnt;
  pdl_launch_dependents();
  pdl_wait();
  const long long row = blockIdx.x;
  unsigned long long* rrow = run + row * ks;
  for (int i = threadIdx.x; i < ks; i += TOPK_TPB) buf[i] = first ? 0ull : rrow[i];
  if (threadIdx.x == 0) cnt = 0;
  __syncthreads();
  unsigned long long thresh = buf[ks - 1];
  const float* s = sim + row * ld;
  for (int base = 0; base < ncols; base += TOPK_TPB) {
    const int c = base + threadIdx.x;
    if (c < ncols) {
      const unsigned long long key = topk_key(__ldg(s + c), col0 + c);
      if (key > thresh) buf[ks + atomicAdd(&cnt, 1)] = key;
    }
    __syncthreads();
    const int m = cnt;
    __syncthreads();
    if (m > 0 && (m > TOPK_CAP - ks - TOPK_TPB || base + TOPK_TPB >= ncols)) {
      int P = 1;
      while (P < ks + m) P <<= 1;
      for (int i = ks + m + threadIdx.x; i < P; i += TOPK_TPB) buf[i] = 0ull;
      __syncthreads();
      topk_sort(buf, P);
      thresh = buf[ks - 1];
      if (threadIdx.x == 0) cnt = 0;
      __syncthreads();
    }
  }
  if (!last) {
    for (int i = threadIdx.x; i < ks; i += TOPK_TPB) rrow[i] = buf[i];
    return;
  }
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  for (int i = warp; i < ks; i += TOPK_TPB / 32) {
    const long long b = (uint32_t)~(uint32_t)buf[i];
    double acc = 0.0;
    for (int j = lane; j < Fp; j += 32) acc = fma((double)__ldg(q + row * Fp + j), (double)__ldg(bank + b * Fp + j), acc);
    acc = warp_sum(acc);
    if (lane == 0) { exact[i] = acc; rankv[i] = isnan(acc) ? -INFINITY : acc; }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < ks; i += TOPK_TPB) {
    const double si = rankv[i];
    const uint32_t bi = ~(uint32_t)buf[i];
    int rank = 0;
    for (int j = 0; j < ks; ++j) {
      const uint32_t bj = ~(uint32_t)buf[j];
      rank += rankv[j] > si || (rankv[j] == si && bj < bi);
    }
    if (rank < k && idx) idx[row * k + rank] = (long long)bi;
    if (rank == k - 1 && knn) knn[row] = (float)(2.0 - 2.0 * exact[i]);
  }
}

}  // namespace

int ood_moments(const float* f, const int64_t* y, int64_t n, int F, int C, int accumulate, double* sums, int64_t* counts,
                double* gram, cudaStream_t st) {
  if (gram) {
    const dim3 grid((unsigned)ceil_div(F, MOM_TILE), (unsigned)ceil_div(F, MOM_TILE));
    launch_pdl(ood_gram_kernel, grid, dim3(MOM_TILE * MOM_TILE), 0, st, f, (long long)n, F, accumulate, gram);
    RD_CHECK_LAUNCH("ood_gram_kernel");
  }
  if (sums) {
    launch_pdl(ood_class_sums_kernel, dim3((unsigned)ceil_div(F, MOM_CLASS_TPB), (unsigned)C), dim3(MOM_CLASS_TPB), 0, st,
               f, y, (long long)n, F, accumulate, sums, reinterpret_cast<long long*>(counts));
    RD_CHECK_LAUNCH("ood_class_sums_kernel");
  }
  return 0;
}

int ood_rows(const float* f, int64_t ldf, int64_t n, int F, const double* mu, int ld, float* out, cudaStream_t st) {
  launch_pdl(ood_rows_kernel, dim3((unsigned)ceil_div(n, ROW_WARPS)), dim3(32 * ROW_WARPS), 0, st, f, (long long)ldf,
             (long long)n, F, mu, ld, out);
  RD_CHECK_LAUNCH("ood_rows_kernel");
  return 0;
}

int ood_logit_scores(const float* logits, int n, int C, float temperature, float* msp, float* energy, cudaStream_t st) {
  launch_pdl(ood_logit_kernel, dim3((unsigned)ceil_div(n, 128)), dim3(128), 0, st, logits, n, C, temperature, msp, energy);
  RD_CHECK_LAUNCH("ood_logit_kernel");
  return 0;
}

int ood_class_dist(const float* Z, const float* M, int n, int C, int rp, float* dist, float* dmin, int64_t* cls,
                   cudaStream_t st) {
  launch_pdl(ood_class_dist_kernel, dim3((unsigned)ceil_div(n, ROW_WARPS)), dim3(32 * ROW_WARPS), 0, st, Z, M, n, C, rp,
             dist, dmin, reinterpret_cast<long long*>(cls));
  RD_CHECK_LAUNCH("ood_class_dist_kernel");
  return 0;
}

int ood_topk(const float* sim, int64_t ld, int n, int ncols, int64_t col0, int k, int ks, int first, int last,
             uint64_t* run, const float* q, const float* bank, int Fp, float* knn, int64_t* idx, cudaStream_t st) {
  launch_pdl(ood_topk_kernel, dim3((unsigned)n), dim3(TOPK_TPB), 0, st, sim, (long long)ld, ncols, (long long)col0, k,
             ks, first, last, reinterpret_cast<unsigned long long*>(run), q, bank, Fp, knn, reinterpret_cast<long long*>(idx));
  RD_CHECK_LAUNCH("ood_topk_kernel");
  return 0;
}

}  // namespace rd
