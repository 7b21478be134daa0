// Early prediction of Raindrop_v2 (rd_raindrop_v2_prefix_logits): the prefix expansion that runs before each chunk's
// eval forward (rd_model.cu orchestrates it), and the same launches for one truncated copy per training step
// (rd_debug_prefix_inputs).
//
// Prefix r of sample b (0 <= r <= T) keeps rows t < r bit for bit and writes +0.0 into both halves of src and into
// times at rows t >= r, which is how a shorter record is padded; the statics are copied.  Its length is lengths[b] for
// r >= T, else min(lengths[b], #{t < r : times[t, b] > 0}), the rule lengths follow (times > 0 counted per sample)
// applied to the truncated record.  By horizon h, r is the number of leading rows with times <= h (counted up to the
// first row whose time exceeds h), so it is a prefix even for unsorted times.
//
// Training cutoffs (rng given, one per slot b): R_b = 1 + the last row with times > 0 and f_b the first (R_b = 0: the
// slot keeps its record).  The first word of the stream (b << 32) + j at key {seed, step}, site SITE_PREFIX, keeps the
// whole record (r = T) when it is below floor(p_full 2^32); otherwise r = lo_b + U(R_b - lo_b + 1), U Lemire's bounded
// integer over the next words and lo_b = max(f_b + 1, ceil(min_fraction R_b)), so the prefix holds row f_b and has
// length >= 1 whenever lengths[b] >= 1.
#include <math.h>

#include "rd_kernels.cuh"

namespace rd {
namespace {

constexpr int CUTOFF_TPB = 128, EXPAND_TPB = 256;

__device__ int horizon_cutoff(const float* __restrict__ times, int B, int T, int b, float h) {
  int r = 0;
  while (r < T && __ldg(times + (long long)r * B + b) <= h) ++r;
  return r;
}

__device__ int drawn_cutoff(const PrefixArgs& a, int b) {
  int first = -1, last = -1;
  for (int t = 0; t < a.T; ++t) {
    if (__ldg(a.times + (long long)t * a.B + b) > 0.f) {
      if (first < 0) first = t;
      last = t;
    }
  }
  if (last < 0) return a.T;
  const int R = last + 1;
  const uint64_t seed = a.rng[0], step = a.rng[1];
  WordStream w;
  w.key = RngKey{(uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(step >> 32), (uint32_t)step};
  w.site = SITE_PREFIX;
  w.idx = (uint64_t)b << 32;
  if ((uint64_t)w.next() < a.full_below) return a.T;
  const int frac = (int)ceil(a.min_fraction * (double)R);
  const int lo = first + 1 > frac ? first + 1 : frac;
  return lo + (int)bounded(w, (uint32_t)(R - lo + 1));
}

// one thread per (m, b): the cutoff and the prefix's length
__global__ void __launch_bounds__(CUTOFF_TPB) prefix_cutoff_kernel(const __grid_constant__ PrefixArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= (long long)a.B * a.nc) return;
  const int m = (int)(j / a.B), b = (int)(j - (long long)m * a.B), k = a.k0 + m;
  int r;
  if (a.rng) {
    r = a.rows && a.rows[b] >= 0 ? min(a.rows[b], a.T) : drawn_cutoff(a, b);
  } else if (a.horizons) {
    r = horizon_cutoff(a.times, a.B, a.T, b, __ldg(a.horizons + k));
  } else {
    r = min(max(__ldg(a.rows + k), 0), a.T);
  }
  a.table[j] = r;
  if (a.cutoffs) a.cutoffs[(long long)k * a.B + b] = r;
  const int64_t len = __ldg(a.lengths + b);
  int64_t n = len;
  if (r < a.T) {
    int c = 0;
    for (int t = 0; t < r; ++t) c += __ldg(a.times + (long long)t * a.B + b) > 0.f;
    n = c < len ? c : len;
  }
  a.lengths_e[j] = n;
  if (a.lengths_out) a.lengths_out[(long long)k * a.B + b] = n;
}

// one thread per output element of the replicate-major expansion (rep_expand_elem), replicate m = prefix k0 + m; the
// lengths were written by prefix_cutoff_kernel
__global__ void __launch_bounds__(EXPAND_TPB) prefix_expand_kernel(const __grid_constant__ PrefixArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const RepElem e = rep_expand_elem((long long)blockIdx.x * blockDim.x + threadIdx.x, a.B, a.nc, a.T, a.N, a.ds);
  if (e.part == REP_NONE || e.part == REP_LENGTHS) return;
  const int r = a.table[(long long)e.m * a.B + e.b];
  switch (e.part) {
    case REP_SRC: a.src_e[e.out] = e.t < r ? __ldg(a.src + e.in) : 0.f; break;
    case REP_TIMES: a.times_e[e.out] = e.t < r ? __ldg(a.times + e.in) : 0.f; break;
    case REP_STATICS: if (a.statics_e) a.statics_e[e.out] = __ldg(a.statics + e.in); break;
    default: break;
  }
}

}  // namespace

int prefix_inputs(const PrefixArgs& a, cudaStream_t st) {
  const int64_t Bc = (int64_t)a.B * a.nc;
  const int64_t n = Bc * a.T * 2 * a.N + Bc * a.T + Bc * a.ds + Bc;
  if (ceil_div(n, EXPAND_TPB) > 0x7fffffffLL) { set_error("prefix_inputs: %lld elements are too many", (long long)n); return -2; }
  launch_pdl(prefix_cutoff_kernel, dim3((unsigned)ceil_div(Bc, CUTOFF_TPB)), dim3(CUTOFF_TPB), 0, st, a);
  RD_CHECK_LAUNCH("prefix_cutoff_kernel");
  launch_pdl(prefix_expand_kernel, dim3((unsigned)ceil_div(n, EXPAND_TPB)), dim3(EXPAND_TPB), 0, st, a);
  RD_CHECK_LAUNCH("prefix_expand_kernel");
  return 0;
}

}  // namespace rd
