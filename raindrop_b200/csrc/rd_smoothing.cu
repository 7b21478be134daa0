// Randomized smoothing of Raindrop_v2 (rd_raindrop_v2_smooth_counts): the noisy replicate expansion and the per-sample
// class votes that run around each chunk's eval forward (rd_model.cu orchestrates them).
//
// Replicate m of sample b is x + sigma z with z ~ N(0, I) on S_b (value cells with mask > 0 of perturbable sensors, plus
// the statics when pst) and x elsewhere.  z of element e (e = t*N + n for value cells, T*N + j for statics) is drawn at
// key {seed, step + m} and index b*(T*N + ds) + e, so a replicate depends on (seed, step + m, b) alone: not on B, not on
// the chunking.  An element whose noise is 0 (sigma = 0) is written as x, not x + 0 (which would turn -0 into +0).
#include <math.h>

#include "rd_kernels.cuh"

namespace rd {
namespace {

constexpr int SMOOTH_TPB = 256, VOTE_THREADS = 128;

struct SmoothExpandArgs {
  const float* src; const float* statics; const float* times; const int64_t* lengths; const uint8_t* sens;
  const uint64_t* rng; float* src_e; float* statics_e; float* times_e; int64_t* lengths_e;
  long long m0;
  float sigma;
  int B, nc, T, N, ds, pst;
};

__device__ __forceinline__ float noisy(const SmoothExpandArgs& a, float x, int m, uint64_t idx) {
  const uint64_t seed = a.rng[0], step = a.rng[1] + (uint64_t)a.m0 + (uint64_t)m;
  const RngKey k{(uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(step >> 32), (uint32_t)step};
  const float d = a.sigma * philox_normal(k, SITE_SMOOTH, idx);
  return d == 0.f ? x : x + d;
}

// one thread per output element of the replicate-major expansion (rep_expand_elem)
__global__ void smooth_expand_kernel(const __grid_constant__ SmoothExpandArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const RepElem e = rep_expand_elem((long long)blockIdx.x * blockDim.x + threadIdx.x, a.B, a.nc, a.T, a.N, a.ds);
  const uint64_t base = (uint64_t)e.b * ((uint64_t)a.T * a.N + a.ds);
  switch (e.part) {
    case REP_SRC: {
      const float x = __ldg(a.src + e.in);
      const bool p = a.sigma > 0.f && e.k < a.N && perturbable_cell(a.src, e.in - e.k, a.N, e.k, a.sens);
      a.src_e[e.out] = p ? noisy(a, x, e.m, base + (uint64_t)e.t * a.N + e.k) : x;
      break;
    }
    case REP_TIMES:
      if (a.times_e) a.times_e[e.out] = __ldg(a.times + e.in);
      break;
    case REP_STATICS: {
      const float x = __ldg(a.statics + e.in);
      a.statics_e[e.out] = a.pst && a.sigma > 0.f ? noisy(a, x, e.m, base + (uint64_t)a.T * a.N + e.k) : x;
      break;
    }
    case REP_LENGTHS:
      if (a.lengths_e) a.lengths_e[e.out] = __ldg(a.lengths + e.in);
      break;
    default: break;
  }
}

// One CTA per sample b: the argmax of each of its nc rows m*B + b (first maximum, as torch.argmax; a row with a
// non-finite logit votes for no class) counted in shared memory, then added to counts[b, :].  Counts are integers, so
// the order of the votes does not matter and the result is exact.
__global__ void __launch_bounds__(VOTE_THREADS) smooth_vote_kernel(const float* __restrict__ logits, int B, int nc, int C,
                                                                   int first, long long* __restrict__ counts) {
  extern __shared__ int votes[];
  pdl_launch_dependents();
  const int b = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += VOTE_THREADS) votes[c] = 0;
  __syncthreads();
  pdl_wait();
  for (int m = threadIdx.x; m < nc; m += VOTE_THREADS) {
    const float* row = logits + ((long long)m * B + b) * C;
    float top = __ldg(row);
    bool ok = isfinite(top);
    int arg = 0;
    for (int c = 1; c < C; ++c) {
      const float v = __ldg(row + c);
      ok = ok && isfinite(v);
      if (v > top) { top = v; arg = c; }
    }
    if (ok) atomicAdd(votes + arg, 1);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += VOTE_THREADS) {
    long long* o = counts + (long long)b * C + c;
    *o = (first ? 0LL : *o) + votes[c];
  }
}

}  // namespace

int smooth_expand(const float* src, const float* statics, const float* times, const int64_t* lengths, const uint8_t* sens,
                  int pst, float sigma, const uint64_t* rng, int64_t m0, int B, int nc, int T, int N, int ds, float* src_e,
                  float* statics_e, float* times_e, int64_t* lengths_e, cudaStream_t st) {
  SmoothExpandArgs a;
  a.src = src; a.statics = ds > 0 ? statics : nullptr; a.times = times; a.lengths = lengths; a.sens = sens; a.rng = rng;
  a.src_e = src_e; a.statics_e = statics_e; a.times_e = times_e; a.lengths_e = lengths_e;
  a.m0 = m0; a.sigma = sigma; a.B = B; a.nc = nc; a.T = T; a.N = N; a.ds = ds; a.pst = pst && ds > 0;
  const int64_t Bc = (int64_t)B * nc;
  const int64_t n = Bc * T * 2 * N + Bc * T + Bc * ds + Bc;
  if (ceil_div(n, SMOOTH_TPB) > 0x7fffffffLL) { set_error("smooth_expand: %lld elements are too many", (long long)n); return -2; }
  launch_pdl(smooth_expand_kernel, dim3((unsigned)ceil_div(n, SMOOTH_TPB)), dim3(SMOOTH_TPB), 0, st, a);
  RD_CHECK_LAUNCH("smooth_expand_kernel");
  return 0;
}

int smooth_vote(const float* logits, int B, int nc, int ncls, int first, int64_t* counts, cudaStream_t st) {
  launch_pdl(smooth_vote_kernel, dim3(B), dim3(VOTE_THREADS), (size_t)ncls * sizeof(int), st, logits, B, nc, ncls, first,
             reinterpret_cast<long long*>(counts));
  RD_CHECK_LAUNCH("smooth_vote_kernel");
  return 0;
}

}  // namespace rd
