// Randomized smoothing of Raindrop_v2 (rd_raindrop_v2_smooth_counts): the noisy replicate expansion and the per-sample
// class votes that run around each chunk's eval forward (rd_model.cu orchestrates them).
//
// Replicate m of sample b is x + sigma z with z ~ N(0, I) on S_b (value cells with mask > 0 of perturbable sensors, plus
// the statics when pst) and x elsewhere.  z of element e (e = t*N + n for value cells, T*N + j for statics) is drawn at
// key {seed, step + m} and index b*(T*N + ds) + e, so a replicate depends on (seed, step + m, b) alone: not on B, not on
// the chunking.  An element whose noise is 0 (sigma = 0) is written as x, not x + 0 (which would turn -0 into +0).
//
// Randomized ablation (rd_raindrop_v2_ablation_counts, Levine & Feizi 2020) shares the vote kernel.  Replicate m of
// sample b keeps k of the P players (the sensors of sens in increasing n, then the statics when ast) and writes +0.0
// into the data of the others.  Its keep table row comes from one thread: the subset of lexicographic rank step + m
// (exhaustive), or a partial Fisher-Yates shuffle of 0..P-1 whose swap targets are Lemire's unbiased bounded integers
// over the 32-bit words (b << 32) + j of key {seed, step + m} at SITE_ABLATE (word idx & 3 of block idx >> 2).  A row
// depends on (seed, step + m, b) alone.  Sorting random keys would be simpler but is not uniform under ties, and the
// certificate assumes an exactly uniform k-subset.
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

// ---- randomized ablation ----------------------------------------------------------------------------------------------
constexpr int ABLATE_ROWS_TPB = 128, ABLATE_PERM_SMEM = 48 * 1024;

struct AblateKeepArgs {
  const uint64_t* rng; uint8_t* keep;
  long long m0, J;
  int B, nc, P, k;
};

// One thread per row j = m*B + b of the chunk.  Sampled mode (J == 0) shuffles in shared memory: thread i's
// permutation holds position q at perm[q * blockDim.x + i] (uint16, P <= RD_ABLATION_MAX_PLAYERS).
__global__ void __launch_bounds__(ABLATE_ROWS_TPB) ablate_keep_kernel(const __grid_constant__ AblateKeepArgs a) {
  extern __shared__ uint16_t perm_s[];
  pdl_launch_dependents();
  pdl_wait();
  const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= (long long)a.B * a.nc) return;
  const int m = (int)(row / a.B), b = (int)(row - (long long)m * a.B), P = a.P, k = a.k;
  uint8_t* out = a.keep + row * P;
  for (int p = 0; p < P; ++p) out[p] = 0;
  const uint64_t seed = a.rng[0], step = a.rng[1] + (uint64_t)a.m0 + (uint64_t)m;
  if (a.J > 0) {
    // unrank: at each position i the next candidate x leads C(P-x-1, k-i-1) subsets; c tracks that binomial as x and i
    // advance (every value is <= C(P, k) = J < 2^31, and each division below is exact)
    if (step >= (uint64_t)a.J) return;
    uint64_t r = step, c = (uint64_t)a.J * k / P;     // C(P-1, k-1)
    int x = 0;
    for (int i = 0; i < k; ++i) {
      const int mm = k - i - 1;                       // c = C(P-x-1, mm)
      while (r >= c) {
        r -= c;
        const int n = P - x - 1;                      // C(n-1, mm) = C(n, mm) (n - mm) / n
        c = c * (uint64_t)(n - mm) / (uint64_t)n;
        ++x;
      }
      out[x] = 1;
      const int n = P - x - 1;                        // next position: C(n-1, mm-1) = C(n, mm) mm / n
      if (mm > 0) c = c * (uint64_t)mm / (uint64_t)n;
      ++x;
    }
    return;
  }
  WordStream w;
  w.key = RngKey{(uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(step >> 32), (uint32_t)step};
  w.site = SITE_ABLATE;
  w.idx = (uint64_t)b << 32;
  uint16_t* perm = perm_s + threadIdx.x;
  const int ld = blockDim.x;
  for (int p = 0; p < P; ++p) perm[p * ld] = (uint16_t)p;
  for (int i = 0; i < k; ++i) {
    const int j = i + (int)bounded(w, (uint32_t)(P - i));
    const uint16_t t = perm[i * ld];
    perm[i * ld] = perm[j * ld];
    perm[j * ld] = t;
  }
  for (int i = 0; i < k; ++i) out[perm[i * ld]] = 1;
}

struct AblateExpandArgs {
  const float* src; const float* statics; const float* times; const int64_t* lengths; const uint8_t* sens;
  const uint8_t* keep; float* src_e; float* statics_e; float* times_e; int64_t* lengths_e;
  int B, nc, T, N, ds, P, G, ast, amask;
};

// One thread per output element of the replicate-major expansion; player [N] (shared) maps a sensor to its player
// index, -1 for a sensor that is not a player.  A player index >= G (n_players smaller than the sensors of sens) is
// read as not a player, so the table is never read past its row.
__global__ void ablate_expand_kernel(const __grid_constant__ AblateExpandArgs a) {
  extern __shared__ int player[];
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x < 32) {
    int carry = 0;
    for (int n0 = 0; n0 < a.N; n0 += 32) {
      const int n = n0 + threadIdx.x;
      const bool v = n < a.N && (!a.sens || a.sens[n]);
      const unsigned bal = __ballot_sync(0xffffffffu, v);
      if (n < a.N) player[n] = v ? carry + __popc(bal & ((1u << threadIdx.x) - 1u)) : -1;
      carry += __popc(bal);
    }
  }
  __syncthreads();
  const RepElem e = rep_expand_elem((long long)blockIdx.x * blockDim.x + threadIdx.x, a.B, a.nc, a.T, a.N, a.ds);
  const uint8_t* kept = a.keep + ((long long)e.m * a.B + e.b) * a.P;
  switch (e.part) {
    case REP_SRC: {
      const float x = __ldg(a.src + e.in);
      const int n = e.k < a.N ? e.k : e.k - a.N, p = player[n];
      const bool ablated = (e.k < a.N || a.amask) && p >= 0 && p < a.G && !kept[p];
      a.src_e[e.out] = ablated ? 0.f : x;
      break;
    }
    case REP_TIMES:
      if (a.times_e) a.times_e[e.out] = __ldg(a.times + e.in);
      break;
    case REP_STATICS:
      a.statics_e[e.out] = a.ast && !kept[a.P - 1] ? 0.f : __ldg(a.statics + e.in);
      break;
    case REP_LENGTHS:
      if (a.lengths_e) a.lengths_e[e.out] = __ldg(a.lengths + e.in);
      break;
    default: break;
  }
}

}  // namespace

int ablate_inputs(const float* src, const float* statics, const float* times, const int64_t* lengths, const uint8_t* sens,
                  int P, int ast, int amask, int k, int64_t J, const uint64_t* rng, int64_t m0, int B, int nc, int T, int N,
                  int ds, uint8_t* keep, float* src_e, float* statics_e, float* times_e, int64_t* lengths_e, cudaStream_t st) {
  const int64_t Bc = (int64_t)B * nc;
  const int64_t n = Bc * T * 2 * N + Bc * T + Bc * ds + Bc;
  if (ceil_div(n, SMOOTH_TPB) > 0x7fffffffLL) { set_error("ablate_inputs: %lld elements are too many", (long long)n); return -2; }
  AblateKeepArgs ka;
  ka.rng = rng; ka.keep = keep; ka.m0 = m0; ka.J = J; ka.B = B; ka.nc = nc; ka.P = P; ka.k = k;
  int tpb = ABLATE_PERM_SMEM / (int)(P * sizeof(uint16_t));
  tpb = tpb > ABLATE_ROWS_TPB ? ABLATE_ROWS_TPB : (tpb < 1 ? 1 : tpb);
  const size_t smem = J > 0 ? 0 : (size_t)tpb * P * sizeof(uint16_t);
  launch_pdl(ablate_keep_kernel, dim3((unsigned)ceil_div(Bc, tpb)), dim3(tpb), smem, st, ka);
  RD_CHECK_LAUNCH("ablate_keep_kernel");
  return ablate_expand(src, statics, times, lengths, sens, P, ast, amask, B, nc, T, N, ds, keep, src_e, statics_e, times_e,
                       lengths_e, st);
}

int ablate_expand(const float* src, const float* statics, const float* times, const int64_t* lengths, const uint8_t* sens,
                  int P, int ast, int amask, int B, int nc, int T, int N, int ds, const uint8_t* keep, float* src_e,
                  float* statics_e, float* times_e, int64_t* lengths_e, cudaStream_t st) {
  const int64_t Bc = (int64_t)B * nc;
  const int64_t n = Bc * T * 2 * N + Bc * T + Bc * ds + Bc;
  if (ceil_div(n, SMOOTH_TPB) > 0x7fffffffLL) { set_error("ablate_expand: %lld elements are too many", (long long)n); return -2; }
  AblateExpandArgs a;
  a.src = src; a.statics = ds > 0 ? statics : nullptr; a.times = times; a.lengths = lengths; a.sens = sens; a.keep = keep;
  a.src_e = src_e; a.statics_e = statics_e; a.times_e = times_e; a.lengths_e = lengths_e;
  a.B = B; a.nc = nc; a.T = T; a.N = N; a.ds = ds; a.P = P; a.ast = ast && ds > 0; a.amask = amask;
  a.G = P - a.ast;
  launch_pdl(ablate_expand_kernel, dim3((unsigned)ceil_div(n, SMOOTH_TPB)), dim3(SMOOTH_TPB), (size_t)N * sizeof(int), st, a);
  RD_CHECK_LAUNCH("ablate_expand_kernel");
  return 0;
}

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
