// Counterfactual explanations of Raindrop_v2 (rd_raindrop_v2_counterfactual): the kernels that run between the chunk's
// eval forward, frozen-parameter backward and dX0 GEMM (rd_model.cu orchestrates them).
//
// A chunk of m samples b = c0 .. c0+m-1 runs on m*R rows, sample-major: row j = i*R + r is replica r of chunk sample i,
// so a chunk always holds whole samples.  The forward reads the FISTA extrapolation point y_k from the chunk's input
// buffers (x_e [T, m*R, 2N], st_e [m*R, ds]).  The deltas of x_k and y_k are kept apart, per row [m*R, E] with
// E = T*N + ds: element e < T*N is value cell (t, n) = (e / N, e % N), the rest the statics.  Mutable elements (S_b):
// value cells with mask > 0 of a mutable sensor, plus the statics when pst.  Every other element of x_e holds the input
// bit for bit; an element with delta == 0 is written as x (not x + 0, which would turn -0 into +0).
//
// Element arithmetic is fp32.  Per-row and per-sample sums, distances and the loss weights c are fp64.  Every per-row or
// per-sample kernel is one CTA that walks its elements in a fixed order and sums with a fixed-order block reduction: no
// atomics, so results are bitwise reproducible and independent of the chunking.
#include <math.h>

#include "rd_kernels.cuh"

namespace rd {
namespace {

constexpr int CF_THREADS = 256, CF_TPB = 256;

struct Elem { float x, w, lo, hi; float* xe; bool p; };

// element e of chunk row j: its input value, weight and effective box [min(lower, x), max(upper, x)], its place in the
// chunk's input buffers, whether it is mutable
__device__ __forceinline__ Elem elem(const CfArgs& a, int j, int e) {
  const int b = a.c0 + j / a.R, TN = a.T * a.N;
  Elem o;
  int col;
  if (e < TN) {
    const int t = e / a.N, n = e - t * a.N;
    const long long r = ((long long)t * a.B + b) * (2 * a.N);
    o.x = __ldg(a.src + r + n);
    o.xe = a.x_e + ((long long)t * a.m * a.R + j) * (2 * a.N) + n;
    o.p = perturbable_cell(a.src, r, a.N, n, a.sens);
    col = n;
  } else {
    const int k = e - TN;
    o.x = __ldg(a.statics + (long long)b * a.ds + k);
    o.xe = a.st_e + (long long)j * a.ds + k;
    o.p = a.pst != 0;
    col = a.N + k;
  }
  o.w = a.w ? __ldg(a.w + col) : 1.f;
  o.lo = fminf(a.lo ? __ldg(a.lo + col) : -INFINITY, o.x);
  o.hi = fmaxf(a.hi ? __ldg(a.hi + col) : INFINITY, o.x);
  return o;
}

// clip_box in delta units, and the iterate written into the chunk's input buffers: x where delta == 0, else x + delta
// clamped to the box (so the box holds on the input the model sees, whatever the rounding of x + delta)
__device__ __forceinline__ float clip_box(const Elem& o, float d) { return fminf(fmaxf(d, o.lo - o.x), o.hi - o.x); }
__device__ __forceinline__ float iterate(const Elem& o, float d) {
  return d == 0.f ? o.x : fminf(fmaxf(o.x + d, o.lo), o.hi);
}

// the distance terms of one element: |w d| and (w d)^2, exact products in fp64
__device__ __forceinline__ void dist_terms(float w, float d, double* l1, double* l2) {
  const double v = (double)w * (double)d;
  *l1 += fabs(v);
  *l2 += v * v;
}

// word (idx & 3) of Philox block idx >> 2 at site SITE_CF_START
__device__ __forceinline__ uint32_t start_word(const RngKey& k, uint64_t idx) {
  const uint4 w = dropout_block(k, SITE_CF_START, idx);
  const uint32_t s = (uint32_t)idx & 3u;
  return s == 0 ? w.x : (s == 1 ? w.y : (s == 2 ? w.z : w.w));
}

// The chunk's inputs: every row j = i*R + r a copy of sample c0 + i (src rows, statics, times, lengths), one launch.
__global__ void cf_expand_kernel(const __grid_constant__ CfArgs a, long long n_src, long long n_tok, long long n_stat) {
  pdl_launch_dependents();
  pdl_wait();
  const long long rows = (long long)a.m * a.R;
  long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o < n_src) {
    const int w = 2 * a.N;
    const long long tj = o / w, t = tj / rows;
    const int c = (int)(o - tj * w), j = (int)(tj - t * rows);
    a.x_e[o] = __ldg(a.src + (t * a.B + a.c0 + j / a.R) * w + c);
    return;
  }
  o -= n_src;
  if (o < n_tok) {
    const long long t = o / rows;
    a.times_e[o] = __ldg(a.times + t * a.B + a.c0 + (o - t * rows) / a.R);
    return;
  }
  o -= n_tok;
  if (o < n_stat) {
    const long long j = o / a.ds;
    a.st_e[o] = __ldg(a.statics + (long long)(a.c0 + j / a.R) * a.ds + (o - j * a.ds));
    return;
  }
  o -= n_stat;
  if (o < rows) a.len_e[o] = __ldg(a.lengths + a.c0 + o / a.R);
}

// Sample b = c0 + blockIdx.x after the forward at x (its logits: row i*R of `logits`): the clean logits, the target
// (target[b], or target == NULL: the first argmax over c != the first argmax), the outputs of a sample without a valid
// point (x, the clean logits, +inf), and its replicas' bisection state c = c_init, lo = 0, hi = +inf.
__global__ void __launch_bounds__(CF_THREADS) cf_init_kernel(const __grid_constant__ CfArgs a,
                                                            const __grid_constant__ CfOut k, const int64_t* target,
                                                            double c_init) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x, b = a.c0 + i, nc = k.ncls;
  const float* l = k.logits + (long long)i * a.R * nc;
  int tgt;
  if (target) {
    tgt = (int)__ldg(target + b);
  } else {
    int pred = 0;
    for (int c = 1; c < nc; ++c)
      if (l[c] > l[pred]) pred = c;
    tgt = -1;
    for (int c = 0; c < nc; ++c)
      if (c != pred && (tgt < 0 || l[c] > l[tgt])) tgt = c;
  }
  for (int c = threadIdx.x; c < nc; c += CF_THREADS) {
    k.logits_clean[(long long)b * nc + c] = l[c];
    k.logits_cf[(long long)b * nc + c] = l[c];
  }
  const int w = 2 * a.N;
  for (long long e = threadIdx.x; e < (long long)a.T * w; e += CF_THREADS) {
    const long long t = e / w, c = e - t * w, r = (t * a.B + b) * w + c;
    k.src_cf[r] = __ldg(a.src + r);
  }
  if (k.st_cf)
    for (int e = threadIdx.x; e < a.ds; e += CF_THREADS) k.st_cf[(long long)b * a.ds + e] = __ldg(a.statics + (long long)b * a.ds + e);
  for (int r = threadIdx.x; r < a.R; r += CF_THREADS) {
    double* s = a.row + (long long)(i * a.R + r) * CF_ROW;
    s[CF_C] = c_init; s[CF_LO] = 0.0; s[CF_HI] = INFINITY;
  }
  if (threadIdx.x == 0) {
    k.target_out[b] = tgt;
    k.valid[b] = 0;
    k.distance[b] = INFINITY;
    a.best[i] = INFINITY;
  }
}

// Row j = blockIdx.x at the start of a round: x_0 = y_0 = the replica's start point (replica 0: delta = 0; replica r >= 1:
// clip_box(init_scale (2u - 1)) on S_b, u = (word >> 8) 2^-24 of index (b*R + r)*E + e at key {seed, step}) into the
// deltas and the chunk's input buffers, its distance, and the round's valid flag cleared.
__global__ void __launch_bounds__(CF_THREADS) cf_start_kernel(const __grid_constant__ CfArgs a, float init_scale,
                                                             float beta, const uint64_t* __restrict__ key) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double red[CF_THREADS / 32];
  const int j = blockIdx.x, r = j % a.R, b = a.c0 + j / a.R;
  const RngKey k = load_rng_key(r > 0 ? key : nullptr);
  const int TN = a.T * a.N, E = TN + a.ds, ne = TN + (a.pst ? a.ds : 0);
  const uint64_t base = ((uint64_t)b * (uint64_t)a.R + (uint64_t)r) * (uint64_t)E;
  float* xd = a.xd + (long long)j * E;
  float* yd = a.yd + (long long)j * E;
  double l1 = 0.0, l2 = 0.0;
  for (int e = threadIdx.x; e < ne; e += CF_THREADS) {
    const Elem o = elem(a, j, e);
    if (!o.p) continue;
    float d = 0.f;
    if (r > 0) {
      const float u = (float)(start_word(k, base + e) >> 8) * (1.f / 16777216.f);
      d = clip_box(o, init_scale * (2.f * u - 1.f));
    }
    xd[e] = d;
    yd[e] = d;
    *o.xe = iterate(o, d);
    dist_terms(o.w, d, &l1, &l2);
  }
  l1 = block_sum_fixed(l1, red);
  l2 = block_sum_fixed(l2, red);
  if (threadIdx.x == 0) {
    double* s = a.row + (long long)j * CF_ROW;
    s[CF_DIST] = __dadd_rn(__dmul_rn((double)beta, l1), l2);
    s[CF_FLAG] = 0.0;
  }
}

// Sample b = c0 + blockIdx.x at the points whose logits are `logits` [m*R, ncls]: per replica row j the margin
// m = z_t - max_{c != t} z_c (first index c* on ties) in fp64, the hinge seed d_logits[j] = c_j (e_{c*} - e_t) when
// m <= kappa (else 0), and validity (m > 0 and m >= kappa), which sets the round's flag.  The valid replica of smallest
// distance (ties: the lowest) replaces the sample's best when its distance is strictly smaller (ties keep the earlier
// point): its input rows, logits and distance are copied out.
__global__ void __launch_bounds__(CF_THREADS) cf_track_kernel(const __grid_constant__ CfArgs a,
                                                             const __grid_constant__ CfOut k, double kappa,
                                                             float* __restrict__ dlogits) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x, b = a.c0 + i, nc = k.ncls;
  const int t = (int)k.target_out[b];
  const double prev = a.best[i];
  double bd = INFINITY;
  int br = -1;
  for (int r = 0; r < a.R; ++r) {
    const int j = i * a.R + r;
    const float* l = k.logits + (long long)j * nc;
    int cs = -1;
    for (int c = 0; c < nc; ++c)
      if (c != t && (cs < 0 || l[c] > l[cs])) cs = c;
    const double mg = (double)l[t] - (double)l[cs];
    const bool active = mg <= kappa, valid = mg > 0.0 && mg >= kappa;
    double* s = a.row + (long long)j * CF_ROW;
    const float cf = active ? (float)s[CF_C] : 0.f;
    for (int c = threadIdx.x; c < nc; c += CF_THREADS)
      dlogits[(long long)j * nc + c] = c == cs ? cf : (c == t ? -cf : 0.f);
    if (valid) {
      const double d = s[CF_DIST];
      if (d < bd) { bd = d; br = r; }
      if (threadIdx.x == 0) s[CF_FLAG] = 1.0;
    }
  }
  __syncthreads();                                    // every thread has read best[i] before thread 0 writes it
  if (br < 0 || !(bd < prev)) return;
  const int j = i * a.R + br;
  if (threadIdx.x == 0) {
    a.best[i] = bd;
    k.distance[b] = bd;
    k.valid[b] = 1;
  }
  for (int c = threadIdx.x; c < nc; c += CF_THREADS) k.logits_cf[(long long)b * nc + c] = k.logits[(long long)j * nc + c];
  const long long rows = (long long)a.m * a.R;
  const int w = 2 * a.N;
  for (long long e = threadIdx.x; e < (long long)a.T * w; e += CF_THREADS) {
    const long long tt = e / w, c = e - tt * w;
    k.src_cf[(tt * a.B + b) * w + c] = a.x_e[(tt * rows + j) * w + c];
  }
  if (k.st_cf)
    for (int e = threadIdx.x; e < a.ds; e += CF_THREADS) k.st_cf[(long long)b * a.ds + e] = a.st_e[(long long)j * a.ds + e];
}

// One FISTA step of row j = blockIdx.x from the backward of its hinge: per element of S_b, in fp32,
//   g = (lift backward of dX0 at y_k, or the statics through dfeat . W_emb) + 2 w^2 y_k
//   x_{k+1} = clip_box(S(y_k - alpha g, alpha beta w)),  S(v, l) = sign(v) max(|v| - l, 0)
//   y_{k+1} = clip_box(x_{k+1} + k/(k+3) (x_{k+1} - x_k))
// then y_{k+1} into the chunk's input buffers and its distance beta ||w y||_1 + ||w y||_2^2 (fp64).
struct CfStepArgs {
  const float* R_u; const float* dX0; const float* dfeat; const float* W_emb;
  int d_ob, Df, D, emb, k;
  float alpha, beta;
};
__device__ __forceinline__ float elem_grad(const CfArgs& a, const CfStepArgs& s, int j, int e, const Elem& o) {
  const int TN = a.T * a.N;
  if (e < TN) {
    const int t = e / a.N, n = e - t * a.N;
    const float* g = s.dX0 + ((long long)j * a.N + n) * ((long long)a.T * s.d_ob) + (long long)t * s.d_ob;
    return lift_bwd(*o.xe, s.R_u, g, n, s.d_ob, 0.f, nullptr, 0);
  }
  return emb_bwd(s.dfeat + (long long)j * s.Df + s.D, s.W_emb, s.emb, a.ds, e - TN);
}
__global__ void __launch_bounds__(CF_THREADS) cf_step_kernel(const __grid_constant__ CfArgs a,
                                                            const __grid_constant__ CfStepArgs s) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double red[CF_THREADS / 32];
  const int j = blockIdx.x;
  const int TN = a.T * a.N, E = TN + a.ds, ne = TN + (a.pst ? a.ds : 0);
  const float mom = (float)s.k / (float)(s.k + 3);
  float* xd = a.xd + (long long)j * E;
  float* yd = a.yd + (long long)j * E;
  double l1 = 0.0, l2 = 0.0;
  for (int e = threadIdx.x; e < ne; e += CF_THREADS) {
    const Elem o = elem(a, j, e);
    if (!o.p) continue;
    const float y = yd[e], xo = xd[e];
    const float g = __fadd_rn(elem_grad(a, s, j, e, o), __fmul_rn(__fmul_rn(2.f, __fmul_rn(o.w, o.w)), y));
    const float v = __fsub_rn(y, __fmul_rn(s.alpha, g));
    const float lam = __fmul_rn(__fmul_rn(s.alpha, s.beta), o.w);
    const float av = fabsf(v) - lam;
    const float xn = clip_box(o, av > 0.f ? copysignf(av, v) : 0.f);
    const float yn = clip_box(o, __fadd_rn(xn, __fmul_rn(mom, __fsub_rn(xn, xo))));
    xd[e] = xn;
    yd[e] = yn;
    *o.xe = iterate(o, yn);
    dist_terms(o.w, yn, &l1, &l2);
  }
  l1 = block_sum_fixed(l1, red);
  l2 = block_sum_fixed(l2, red);
  if (threadIdx.x == 0) a.row[(long long)j * CF_ROW + CF_DIST] = __dadd_rn(__dmul_rn((double)s.beta, l1), l2);
}

// After round `round`: row j's flag into round_valid [B, R, n_search], the bisection of its c in fp64
//   valid round: hi = min(hi, c), c = (lo + hi) / 2;  else lo = max(lo, c), c = hi < inf ? (lo + hi) / 2 : 10 c
// and c into c_final [B, R].
__global__ void cf_round_kernel(const __grid_constant__ CfArgs a, int round, int n_search, uint8_t* __restrict__ round_valid,
                                double* __restrict__ c_final) {
  pdl_launch_dependents();
  pdl_wait();
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.m * a.R) return;
  double* s = a.row + (long long)j * CF_ROW;
  const long long br = (long long)a.c0 * a.R + j;      // = (b*R + r)
  const bool ok = s[CF_FLAG] != 0.0;
  double c = s[CF_C], lo = s[CF_LO], hi = s[CF_HI];
  if (ok) {
    hi = fmin(hi, c);
    c = __dadd_rn(lo, hi) / 2.0;
  } else {
    lo = fmax(lo, c);
    c = hi < INFINITY ? __dadd_rn(lo, hi) / 2.0 : __dmul_rn(10.0, c);
  }
  s[CF_C] = c; s[CF_LO] = lo; s[CF_HI] = hi;
  round_valid[br * n_search + round] = ok ? 1 : 0;
  c_final[br] = c;
}

}  // namespace

int cf_expand(const CfArgs& a, cudaStream_t st) {
  const long long rows = (long long)a.m * a.R;
  const long long n_src = (long long)a.T * rows * 2 * a.N, n_tok = (long long)a.T * rows, n_stat = rows * a.ds;
  const long long n = n_src + n_tok + n_stat + rows;
  launch_pdl(cf_expand_kernel, dim3((unsigned)ceil_div(n, CF_TPB)), dim3(CF_TPB), 0, st, a, n_src, n_tok, n_stat);
  RD_CHECK_LAUNCH("cf_expand_kernel");
  return 0;
}

int cf_init(const CfArgs& a, const CfOut& k, const int64_t* target, double c_init, cudaStream_t st) {
  launch_pdl(cf_init_kernel, dim3(a.m), dim3(CF_THREADS), 0, st, a, k, target, c_init);
  RD_CHECK_LAUNCH("cf_init_kernel");
  return 0;
}

int cf_start(const CfArgs& a, float init_scale, float beta, const uint64_t* key, cudaStream_t st) {
  launch_pdl(cf_start_kernel, dim3(a.m * a.R), dim3(CF_THREADS), 0, st, a, init_scale, beta, key);
  RD_CHECK_LAUNCH("cf_start_kernel");
  return 0;
}

int cf_track(const CfArgs& a, const CfOut& k, double kappa, float* dlogits, cudaStream_t st) {
  launch_pdl(cf_track_kernel, dim3(a.m), dim3(CF_THREADS), 0, st, a, k, kappa, dlogits);
  RD_CHECK_LAUNCH("cf_track_kernel");
  return 0;
}

int cf_step(const CfArgs& a, int k, float alpha, float beta, const float* R_u, int d_ob, const float* dX0,
            const float* dfeat, int Df, int D, const float* W_emb, int emb, cudaStream_t st) {
  CfStepArgs s;
  s.R_u = R_u; s.dX0 = dX0; s.dfeat = dfeat; s.W_emb = W_emb;
  s.d_ob = d_ob; s.Df = Df; s.D = D; s.emb = emb; s.k = k; s.alpha = alpha; s.beta = beta;
  launch_pdl(cf_step_kernel, dim3(a.m * a.R), dim3(CF_THREADS), 0, st, a, s);
  RD_CHECK_LAUNCH("cf_step_kernel");
  return 0;
}

int cf_round(const CfArgs& a, int round, int n_search, uint8_t* round_valid, double* c_final, cudaStream_t st) {
  const int rows = a.m * a.R;
  launch_pdl(cf_round_kernel, dim3((unsigned)ceil_div(rows, 128)), dim3(128), 0, st, a, round, n_search, round_valid,
             c_final);
  RD_CHECK_LAUNCH("cf_round_kernel");
  return 0;
}

}  // namespace rd
