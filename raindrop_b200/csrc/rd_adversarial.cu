// Projected gradient descent (PGD) adversarial examples of Raindrop_v2 (rd_raindrop_v2_pgd): the kernels that run between
// the chunk's eval forward, frozen-parameter backward and dX0 GEMM (rd_model.cu orchestrates them).
//
// A chunk of m samples b = c0 .. c0+m-1 runs on m rows; its forward reads the iterate x_k from the chunk's input
// buffers (x_e [T, m, 2N], st_e [m, ds]).  The perturbation delta is kept apart from x_e, per sample [m, E] with
// E = T*N + ds: element e < T*N is value cell (t, n) = (e / N, e % N), the rest the statics.  Perturbable elements
// (S_b): value cells with mask > 0 of a perturbable sensor, plus the statics when perturb_static, of attacked samples.
// Every other element of x_e holds the input bit for bit and its delta stays 0; an element with delta == 0 is written
// as x (not x + 0, which would turn -0 into +0).
//
// Every per-sample kernel is one CTA per sample that walks the sample's elements in a fixed order and sums in fp64
// with a fixed-order block reduction: no atomics, so results are bitwise reproducible and independent of the chunking.
#include <math.h>

#include "rd_kernels.cuh"

namespace rd {
namespace {

constexpr int PGD_THREADS = 256, PGD_TPB = 256;

struct Elem { float x; float* xe; bool p; };

// element e of chunk sample j: its input value, its place in the chunk's input buffers, whether it is perturbable
__device__ __forceinline__ Elem elem(const PgdArgs& a, int j, int e) {
  const int b = a.c0 + j, TN = a.T * a.N;
  Elem o;
  if (e < TN) {
    const int t = e / a.N, n = e - t * a.N;
    const long long r = ((long long)t * a.B + b) * (2 * a.N);
    o.x = __ldg(a.src + r + n);
    o.xe = a.x_e + ((long long)t * a.m + j) * (2 * a.N) + n;
    o.p = perturbable_cell(a.src, r, a.N, n, a.sens);
  } else {
    const int k = e - TN;
    o.x = __ldg(a.statics + (long long)b * a.ds + k);
    o.xe = a.st_e + (long long)j * a.ds + k;
    o.p = a.pst != 0;
  }
  return o;
}

__device__ __forceinline__ float iterate(float x, float d) { return d == 0.f ? x : x + d; }

__device__ __forceinline__ bool attacked(const PgdArgs& a, int j) { return !a.attacked || a.attacked[a.c0 + j]; }

// word (idx & 3) of Philox block idx >> 2 at site SITE_PGD_START
__device__ __forceinline__ uint32_t start_word(const RngKey& k, uint64_t idx) {
  const uint4 w = dropout_block(k, SITE_PGD_START, idx);
  const uint32_t s = (uint32_t)idx & 3u;
  return s == 0 ? w.x : (s == 1 ? w.y : (s == 2 ? w.z : w.w));
}

// The chunk's inputs (src rows, statics, times, lengths of samples c0 .. c0+m-1) and delta = 0, one launch.
__global__ void pgd_expand_kernel(const __grid_constant__ PgdArgs a, long long n_src, long long n_tok, long long n_stat,
                                  long long n_delta) {
  pdl_launch_dependents();
  pdl_wait();
  long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o < n_src) {
    const int w = 2 * a.N;
    const long long tj = o / w, t = tj / a.m;
    const int c = (int)(o - tj * w), j = (int)(tj - t * a.m);
    a.x_e[o] = __ldg(a.src + (t * a.B + a.c0 + j) * w + c);
    return;
  }
  o -= n_src;
  if (o < n_tok) {
    const long long t = o / a.m;
    a.times_e[o] = __ldg(a.times + t * a.B + a.c0 + (o - t * a.m));
    return;
  }
  o -= n_tok;
  if (o < n_stat) {
    a.st_e[o] = __ldg(a.statics + (long long)a.c0 * a.ds + o);
    return;
  }
  o -= n_stat;
  if (o < a.m) {
    a.len_e[o] = __ldg(a.lengths + a.c0 + o);
    return;
  }
  o -= a.m;
  if (o < n_delta) a.delta[o] = 0.f;
}

// Random start of sample b = c0 + blockIdx.x.  Element e draws at index b*(E + 1) + e, the radius at b*(E + 1) + E:
//   linf: delta = eps * (2u - 1), u = (word >> 8) 2^-24 (exact until the one fp32 rounding of the product)
//   l2:   delta = eps * r^(1/d) * z / ||z||, z the element's normal, r = (word >> 8) 2^-24, d = |S_b|, in fp64
__global__ void __launch_bounds__(PGD_THREADS) pgd_start_kernel(const __grid_constant__ PgdArgs a, int norm, float eps,
                                                                const uint64_t* __restrict__ key) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double red[PGD_THREADS / 32];
  const int j = blockIdx.x;
  if (!attacked(a, j)) return;
  const RngKey k = load_rng_key(key);
  const int TN = a.T * a.N, E = TN + a.ds, ne = TN + (a.pst ? a.ds : 0);
  const uint64_t base = (uint64_t)(a.c0 + j) * (uint64_t)(E + 1);
  float* dl = a.delta + (long long)j * E;
  if (norm == RD_PGD_LINF) {
    for (int e = threadIdx.x; e < ne; e += PGD_THREADS) {
      const Elem o = elem(a, j, e);
      if (!o.p) continue;
      const float u = (float)(start_word(k, base + e) >> 8) * (1.f / 16777216.f);
      const float d = eps * (2.f * u - 1.f);
      dl[e] = d;
      *o.xe = iterate(o.x, d);
    }
    return;
  }
  double zz = 0.0, cnt = 0.0;
  for (int e = threadIdx.x; e < ne; e += PGD_THREADS) {
    if (!elem(a, j, e).p) continue;
    const float z = philox_normal(k, SITE_PGD_START, base + e);
    dl[e] = z;
    zz += (double)z * (double)z;
    cnt += 1.0;
  }
  zz = block_sum_fixed(zz, red);
  cnt = block_sum_fixed(cnt, red);
  const double r = (double)(start_word(k, base + E) >> 8) * (1.0 / 16777216.0);
  const double s = zz > 0.0 ? (double)eps * pow(r, 1.0 / cnt) / sqrt(zz) : 0.0;
  for (int e = threadIdx.x; e < ne; e += PGD_THREADS) {
    const Elem o = elem(a, j, e);
    if (!o.p) continue;
    const float d = (float)((double)dl[e] * s);
    dl[e] = d;
    *o.xe = iterate(o.x, d);
  }
}

// Sample b = c0 + blockIdx.x at the iterate whose logits are `logits` [m, ncls]: cross-entropy in fp64 against
// y[b] (y == NULL: the first argmax of logits_clean[b]); d_logits = softmax - onehot; when the loss beats the best
// so far (first: always) it becomes the best and the iterate's inputs, logits and loss are copied out.
struct PgdTrackArgs {
  const float* logits; const float* logits_clean; const int64_t* y; double* best; float* dlogits;
  float* src_adv; float* st_adv; float* logits_adv; float* loss_adv; int ncls, first;
};
__global__ void __launch_bounds__(PGD_THREADS) pgd_track_kernel(const __grid_constant__ PgdArgs a,
                                                                const __grid_constant__ PgdTrackArgs k) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double red[PGD_THREADS / 32];
  const int j = blockIdx.x, b = a.c0 + j, nc = k.ncls;
  const float* l = k.logits + (long long)j * nc;
  int lab = 0;
  if (k.y) {
    lab = (int)__ldg(k.y + b);
  } else {
    const float* lc = k.logits_clean + (long long)b * nc;
    float top = lc[0];
    for (int c = 1; c < nc; ++c)
      if (lc[c] > top) { top = lc[c]; lab = c; }
  }
  double mx = (double)l[0];
  for (int c = 1; c < nc; ++c) mx = fmax(mx, (double)l[c]);
  double se = 0.0;
#pragma unroll 1
  for (int c = threadIdx.x; c < nc; c += PGD_THREADS) se += exp((double)l[c] - mx);
  const double prev = k.first ? 0.0 : k.best[j];      // read before thread 0 can write it (the sum below syncs)
  se = block_sum_fixed(se, red);
  const double lse = mx + log(se), loss = lse - (double)l[lab];
#pragma unroll 1
  for (int c = threadIdx.x; c < nc; c += PGD_THREADS)
    k.dlogits[(long long)j * nc + c] = (float)(exp((double)l[c] - lse) - (c == lab ? 1.0 : 0.0));
  if (!k.first && !(loss > prev)) return;           // ties keep the earlier iterate
  if (threadIdx.x == 0) {
    k.best[j] = loss;
    k.loss_adv[b] = (float)loss;
  }
  for (int c = threadIdx.x; c < nc; c += PGD_THREADS) k.logits_adv[(long long)b * nc + c] = l[c];
  const int w = 2 * a.N;
  for (long long i = threadIdx.x; i < (long long)a.T * w; i += PGD_THREADS) {
    const long long t = i / w, c = i - t * w;
    k.src_adv[(t * a.B + b) * w + c] = a.x_e[(t * a.m + j) * w + c];
  }
  if (k.st_adv)
    for (int i = threadIdx.x; i < a.ds; i += PGD_THREADS) k.st_adv[(long long)b * a.ds + i] = a.st_e[(long long)j * a.ds + i];
}

// One PGD step of sample b = c0 + blockIdx.x from the backward of its loss: g = d(loss_b)/d(element) (the lift backward
// of dX0 at the iterate's value, eval: no dropout; the statics through d(loss)/d(emb output) . W_emb), then
//   linf: delta = clip(delta + alpha sign(g), -eps, eps) in fp32
//   l2:   delta += alpha g / ||g|| (no step when ||g|| = 0), then delta *= min(1, eps / ||delta||), norms in fp64
// and x_{k+1} into the chunk's input buffers.
struct PgdStepArgs {
  const float* R_u; const float* dX0; const float* dfeat; const float* W_emb;
  int d_ob, Df, D, emb, norm;
  float eps, alpha;
};
__device__ __forceinline__ float elem_grad(const PgdArgs& a, const PgdStepArgs& s, int j, int e, const Elem& o) {
  const int TN = a.T * a.N;
  if (e < TN) {
    const int t = e / a.N, n = e - t * a.N;
    const float* g = s.dX0 + ((long long)j * a.N + n) * ((long long)a.T * s.d_ob) + (long long)t * s.d_ob;
    return lift_bwd(*o.xe, s.R_u, g, n, s.d_ob, 0.f, nullptr, 0);
  }
  return emb_bwd(s.dfeat + (long long)j * s.Df + s.D, s.W_emb, s.emb, a.ds, e - TN);
}
__global__ void __launch_bounds__(PGD_THREADS) pgd_step_kernel(const __grid_constant__ PgdArgs a,
                                                               const __grid_constant__ PgdStepArgs s) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ double red[PGD_THREADS / 32];
  const int j = blockIdx.x;
  if (!attacked(a, j)) return;
  const int TN = a.T * a.N, E = TN + a.ds, ne = TN + (a.pst ? a.ds : 0);
  float* dl = a.delta + (long long)j * E;
  if (s.norm == RD_PGD_LINF) {
    for (int e = threadIdx.x; e < ne; e += PGD_THREADS) {
      const Elem o = elem(a, j, e);
      if (!o.p) continue;
      const float g = elem_grad(a, s, j, e, o);
      const float sg = g > 0.f ? 1.f : (g < 0.f ? -1.f : 0.f);
      const float d = fminf(fmaxf(dl[e] + s.alpha * sg, -s.eps), s.eps);
      dl[e] = d;
      *o.xe = iterate(o.x, d);
    }
    return;
  }
  float* gb = a.grad + (long long)j * E;
  double gg = 0.0;
  for (int e = threadIdx.x; e < ne; e += PGD_THREADS) {
    const Elem o = elem(a, j, e);
    if (!o.p) continue;
    const float g = elem_grad(a, s, j, e, o);
    gb[e] = g;
    gg += (double)g * (double)g;
  }
  const double gn = sqrt(block_sum_fixed(gg, red));
  if (gn == 0.0) return;
  const double step = (double)s.alpha / gn;
  double dd = 0.0;
  for (int e = threadIdx.x; e < ne; e += PGD_THREADS) {
    if (!elem(a, j, e).p) continue;
    const float d = (float)((double)dl[e] + step * (double)gb[e]);
    dl[e] = d;
    dd += (double)d * (double)d;
  }
  const double dn = sqrt(block_sum_fixed(dd, red));
  const double sc = dn > (double)s.eps ? (double)s.eps / dn : 1.0;
  for (int e = threadIdx.x; e < ne; e += PGD_THREADS) {
    const Elem o = elem(a, j, e);
    if (!o.p) continue;
    const float d = sc < 1.0 ? (float)((double)dl[e] * sc) : dl[e];
    dl[e] = d;
    *o.xe = iterate(o.x, d);
  }
}

}  // namespace

int pgd_expand(const PgdArgs& a, cudaStream_t st) {
  const long long n_src = (long long)a.T * a.m * 2 * a.N, n_tok = (long long)a.T * a.m, n_stat = (long long)a.m * a.ds;
  const long long n_delta = (long long)a.m * ((long long)a.T * a.N + a.ds);
  const long long n = n_src + n_tok + n_stat + a.m + n_delta;
  launch_pdl(pgd_expand_kernel, dim3((unsigned)ceil_div(n, PGD_TPB)), dim3(PGD_TPB), 0, st, a, n_src, n_tok, n_stat, n_delta);
  RD_CHECK_LAUNCH("pgd_expand_kernel");
  return 0;
}

int pgd_start(const PgdArgs& a, int norm, float eps, const uint64_t* key, cudaStream_t st) {
  launch_pdl(pgd_start_kernel, dim3(a.m), dim3(PGD_THREADS), 0, st, a, norm, eps, key);
  RD_CHECK_LAUNCH("pgd_start_kernel");
  return 0;
}

int pgd_track(const PgdArgs& a, int ncls, const float* logits, const float* logits_clean, const int64_t* y, double* best,
              int first, float* dlogits, float* src_adv, float* st_adv, float* logits_adv, float* loss_adv, cudaStream_t st) {
  PgdTrackArgs k;
  k.logits = logits; k.logits_clean = logits_clean; k.y = y; k.best = best; k.dlogits = dlogits;
  k.src_adv = src_adv; k.st_adv = a.ds > 0 ? st_adv : nullptr; k.logits_adv = logits_adv; k.loss_adv = loss_adv;
  k.ncls = ncls; k.first = first;
  launch_pdl(pgd_track_kernel, dim3(a.m), dim3(PGD_THREADS), 0, st, a, k);
  RD_CHECK_LAUNCH("pgd_track_kernel");
  return 0;
}

int pgd_step(const PgdArgs& a, int norm, float eps, float alpha, const float* R_u, int d_ob, const float* dX0,
             const float* dfeat, int Df, int D, const float* W_emb, int emb, cudaStream_t st) {
  PgdStepArgs s;
  s.R_u = R_u; s.dX0 = dX0; s.dfeat = dfeat; s.W_emb = W_emb;
  s.d_ob = d_ob; s.Df = Df; s.D = D; s.emb = emb; s.norm = norm; s.eps = eps; s.alpha = alpha;
  launch_pdl(pgd_step_kernel, dim3(a.m), dim3(PGD_THREADS), 0, st, a, s);
  RD_CHECK_LAUNCH("pgd_step_kernel");
  return 0;
}

}  // namespace rd
