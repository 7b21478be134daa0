// Launch wrappers for the non-GEMM kernels of the hot path (rd_kernels.cu).
#pragma once
#include "rd_common.cuh"

namespace rd {

// out[t, j, :] = src[t, idx[j], :] for a device-resident training set (code/Raindrop.py:311-315 does this on the host)
int gather_batch(const float* src, const int64_t* idx, int64_t T, int64_t n_total, int width, int B, float* out,
                 cudaStream_t st);

int rng_capture(uint64_t* rng_state, uint64_t* captured, int advance, cudaStream_t st);

// device-side input pipeline (rd_kernels.cu; mirrors code/utils_rd.py:149-175,221-257 and code/Raindrop.py:214-231,311-317)
int64_t feature_stats_scratch_bytes(int64_t n, int T, int F);
int feature_stats(const float* raw, int64_t n, int T, int F, float* mean, float* stdv, void* scratch, cudaStream_t st);
int mask_normalize(const float* raw, const float* mean, const float* stdv, int64_t n, int T, int F, float* out,
                   const float* minutes, float* times_out, cudaStream_t st);
int zero_features(float* P, int64_t T, int B, int width, const int64_t* idx, int K, int per_sample, cudaStream_t st);
int assemble_batch(const float* P, const float* Pt, const float* Ps, const int64_t* y, const int64_t* idx, int T, int64_t n_total,
                   int width, int ds, int B, float* src, float* times, float* statics, int64_t* y_out, int64_t* lengths,
                   cudaStream_t st);

// X0[(b*N+n), t*d_ob+k] = dropout(relu(src[t,b,n] * R_u[n*d_ob+k]))    code/models_rd.py:285-296,323-327
// round != 0: values are rounded (RN) to TF32 so the tensor-core layer reads them exactly.
// The same launch writes the positional encoding of `times` into pe_out[tok*ld + col0 ..+16] (src == nullptr
// or times == nullptr skips that half).
// rep.B > 0: the lift dropout of replicate-major rows (rep_remap, rd_common.cuh).
int lift_posenc(const float* src, const float* R_u, int B, int T, int N, int d_ob, float drop_p, const uint64_t* rng,
                int round, float* X0, const float* times, int64_t n_tokens, const float* ts_host, int d_pe, float* pe_out,
                int64_t ld, int col0, cudaStream_t st, DropRep rep = {});

// y [cols, rows] = RN_tf32(x [rows, cols])^T
int transpose_round(const float* x, int rows, int cols, float* y, cudaStream_t st);

int posenc(const float* times, int64_t n_tokens, const float* ts_host, int d_pe, float* out, int64_t ld, int col0,
           cudaStream_t st);

// Backward of lift_posenc and of the static embedding in one launch (each output may be null, which skips its part):
//   d_src [T, B, 2N]  from dX0 = d(loss)/d(X0) [B*N, T*d_ob] (the forward's lift dropout mask is replayed from rng;
//                     the mask half is written as 0)
//   d_times [n_tokens] from the positional-encoding columns g_pe[tok*ld + col0 .. + d_pe); lengths (optional, token
//                     = t*B + b) zeroes the padded rows t >= lengths[b]
//   d_static [B, ds]  = dfeat[:, feat_col0 : feat_col0 + emb] . W_emb   (W_emb: [emb, ds])
int input_grad(const float* src, const float* R_u, const float* dX0, int B, int T, int N, int d_ob, float drop_p,
               const uint64_t* rng, float* d_src, const float* times, const float* g_pe, int64_t n_tokens, int64_t ld, int col0,
               const float* ts_host, int d_pe, const int64_t* lengths, float* d_times, const float* dfeat, int Df, int feat_col0,
               const float* W_emb, int emb, int ds, float* d_static, cudaStream_t st);

// The lift backward of one (sample, t, sensor n) with value sv: sum_k g[k] * keep_k/(1-p) * [sv*R_u[n*d_ob+k] > 0] *
// R_u[n*d_ob+k], g = d(loss)/d(X0) of that (row, t); idx0 = the forward's dropout element index of channel 0
__device__ __forceinline__ float lift_bwd(float sv, const float* __restrict__ R_u, const float* __restrict__ g, int n,
                                          int d_ob, float drop_p, const uint64_t* __restrict__ rng, uint64_t idx0) {
  const float ik = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  float acc = 0.f;
  if (d_ob == 4) {
    const float4 r = __ldg(reinterpret_cast<const float4*>(R_u) + n);
    float4 d = __ldg(reinterpret_cast<const float4*>(g));
    if (drop_p > 0.f) {
      const float4 m = dropout_scale4(rng, SITE_LIFT, idx0, drop_p, ik);
      d.x *= m.x; d.y *= m.y; d.z *= m.z; d.w *= m.w;
    }
    acc = (sv * r.x > 0.f ? d.x * r.x : 0.f) + (sv * r.y > 0.f ? d.y * r.y : 0.f) +
          (sv * r.z > 0.f ? d.z * r.z : 0.f) + (sv * r.w > 0.f ? d.w * r.w : 0.f);
  } else {
    for (int k = 0; k < d_ob; ++k) {
      const float r = __ldg(R_u + n * d_ob + k);
      float d = __ldg(g + k);
      if (drop_p > 0.f) d *= dropout_scale(rng, SITE_LIFT, idx0 + k, drop_p, ik);
      acc += sv * r > 0.f ? d * r : 0.f;
    }
  }
  return acc;
}
// d(loss)/d(static[b, k]) = sum_n df[n] * W_emb[n*ds + k], df = d(loss)/d(emb output) of sample b
__device__ __forceinline__ float emb_bwd(const float* __restrict__ df, const float* __restrict__ W_emb, int emb, int ds, int k) {
  float acc = 0.f;
  for (int n = 0; n < emb; ++n) acc = fmaf(__ldg(df + n), __ldg(W_emb + (long long)n * ds + k), acc);
  return acc;
}

// Integrated gradients along the straight path x0 + alpha (x - x0), chunks of m steps on B*m rows, step-major (j = k*B + b).
// ig_expand: the chunk's inputs src_e [T, B*m, 2N] (value half interpolated, mask half copied from src), statics_e,
// times_e, lengths_e and one-hot d_logits [B*m, ncls] of target[b] (target == nullptr: argmax of logits_x [B, ncls];
// d_logits == nullptr skips it).  alphas == nullptr: the two endpoints alpha = 0, 1 (m = 2).
int ig_expand(const float* src, const float* src0, const float* statics, const float* statics0, const float* times,
              const int64_t* lengths, const float* alphas, int m, int B, int T, int N, int ds, int ncls, const int64_t* target,
              const float* logits_x, float* src_e, float* statics_e, float* times_e, int64_t* lengths_e, float* d_logits,
              cudaStream_t st);
// ig_accumulate: running sums over the chunk's steps of weights[k] * (lift backward of dX0 [B*m*N, T*d_ob]) per (b, n, t)
// in acc_src [B*N*T], and of weights[k] * dfeat[:, feat_col0 : +emb] . W_emb per (b, j) in acc_static [B, ds];
// first: start from 0; last: write attr_src [T, B, 2N] = (src - src0) * sum (mask half 0) and attr_static = (statics -
// statics0) * sum instead of the running sums.  attr_static == nullptr skips the statics.
int ig_accumulate(const float* src, const float* src0, const float* alphas, const float* weights, int m, int B, int T, int N,
                  int d_ob, const float* R_u, const float* dX0, float* acc_src, float* attr_src, const float* statics,
                  const float* statics0, const float* dfeat, int Df, int feat_col0, const float* W_emb, int emb, int ds,
                  float* acc_static, float* attr_static, int first, int last, cudaStream_t st);

// The attributed class of sample b: target[b], or (target == NULL) the first maximum of logits_x[b, :], as torch.argmax
__device__ __forceinline__ int target_class(const int64_t* __restrict__ target, const float* __restrict__ logits_x, int b,
                                            int ncls) {
  if (target) return (int)__ldg(target + b);
  const float* l = logits_x + (long long)b * ncls;
  float best = __ldg(l);
  int tgt = 0;
  for (int c = 1; c < ncls; ++c) {
    const float v = __ldg(l + c);
    if (v > best) { best = v; tgt = c; }
  }
  return tgt;
}

// Coalition attribution over P players (value cell (t, b, n) belongs to player[t*stride_t + b*stride_b + n], ids in
// [0, G) are players, any other id none; the static player G = P-1 when ds > 0), chunks of nc coalitions c0 .. c0+nc-1
// on B*nc rows, coalition-major (j = ci*B + b); method RD_ATTR_SHAPLEY: coalition c = p*(P-1) + k-1 keeps orders[p, :k],
// RD_ATTR_ABLATION: coalition c keeps every player but c; COALITION_ENDPOINTS (nc = 2): the rows of x' (no player kept:
// the cells of no player keep x) and of x.
// coalition_expand: for Shapley one launch fills the chunk's keep table keep [nc, P] (uint8); then one launch writes
// src_e [T, B*nc, 2N] (value cell of a kept player or of no player from src, else from src0; mask half copied),
// statics_e, times_e, lengths_e.
#define COALITION_ENDPOINTS 2
int coalition_expand(const float* src, const float* src0, const float* statics, const float* statics0, const float* times,
                     const int64_t* lengths, const int32_t* player, int64_t stride_t, int64_t stride_b, const int32_t* orders,
                     int P, int G, int method, int c0, int nc, int B, int T, int N, int ds, uint8_t* keep, float* src_e,
                     float* statics_e, float* times_e, int64_t* lengths_e, cudaStream_t st);
// coalition_accumulate: adds the chunk's F = logits_c [B*nc, ncls] at target[b] (nullptr: argmax of ends[1]) into the
// fp64 running sums acc [B, P]; first: start from the endpoints ends [2, B, ncls] (at x', at x); last: write attr [B, P].
int coalition_accumulate(const float* logits_c, const float* ends, const int64_t* target, const int32_t* orders, int P,
                         int method, int m, int c0, int nc, int B, int ncls, double* acc, float* attr, int first, int last,
                         cudaStream_t st);
// COALITION_TABLE (KernelSHAP): coalition_expand reads `keep` as the chunk's rows of the caller's coalition table
// [nc, P] (uint8, nonzero = kept) and launches nothing to fill it; orders is not read.
#define COALITION_TABLE 3
// COALITION_ROWS (removal curves, infidelity): coalition_expand reads `keep` as a per-row table [nc*B, P] (uint8,
// nonzero = kept; row j = ci*B + b), which the caller filled, and launches nothing to fill it; orders is not read.
#define COALITION_ROWS 4
// kernel_shap_accumulate: adds sum_ci w[c] z[c, g] (F(c) - F(x')) over the chunk's coalitions c = c0 .. c0+nc-1 (F at
// target[b], nullptr: argmax of ends[1]) into the fp64 sums acc [B, P]; first: start from 0.
int kernel_shap_accumulate(const float* logits_c, const float* ends, const int64_t* target, const uint8_t* z,
                           const double* w, int P, int c0, int nc, int B, int ncls, double* acc, int first, cudaStream_t st);
// kernel_shap_solve: attr [B, P] = acc [B, P] . K^T + (F(x) - F(x')) k^T in fp64, solve = [K | k] [P, P+1]; P <= 4096.
int kernel_shap_solve(const double* acc, const double* solve, const float* ends, const int64_t* target, int P, int B,
                      int ncls, float* attr, cudaStream_t st);

// Replicate-major expansion of a B-sample batch into Bc = nc*B rows (row j = m*B + b): output element o of the
// concatenation src_e [T, Bc, 2N] | times_e [T, Bc] | statics_e [Bc, ds] | lengths_e [Bc] is element `out` of its part
// and reads element `in` of the batch's src [T, B, 2N] / times [T, B] / statics [B, ds] / lengths [B]; (m, b) is its
// row's replicate and sample, t its time step (src, times) and k its column (src, statics).
enum RepPart { REP_SRC, REP_TIMES, REP_STATICS, REP_LENGTHS, REP_NONE };
struct RepElem { int part, m, b, t, k; long long out, in; };
__device__ __forceinline__ RepElem rep_expand_elem(long long o, int B, int nc, int T, int N, int ds) {
  const long long Bc = (long long)B * nc, W = 2LL * N;
  const long long n_src = T * Bc * W, n_times = T * Bc, n_stat = Bc * ds;
  RepElem e;
  e.t = 0; e.k = 0;
  long long j = 0;
  if (o < n_src) {
    const long long r = o / W, t = r / Bc;
    e.part = REP_SRC; e.out = o; e.t = (int)t; e.k = (int)(o - r * W); j = r - t * Bc;
  } else if ((o -= n_src) < n_times) {
    const long long t = o / Bc;
    e.part = REP_TIMES; e.out = o; e.t = (int)t; j = o - t * Bc;
  } else if ((o -= n_times) < n_stat) {
    j = o / ds;
    e.part = REP_STATICS; e.out = o; e.k = (int)(o - j * ds);
  } else if ((o -= n_stat) < Bc) {
    e.part = REP_LENGTHS; e.out = o; j = o;
  } else {
    e.part = REP_NONE; e.out = e.in = 0; e.m = e.b = 0;
    return e;
  }
  e.m = (int)(j / B);
  e.b = (int)(j - (long long)e.m * B);
  switch (e.part) {
    case REP_SRC: e.in = ((long long)e.t * B + e.b) * W + e.k; break;
    case REP_TIMES: e.in = (long long)e.t * B + e.b; break;
    case REP_STATICS: e.in = (long long)e.b * ds + e.k; break;
    default: e.in = e.b;
  }
  return e;
}

// The 32-bit words (b << 32) + j, j = 0, 1, ... of one key at one Philox site: word idx & 3 of the block at counter
// idx >> 2, one block per four words (randomized ablation's subsets, early prediction's training cutoffs).
struct WordStream {
  RngKey key;
  uint32_t site;
  uint64_t idx;
  uint4 blk;
  __device__ uint32_t next() {
    if ((idx & 3) == 0) blk = dropout_block(key, site, idx);
    const uint32_t s = (uint32_t)idx++ & 3u;
    return s == 0 ? blk.x : (s == 1 ? blk.y : (s == 2 ? blk.z : blk.w));
  }
};

// Lemire's unbiased integer in [0, r), r >= 1: the high word of x * r, redrawn while the low word is below 2^32 mod r.
__device__ __forceinline__ uint32_t bounded(WordStream& w, uint32_t r) {
  uint64_t x = (uint64_t)w.next() * r;
  if ((uint32_t)x < r) {
    const uint32_t t = (0u - r) % r;
    while ((uint32_t)x < t) x = (uint64_t)w.next() * r;
  }
  return (uint32_t)(x >> 32);
}

// The PGD / randomized-smoothing threat model: value cell n of the src row starting at `row` (= (t*B + b) * 2N) may be
// perturbed when it is observed (mask > 0) and its sensor is perturbable (sens [N] uint8, NULL: every sensor).
__device__ __forceinline__ bool perturbable_cell(const float* __restrict__ src, long long row, int N, int n,
                                                 const uint8_t* __restrict__ sens) {
  return (!sens || sens[n]) && __ldg(src + row + N + n) > 0.f;
}

// Monte Carlo dropout over chunks of nc replicates on B*nc rows, replicate-major (j = m*B + b).
// mc_expand: src_e [T, B*nc, 2N], statics_e (ds > 0), times_e, lengths_e = nc copies of the batch.
int mc_expand(const float* src, const float* statics, const float* times, const int64_t* lengths, int B, int nc, int T,
              int N, int ds, float* src_e, float* statics_e, float* times_e, int64_t* lengths_e, cudaStream_t st);
// mc_accumulate: adds replicates m0 .. m0+nc-1 (logits [B*nc, ncls]) to the fp64 sums acc [B, 2*ncls + 1] in replicate
// order (first: from 0); samples (optional) [M, B, ncls] gets their logits; last: mean [B, ncls], var [B, ncls] and
// ent [3, B] = (predictive entropy, expected entropy, mutual information) over all M replicates.
int mc_accumulate(const float* logits, int nc, int B, int ncls, int64_t m0, int64_t M, double* acc, float* samples,
                  float* mean, float* var, float* ent, int first, int last, cudaStream_t st);

// ---- PGD adversarial examples (rd_adversarial.cu; rd_raindrop_v2_pgd) ----------------------------------------------
// A chunk of m samples c0 .. c0+m-1 of a B-sample batch on m rows: the chunk's input buffers x_e [T, m, 2N], st_e [m, ds]
// (ds = 0: NULL), times_e [T, m], len_e [m], the perturbation delta and the l2 gradient buffer grad [m, T*N + ds].
// sens [N] / attacked [B] (uint8, NULL = all) and pst (perturb the statics) select the perturbable elements.
constexpr uint32_t SITE_PGD_START = 98;     // Philox site of the random start (its key is the attack key {seed, step})
struct PgdArgs {
  const float* src; const float* statics; const float* times; const int64_t* lengths;
  const uint8_t* sens; const uint8_t* attacked;
  float* x_e; float* st_e; float* times_e; int64_t* len_e; float* delta; float* grad;
  int B, T, N, ds, m, c0, pst;
};
// the chunk's inputs copied from the batch, delta = 0
int pgd_expand(const PgdArgs& a, cudaStream_t st);
// delta_0 drawn at key {seed, step} (device uint64[2]) and x_0 = x + delta_0 into x_e / st_e; one CTA per sample
int pgd_start(const PgdArgs& a, int norm, float eps, const uint64_t* key, cudaStream_t st);
// per-sample fp64 cross-entropy of logits [m, ncls] (label y[b], y == NULL: argmax of logits_clean [B, ncls]),
// d_logits [m, ncls] = softmax - onehot, and when it beats best[j] (first: always) the iterate's src / statics / logits
// rows and loss copied out to the batch-wide outputs (st_adv may be NULL)
int pgd_track(const PgdArgs& a, int ncls, const float* logits, const float* logits_clean, const int64_t* y, double* best,
              int first, float* dlogits, float* src_adv, float* st_adv, float* logits_adv, float* loss_adv, cudaStream_t st);
// the step from dX0 [m*N, T*d_ob] and dfeat [m, Df] (statics gradient from columns D .. D+emb through W_emb [emb, ds])
int pgd_step(const PgdArgs& a, int norm, float eps, float alpha, const float* R_u, int d_ob, const float* dX0,
             const float* dfeat, int Df, int D, const float* W_emb, int emb, cudaStream_t st);

// ---- counterfactual explanations (rd_counterfactual.cu; rd_raindrop_v2_counterfactual) -----------------------------
// A chunk of m samples c0 .. c0+m-1 of a B-sample batch on m*R rows, sample-major (row j = i*R + r: replica r of chunk
// sample i): the chunk's input buffers x_e [T, m*R, 2N], st_e [m*R, ds] (ds = 0: NULL), times_e [T, m*R], len_e [m*R],
// the deltas of the FISTA iterates x_k and y_k, xd and yd [m*R, T*N + ds], the per-row state row [m*R, CF_ROW] (fp64)
// and the per-sample best distance best [m].  sens [N] (uint8, NULL = all) and pst (the statics too) select the mutable
// elements; w, lo, hi [N + ds] (NULL: 1, -inf, +inf) are the per-sensor / per-static-column weights and bounds.
constexpr uint32_t SITE_CF_START = 103;     // Philox site of the restarts' start points (key {seed, step})
enum CfRow { CF_C, CF_LO, CF_HI, CF_DIST, CF_FLAG, CF_ROW };   // c, bisection bounds, distance of y, round found valid
struct CfArgs {
  const float* src; const float* statics; const float* times; const int64_t* lengths;
  const uint8_t* sens; const float* w; const float* lo; const float* hi;
  float* x_e; float* st_e; float* times_e; int64_t* len_e; float* xd; float* yd; double* row; double* best;
  int B, T, N, ds, m, c0, R, pst;
};
// the chunk's logits [m*R, ncls] and the batch-wide outputs (st_cf may be NULL)
struct CfOut {
  const float* logits; float* logits_clean; float* logits_cf; float* src_cf; float* st_cf; int64_t* target_out;
  uint8_t* valid; double* distance; int ncls;
};
// every row a copy of its sample's inputs
int cf_expand(const CfArgs& a, cudaStream_t st);
// after the forward at x: clean logits, target (NULL: the runner-up), the outputs of "no valid point", c = c_init
int cf_init(const CfArgs& a, const CfOut& k, const int64_t* target, double c_init, cudaStream_t st);
// each row at its start point (key {seed, step}: device uint64[2], read for replicas r >= 1), its distance, flag cleared
int cf_start(const CfArgs& a, float init_scale, float beta, const uint64_t* key, cudaStream_t st);
// margins, hinge seeds d_logits [m*R, ncls], validity, and the best point per sample copied out
int cf_track(const CfArgs& a, const CfOut& k, double kappa, float* dlogits, cudaStream_t st);
// FISTA step k from dX0 [m*R*N, T*d_ob] and dfeat [m*R, Df] (statics gradient from columns D .. D+emb through W_emb)
int cf_step(const CfArgs& a, int k, float alpha, float beta, const float* R_u, int d_ob, const float* dX0,
            const float* dfeat, int Df, int D, const float* W_emb, int emb, cudaStream_t st);
// the bisection after round `round`; round_valid [B, R, n_search] (uint8), c_final [B, R]
int cf_round(const CfArgs& a, int round, int n_search, uint8_t* round_valid, double* c_final, cudaStream_t st);

// ---- randomized smoothing (rd_smoothing.cu; rd_raindrop_v2_smooth_counts) -------------------------------------------
constexpr uint32_t SITE_SMOOTH = 100;       // Philox site of the smoothing noise (its key is {seed, step + replicate})
// smooth_expand: replicates m0 .. m0+nc-1 of the batch as mc_expand lays them out, with x + sigma z on the perturbable
// elements (perturbable_cell over sens, the statics when pst), z drawn at key {rng[0], rng[1] + m0 + m} and index
// b*(T*N + ds) + e.  times_e / lengths_e may be NULL (skipped).
int smooth_expand(const float* src, const float* statics, const float* times, const int64_t* lengths, const uint8_t* sens,
                  int pst, float sigma, const uint64_t* rng, int64_t m0, int B, int nc, int T, int N, int ds, float* src_e,
                  float* statics_e, float* times_e, int64_t* lengths_e, cudaStream_t st);
// smooth_vote: counts [B, ncls] (+)= the argmax votes of logits [nc*B, ncls] (replicate-major; first: from 0)
int smooth_vote(const float* logits, int B, int nc, int ncls, int first, int64_t* counts, cudaStream_t st);

// ---- randomized ablation (rd_smoothing.cu; rd_raindrop_v2_ablation_counts) ------------------------------------------
constexpr uint32_t SITE_ABLATE = 101;       // Philox site of the sampled subsets (its key is {seed, step + replicate})
// The P players: the sensors n with sens[n] != 0 (sens NULL: every sensor) in increasing n, then the static vector when
// ast.  ablate_inputs runs two launches for replicates m0 .. m0+nc-1: the keep table keep [nc*B, P] (uint8, row
// j = m*B + b; J > 0: the subset of lexicographic rank rng[1] + m0 + m among the J = C(P, k) k-subsets, none for a rank
// >= J; J = 0: a partial Fisher-Yates shuffle drawn at key {rng[0], rng[1] + m0 + m}), then the replicate-major rows of
// mc_expand with each ablated player's value column (and mask column when amask, the statics for the static player)
// written as +0.0.  times_e / lengths_e may be NULL (skipped).
int ablate_inputs(const float* src, const float* statics, const float* times, const int64_t* lengths, const uint8_t* sens,
                  int P, int ast, int amask, int k, int64_t J, const uint64_t* rng, int64_t m0, int B, int nc, int T, int N,
                  int ds, uint8_t* keep, float* src_e, float* statics_e, float* times_e, int64_t* lengths_e, cudaStream_t st);
// ablate_expand: ablate_inputs' second launch alone, the rows of a keep table [nc*B, P] the caller wrote.
int ablate_expand(const float* src, const float* statics, const float* times, const int64_t* lengths, const uint8_t* sens,
                  int P, int ast, int amask, int B, int nc, int T, int N, int ds, const uint8_t* keep, float* src_e,
                  float* statics_e, float* times_e, int64_t* lengths_e, cudaStream_t st);

// ---- worst-case sensor removal (rd_sensor_attack.cu; rd_raindrop_v2_sensor_attack) --------------------------------
// One round's candidates are slots s0 .. s0+nc-1 of the chunk on nc*B rows, slot-major (row j = m*B + b for slot s0 + m).
// A candidate is a set of removed players, written as a keep row of P bytes (0 = removed), the table
// ablate_expand reads.  The beam of sample b is beam_n[b] sets of r - 1 players, sorted index lists
// beam [B, W, R] (int16).
struct SaKeepArgs {
  const int16_t* beam; const int32_t* beam_n; uint8_t* keep; uint8_t* valid;
  long long s0;
  int B, nc, P, W, R, r;
};
// sa_keep: the keep row of slot (w, p) = (s / P, s % P) is beam set w with player p also removed; valid[j] = 0 when
// w >= beam_n[b] or p is in set w (the row is then evaluated and ignored).
int sa_keep(const SaKeepArgs& a, cudaStream_t st);
// The running selection of one round and the result, per sample (sa_select: one CTA per sample).  Candidates and list
// entries are ordered by (score, sorted tuple of removed players); the list keeps the wsel smallest distinct ones.
struct SaSelectArgs {
  const float* logits; const uint8_t* keep; const uint8_t* valid;   // the chunk's rows; valid NULL: every row
  const int64_t* cls;                                               // y or the target [B] (NULL: the clean prediction)
  float* cscore; uint8_t* csucc;                                    // per candidate [B, cc]
  int32_t* yref; int32_t* done;                                     // [B]
  float* top_score; uint8_t* top_keep; int32_t* top_n;              // list ping-pong [2][B*W], [2][B*W*P], [2][B]
  float* trk_score; uint8_t* trk_keep; float* trk_logits; int32_t* trk_ok;   // best, best successful: [2][B], [2][B*P], ...
  int16_t* beam; int32_t* beam_n;
  uint8_t* removed; int64_t* n_removed; float* logits_out; float* clean_logits; float* score; float* best_score;
  int B, C, P, W, R, r, nc, cc, wsel, cur, first, last, targeted;
};
int sa_select(const SaSelectArgs& a, cudaStream_t st);

// ---- early prediction (rd_prefix.cu; rd_raindrop_v2_prefix_logits) -----------------------------------------------
constexpr uint32_t SITE_PREFIX = 104;       // Philox site of the training cutoffs (its key is {seed, step})
// prefix_inputs: prefixes k0 .. k0+nc-1 of the batch as mc_expand lays them out (row j = m*B + b for prefix k0 + m).
// One launch writes the cutoff r of each (m, b) into table [nc, B] and the prefix's length into lengths_e (and both into
// cutoffs / lengths_out [K, B] at row k0 + m when not NULL); one launch writes src_e, times_e (rows t >= r as +0.0) and statics_e
// (copied; NULL: skipped).  The cutoff of prefix k comes from horizons[k] (NULL: from rows[k], clipped to [0, T]); with
// rng the nc = 1 training cutoffs are drawn per slot instead (rows, when given, is per slot: rows[b] >= 0 overrides).
struct PrefixArgs {
  const float* src; const float* statics; const float* times; const int64_t* lengths;
  const float* horizons; const int32_t* rows; const uint64_t* rng;
  int32_t* table; int32_t* cutoffs; int64_t* lengths_out; float* src_e; float* statics_e; float* times_e;
  int64_t* lengths_e;
  uint64_t full_below;     // a first word below this keeps the whole record: floor(p_full 2^32)
  double min_fraction;
  int B, T, N, ds, k0, nc;
};
int prefix_inputs(const PrefixArgs& a, cudaStream_t st);

// ---- faithfulness of attributions by removal (rd_faithfulness.cu; rd_raindrop_v2_removal_curves / _infidelity) -----
constexpr uint32_t SITE_REMOVAL = 107;      // Philox site of infidelity's removal sets (its key is {seed, step + replicate})
// removal_rank: rank [B, P] (int32) = position of each player when sample b's attributions attr [B, P] are sorted by
// `order` (RD_REMOVAL_*), ties to the lower index, -0 as +0, NaN last; one CTA per sample, P <= RD_REMOVAL_MAX_PLAYERS.
int removal_rank(const float* attr, int B, int P, int order, int32_t* rank, cudaStream_t st);
// removal_curve_keep: the keep table [nc*B, P] of (curve, count) pairs q0 .. q0+nc-1 (pair q: deletion at counts[q] for
// q < K, insertion at counts[q - K] after), row j = (q - q0)*B + b: deletion keeps rank >= count, insertion rank < count.
int removal_curve_keep(const int32_t* rank, const int32_t* counts, int K, int64_t q0, int nc, int B, int P, uint8_t* keep,
                       cudaStream_t st);
// removal_sample_keep: the keep table [nc*B, P] of replicates m0 .. m0+nc-1: player g of row (m, b) is removed iff word
// b*P + g at SITE_REMOVAL, key {rng[0], rng[1] + m}, is below `below` (= floor(p_remove 2^32)).
int removal_sample_keep(const uint64_t* rng, uint64_t below, int64_t m0, int nc, int B, int P, uint8_t* keep,
                        cudaStream_t st);
// removal_curve_summary: from curve_logits [2, K, B, ncls] and ends [2, B, ncls] (x', x): values [2, B, K] (F at the
// target), summaries [B, RD_REMOVAL_SUMMARIES] (fp64) and target_out [B] (target NULL: the argmax at x).
int removal_curve_summary(const float* curve_logits, const float* ends, const int64_t* target, const int32_t* counts,
                          int K, int B, int P, int ncls, float* values, double* summaries, int64_t* target_out,
                          cudaStream_t st);
// removal_moments: adds replicates (logits [nc*B, ncls], keep [nc*B, P]) into moments [B, RD_REMOVAL_MOMENTS] in
// replicate order (first: from 0, and target_out [B] written when not NULL); clean [B, ncls] are the logits at x.
int removal_moments(const float* logits, const float* clean, const int64_t* target, const float* attr,
                    const uint8_t* keep, int nc, int B, int P, int ncls, int first, double* moments, int64_t* target_out,
                    cudaStream_t st);

// ---- SWA / SWAG (rd_swag.cu; rd_swag_collect, rd_swag_sample, rd_raindrop_v2_swag_predictive) ----------------------
constexpr uint32_t SITE_SWAG = 102;         // Philox site of the SWAG weight draws (its key is {seed, step + replicate})
// swag_collect: with c snapshots folded in, mean = (c mean + theta) / (c + 1) and sq = (c sq + theta^2) / (c + 1) in
// fp64, and (rank > 0) slot c % rank of dev [rank, n] = fp32(theta - mean).  n % 4 == 0, 16-byte aligned buffers.
int swag_collect(const float* theta, int64_t n, int64_t c, int rank, double* mean, double* sq, float* dev, cudaStream_t st);
// swag_sample: out [n] = fp32(mean + sqrt(scale) (sqrt(max(sq - mean^2, 0)) z1 + [k >= 2] sum_{j<k} dev[j] z2_j /
// sqrt(k - 1))) in fp64, z drawn at key {rng[0], rng[1] + replicate}, element i for z1[i] and n + j for z2_j.
int swag_sample(const double* mean, const double* sq, const float* dev, int64_t n, int k, double scale,
                const uint64_t* rng, int64_t replicate, float* out, cudaStream_t st);
int swag_sample_check(const char* fn, const double* mean, const double* sq, const float* dev, int64_t n, int k,
                      double scale);

// ---- out-of-distribution detection (rd_ood.cu; rd_feature_moments, rd_raindrop_v2_ood_scores) ------------------------
// ood_moments: for feats f [n, F] and labels y [n], sums [C, F] (+)= the per-class sums and counts [C] (+)= the class
// sizes (sums NULL: both skipped), gram [F, F] (+)= f^T f (NULL: skipped), fp64, each entry one sample at a time in index
// order.  Labels outside [0, C) count nowhere.
int ood_moments(const float* f, const int64_t* y, int64_t n, int F, int C, int accumulate, double* sums, int64_t* counts,
                double* gram, cudaStream_t st);
// ood_rows: out [n, ld] from f [n, F] (row stride ldf): mu NULL: the L2-normalised rows (F.normalize, eps 1e-12); else
// fp32(f - mu).  Columns F .. ld-1 are 0.
int ood_rows(const float* f, int64_t ldf, int64_t n, int F, const double* mu, int ld, float* out, cudaStream_t st);
// ood_logit_scores: msp [n] = -max softmax, energy [n] = -T logsumexp(logits / T) (either may be NULL)
int ood_logit_scores(const float* logits, int n, int C, float temperature, float* msp, float* energy, cudaStream_t st);
// ood_class_dist: dist [n, C] = ||Z[r] - M[c]||^2 over rp columns (NULL: skipped), dmin [n] its minimum, cls [n] the
// first argmin (each may be NULL)
int ood_class_dist(const float* Z, const float* M, int n, int C, int rp, float* dist, float* dmin, int64_t* cls,
                   cudaStream_t st);
// ood_topk: merges sim [n, ncols] (row stride ld; column c is bank row col0 + c) into the running list run [n, ks] of
// the ks largest (3xTF32 similarity, index) keys (first: it starts empty); last: recomputes the ks candidates'
// similarities as fp64 dots of the query rows q [n, Fp] and the bank rows [., Fp], and writes the k largest of those,
// idx [n, k] in (similarity descending, index ascending) order and knn [n] = 2 - 2 s_(k) (either may be NULL), instead
// of run.  k <= ks <= RD_OOD_MAX_K + RD_OOD_SEL_EXTRA.
int ood_topk(const float* sim, int64_t ld, int n, int ncols, int64_t col0, int k, int ks, int first, int last,
             uint64_t* run,
             const float* q, const float* bank, int Fp, float* knn, int64_t* idx, cudaStream_t st);

int node_scale(const int64_t* edge_tgt, const float* edge_w, int E, int N, float* s, cudaStream_t st);

// The kernel classes of the LayerNorm launches (RD_LN_* in the public header): the forward's and the backward fused
// kernel's ITERS (1, 2, 5: D <= 128, 256, 640, D % 4 == 0, every pointer 16-byte aligned), else the generic forward,
// and the split backward with layernorm_bwd_dx_kernel's 128-bit or scalar path.
constexpr int LN_GENERIC = RD_LN_GENERIC, LN_SPLIT_VEC = RD_LN_SPLIT_VEC, LN_SPLIT_SCALAR = RD_LN_SPLIT_SCALAR;
int layernorm_fwd_class(const float* x, const float* gamma, const float* beta, const float* y, int D);
int layernorm_bwd_class(const float* x, const float* gamma, const float* dy, const float* dx, const float* dx_drop,
                        float drop_p, int D);
// y = LN(x) * gamma + beta over the last dim (width D); stats[row] = {mean, rstd}
int layernorm_fwd(const float* x, const float* gamma, const float* beta, int64_t rows, int D, float eps,
                  float* y, float* stats, cudaStream_t st);
// dx from dy; the dgamma / dbeta column sums as per-CTA partial rows scratch[chunks][2][D] (dgamma row, dbeta row),
// scratch >= ln_bwd_scratch_floats(rows, D).  Their reduction is the caller's (*chunks = chunks): it is folded into a
// later grouped reduction launch (tc_wgrad_group column sums).
int64_t ln_bwd_scratch_floats(int64_t rows, int D);
// dx_drop (written when drop_p > 0): dx with the dropout mask of `site` re-applied, i.e. the gradient w.r.t. the
// sub-layer output that was dropped before the residual add.  keep_bits (optional, [rows][keep_ld] words, bit j % 32 of
// word j / 32): the decisions the forward GEMM epilogue stored.  Only the fused kernel reads them; the split path draws
// Philox (site, index row * D + j) whether or not they are passed.  So stored bits must be exactly the Philox decisions
// of that site and index, as the tensor-core epilogue writes them: then both paths apply the same mask.
int layernorm_bwd(const float* x, const float* stats, const float* gamma, const float* dy, int64_t rows,
                  int D, float* dx, float* scratch, float* dx_drop, float drop_p, const uint64_t* rng, uint32_t site,
                  int* chunks, cudaStream_t st, const uint32_t* keep_bits = nullptr, int keep_ld = 0);

// in-place masked softmax over rows of S [B,H,T,T]; key j masked when j >= lengths[b].
// If Pd != nullptr also writes the dropped probabilities (training; rep.B > 0: of replicate-major rows, rep_remap).
int attn_softmax_fwd(float* S, const int64_t* lengths, int B, int H, int T, float drop_p,
                     const uint64_t* rng, uint32_t site, float* Pd, cudaStream_t st, DropRep rep = {});
// dS = P * (dP - sum_j dP_j P_j), dP = dPd * mask/(1-p); in place on dP
int attn_softmax_bwd(const float* P, float* dP, int B, int H, int T, float drop_p, const uint64_t* rng,
                     uint32_t site, cudaStream_t st);

// fused pooling + classification head (rd_head.cu).  x = encoder output [T, B, D]; writes feat [B, Df], hpre [B, Df],
// logits [B, ncls]; with labels y also the per-sample losses, d(loss)/d(logits) of the batch-mean CrossEntropy and
// the scalar loss (summed by the last CTA, ticket in *counter which must be 0 on entry).
int head_fwd(int B, int T, int D, int N, int ds, int ncls, const float* x, const int64_t* lengths, const float* statics,
             const float* emb_w, const float* emb_b, const float* w0, const float* b0, const float* w2, const float* b2,
             float* feat, float* hpre, float* logits, const int64_t* y, float* loss_ps, float* dlogits, float* loss,
             unsigned* counter, cudaStream_t st);
// dx = d(loss)/d(encoder output) [T, B, D] (masked-mean backward); g_w0 == nullptr skips the weight gradients
bool head_bwd_supported(int Df);
int head_bwd(int B, int T, int D, int N, int ds, int ncls, const int64_t* lengths, const float* statics, const float* w0,
             const float* w2, const float* feat, const float* hpre, const float* dlogits, float* dh, float* dfeat, float* dx,
             float* g_w0, float* g_b0, float* g_w2, float* g_b2, float* g_emb_w, float* g_emb_b, cudaStream_t st);

// fused attention for short sequences (rd_attn_small.cu): ctx from qkv in one launch, dqkv in one launch
bool attn_small_supported(int T, int hd);
// rep.B > 0 (forwards): attention dropout of replicate-major rows (rep_remap, rd_common.cuh)
int attn_small_fwd(const float* qkv, const int64_t* lengths, int B, int H, int T, int hd, float drop_p,
                   const uint64_t* rng, uint32_t site, float* ctx, cudaStream_t st, DropRep rep = {});
int attn_small_bwd(const float* qkv, const float* dctx, const int64_t* lengths, int B, int H, int T, int hd,
                   float drop_p, const uint64_t* rng, uint32_t site, float* dqkv, cudaStream_t st);

// the same on the tensor cores (rd_attn_tc.cu: mma.sync 3xTF32, T <= 64, hd <= 96, hd % 4 == 0)
bool attn_tc_supported(int T, int hd);
void attn_tc_set_debug(unsigned long long* buf);   // clock64 phase stamps per CTA: [CTA][16], slots 0-5 and 12 (debug)
int attn_tc_fwd(const float* qkv, const int64_t* lengths, int B, int H, int T, int hd, float drop_p,
                const uint64_t* rng, uint32_t site, float* ctx, cudaStream_t st, DropRep rep = {});
int attn_tc_bwd(const float* qkv, const float* dctx, const int64_t* lengths, int B, int H, int T, int hd,
                float drop_p, const uint64_t* rng, uint32_t site, float* dqkv, cudaStream_t st);

// dZ2[(b*N+n), t*d_ob+k] = dZ[t,b,n*d_ob+k] * s[n] * (Z[t,b,n*d_ob+k] > 0)
int obprop_out_grad(const float* dZ, const float* Z, const float* s, int B, int T, int N, int d_ob, int D,
                    int round, float* dZ2, cudaStream_t st);

// y[i] = x[i] * mask(site, i)   (re-generates the forward's dropout mask)
int apply_dropout(const float* x, int64_t n, float p, const uint64_t* rng, uint32_t site, float* y,
                  cudaStream_t st);

// d_pre = d_out * scale[r % mod] * (out > 0)
int relu_scale_bwd(const float* d_out, const float* out, const float* scale, int mod, int64_t rows, int C,
                   float* d_pre, cudaStream_t st);

int cross_entropy(const float* logits, const int64_t* y, int B, int ncls, float* loss, float* dlogits,
                  cudaStream_t st);
// step: int64[2] = {count, ticket}; the ticket word must be 0 on entry (it is reset by the launch).  The count is
// incremented by the last CTA of the launch, so one launch does tick + update.  lr_dev (optional, device) overrides lr.
int adam(float* p, const float* g, float* m, float* v, int64_t n, float lr, const float* lr_dev, float b1, float b2,
         float eps, float gscale, int64_t* step, cudaStream_t st);

// ---- differentially private training (rd_dp.cu) ---------------------------------------------------------------------
// Per-sample squared gradient norms of the linear layers.  Item = one (dY, X) operand pair of a weight gradient; sample
// b's rows are r = b*sstride + t*rstride, t < R (encoder: sstride 1, rstride B, R = T; ob-prop: sstride N, rstride 1,
// R = N).  Its weight and bias sums land in sqnorms[b*nf + fw] and [b*nf + fb].  ghost is the item's form (dp_ghost's
// choice in the backward), tm / tn / ntiles come from dp_norm_tiles for that form; blk0 = the item's first CTA in the
// group launch (items in order, B*ntiles CTAs each).
constexpr uint32_t SITE_DP_NOISE = 96;      // Philox site of the DP-SGD noise (its key is the noise key, not the dropout key)
constexpr int DP_MAX_ITEMS = 4 * RD_MAX_LAYERS;
constexpr int DP_MAX_FIELDS = 128;
struct DpNormItem {
  const float* Y; const float* X;
  long long ldy, ldx, sstride, rstride, blk0;
  int Nout, Kin, R, ghost, tm, tn, ntiles, fw, fb;
};
struct DpNormGroup { DpNormItem it[DP_MAX_ITEMS]; int n; };
// ghost iff R (Nout + Kin + 1) < Nout (Kin + 1): the form with fewer multiply-adds
bool dp_ghost(int R, int Nout, int Kin);
// tiles per sample of the given form (ghost: the R x R upper triangle, else the [Nout, Kin + 1] product); sets tm, tn
int dp_norm_tiles(int R, int Nout, int Kin, bool ghost, int* tm, int* tn);
// one launch over every item's tiles (partial: 2 doubles per CTA), one launch adding them into sqnorms
int dp_norm_group(const DpNormGroup& g, int B, double* partial, double* sqnorms, int nf, cudaStream_t st);
// LayerNorm gamma / beta of each sample (rows t*B + b, t < T) from its input x, stats {mean, rstd} and output gradient dy
int dp_ln_sqnorm(const float* x, const float* stats, const float* dy, int T, int B, int D, double* sqnorms, int nf, int fw,
                 int fb, cudaStream_t st);
// emb (ds > 0), mlp_static.0, mlp_static.2 weight and bias, in that order from field 0
int dp_head_sqnorm(int B, int D, int Df, int ds, int ncls, const float* dlogits, const float* hpre, const float* dh,
                   const float* feat, const float* dfeat, const float* statics, double* sqnorms, int nf, cudaStream_t st);
int dp_clip(const double* sqnorms, int B, int nf, int ncls, const float* weight, double max_norm, double L,
            const float* loss_ps, float* dlogits, float* clip, float* loss, cudaStream_t st);
// the used ranges [off, off + numel) of the flat bucket, ascending, off % 4 == 0
struct DpFields { long long off[DP_MAX_FIELDS]; long long numel[DP_MAX_FIELDS]; int n; };
int dp_noise(float* g, int64_t n, const DpFields& fields, float stdv, uint64_t* key, cudaStream_t st);

// ---- per-sample gradients, materialised (rd_dp.cu; TracIn influence) -------------------------------------------------
// Sample b's gradient row G[b, :] (ldg floats) in flat-bucket layout, every value scale * (its fp64 sum) rounded once.
// Item = one (dY, X) pair as in DpNormItem; the sample's [Nout, Kin + 1] product dY_b^T [X_b | 1] goes to the weight
// field at column gw (row-major [Nout, Kin]) and the bias field at gb.  tn = ceil((Kin + 1) / 64), ntiles = tn *
// ceil(Nout / 64), blk0 as in DpNormGroup.
struct PsgItem {
  const float* Y; const float* X;
  long long ldy, ldx, sstride, rstride, blk0, gw, gb;
  int Nout, Kin, R, tn, ntiles;
};
struct PsgGroup { PsgItem it[DP_MAX_ITEMS]; int n; };
int psg_tiles(int Nout, int Kin, int* tn);
// rotated (EK-FAC): X holds Kin + 1 columns of [X | 1] Q_A (ldx >= Kin + 1) and no ones column is appended
int psg_group(const PsgGroup& g, int B, float* G, long long ldg, float scale, cudaStream_t st, bool rotated = false);
// LayerNorm gamma -> G[b, gw + d], beta -> G[b, gb + d] (sums over the rows t*B + b, t < T)
int psg_ln(const float* x, const float* stats, const float* dy, int T, int B, int D, float* G, long long ldg, long long gw,
           long long gb, float scale, cudaStream_t st);
// the head's fields: off[0..5] = emb weight, bias (ds > 0), mlp_static.0 weight, bias, mlp_static.2 weight, bias
int psg_head(int B, int D, int Df, int ds, int ncls, const float* dlogits, const float* hpre, const float* dh, const float* feat,
             const float* dfeat, const float* statics, float* G, long long ldg, const long long* off, float scale,
             cudaStream_t st);
// EK-FAC factors (rd_ekfac.cu): A [(Kin + 1)^2] += [[Aw, Ab], [Ab^T, rows]], S [Nout^2] += sscale * Sw (fp64)
int kfac_accumulate(const float* Aw, const float* Ab, const float* Sw, int Kin, int Nout, long long rows, double sscale,
                    double* A, double* S, cudaStream_t st);
// zeroes G[b, off[f] + numel[f] .. next field's offset) and the tail up to ldg: the bucket's padding columns
int psg_pad(const DpFields& fields, int B, float* G, long long ldg, cudaStream_t st);

// ---- Laplace approximation (rd_laplace.cu) ---------------------------------------------------------------------------
// laplace_seed: d_logits [B, ncls] = e_c / B.  laplace_gram: cov [B, ncls, ncls] (fp64) = sum_j w_j G_c[b, j] G_c'[b, j]
// over the rows G [ncls][B][ldg] (class-major, ldg % 4 == 0, 16-byte aligned), through the fp64 slab partials
// `partial` [laplace_gram_partial_doubles(B, ncls, ldg)]; ncls <= RD_LAPLACE_MAX_CLASSES.
int64_t laplace_gram_partial_doubles(int B, int ncls, int64_t ldg);
int laplace_seed(float* d_logits, int B, int ncls, int c, cudaStream_t st);
int laplace_gram(const float* G, int B, int ncls, int64_t ldg, const float* w, double* partial, double* cov,
                 cudaStream_t st);

}  // namespace rd
