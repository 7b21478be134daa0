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
// kernel_shap_accumulate: adds sum_ci w[c] z[c, g] (F(c) - F(x')) over the chunk's coalitions c = c0 .. c0+nc-1 (F at
// target[b], nullptr: argmax of ends[1]) into the fp64 sums acc [B, P]; first: start from 0.
int kernel_shap_accumulate(const float* logits_c, const float* ends, const int64_t* target, const uint8_t* z,
                           const double* w, int P, int c0, int nc, int B, int ncls, double* acc, int first, cudaStream_t st);
// kernel_shap_solve: attr [B, P] = acc [B, P] . K^T + (F(x) - F(x')) k^T in fp64, solve = [K | k] [P, P+1]; P <= 4096.
int kernel_shap_solve(const double* acc, const double* solve, const float* ends, const int64_t* target, int P, int B,
                      int ncls, float* attr, cudaStream_t st);

// Monte Carlo dropout over chunks of nc replicates on B*nc rows, replicate-major (j = m*B + b).
// mc_expand: src_e [T, B*nc, 2N], statics_e (ds > 0), times_e, lengths_e = nc copies of the batch.
int mc_expand(const float* src, const float* statics, const float* times, const int64_t* lengths, int B, int nc, int T,
              int N, int ds, float* src_e, float* statics_e, float* times_e, int64_t* lengths_e, cudaStream_t st);
// mc_accumulate: adds replicates m0 .. m0+nc-1 (logits [B*nc, ncls]) to the fp64 sums acc [B, 2*ncls + 1] in replicate
// order (first: from 0); samples (optional) [M, B, ncls] gets their logits; last: mean [B, ncls], var [B, ncls] and
// ent [3, B] = (predictive entropy, expected entropy, mutual information) over all M replicates.
int mc_accumulate(const float* logits, int nc, int B, int ncls, int64_t m0, int64_t M, double* acc, float* samples,
                  float* mean, float* var, float* ent, int first, int last, cudaStream_t st);

int node_scale(const int64_t* edge_tgt, const float* edge_w, int E, int N, float* s, cudaStream_t st);

// y = LN(x) * gamma + beta over the last dim (width D); stats[row] = {mean, rstd}
int layernorm_fwd(const float* x, const float* gamma, const float* beta, int64_t rows, int D, float eps,
                  float* y, float* stats, cudaStream_t st);
// dx from dy; dgamma/dbeta via partials. scratch >= ln_bwd_scratch_floats(rows, D)
int64_t ln_bwd_scratch_floats(int64_t rows, int D);
// dx_drop (optional, used when drop_p > 0): dx with the dropout mask of `site` re-applied, i.e. the
// gradient w.r.t. the sub-layer output that was dropped before the residual add
// deferred_chunks != nullptr: the reduction of the per-CTA partial rows scratch[chunks][2][D] is left to the caller
// (*deferred_chunks = chunks), who folds it into a later grouped reduction launch (tc_wgrad_group)
int layernorm_bwd(const float* x, const float* stats, const float* gamma, const float* dy, int64_t rows,
                  int D, float* dx, float* dgamma, float* dbeta, float* scratch, float* dx_drop, float drop_p,
                  const uint64_t* rng, uint32_t site, int* deferred_chunks, cudaStream_t st,
                  const uint32_t* keep_bits = nullptr, int keep_ld = 0);   // keep_bits: decisions stored by the forward (else Philox)

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
void attn_tc_set_debug(unsigned long long* buf);   // start / end clock64 stamps per CTA: [CTA][16], slots 0 and 12 (debug)
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
// R = N).  Its weight and bias sums land in sqnorms[b*nf + fw] and [b*nf + fb].  ghost / tm / tn / ntiles come from
// dp_norm_tiles; blk0 = the item's first CTA in the group launch (items in order, B*ntiles CTAs each).
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
int dp_norm_tiles(int R, int Nout, int Kin, int* tm, int* tn);     // tiles per sample; sets tm, tn
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

}  // namespace rd
