/*
 * raindrop_b200.h -- C ABI of librd_b200.so (sm_90a, H100), the device side of the Raindrop hot path.
 *
 * The reference (mims-harvard/Raindrop) is pure Python; it has no FFI of its own.  The boundary
 * a maintainer binds is therefore the set of Python call sites listed beside each entry point
 * (paths relative to the reference tree).  Our `raindrop_b200/models_rd.py` binds them through
 * ctypes; INTEGRATION.md shows the same stubs applied to the reference's own files.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host; all tensors are dense,
 *     row-major fp32 (indices int64) exactly as the reference's torch tensors are laid out;
 *   - `stream` is a cudaStream_t passed as void*; every call is stream-ordered, allocation-free
 *     and sync-free (CUDA-graph capturable).  Scratch memory is provided by the caller: query
 *     the size first;
 *   - return value 0 = ok, negative = error (rd_last_error_string() describes it); nothing
 *     throws across the ABI.
 */
#ifndef RAINDROP_B200_H
#define RAINDROP_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RD_ABI_VERSION 2
#define RD_MAX_LAYERS 8
#define RD_D_PE 16 /* d_pe, code/models_rd.py:215 */

/* Shapes of one Raindrop_v2 instance + one batch (code/models_rd.py:208-264, 278-284). */
typedef struct rd_dims {
  int32_t B;         /* samples in this batch (any >= 1)                                  */
  int32_t T;         /* max_len                                                           */
  int32_t N;         /* d_inp = sensors                                                   */
  int32_t d_ob;      /* d_model / d_inp (4 in code/Raindrop.py:125)                       */
  int32_t nhead;     /* temporal attention heads                                          */
  int32_t nhid;      /* feed-forward width                                                */
  int32_t nlayers;   /* encoder layers (<= RD_MAX_LAYERS)                                 */
  int32_t d_static;  /* 0 = no static branch (static=False)                               */
  int32_t n_classes;
  int32_t training;  /* 1: dropout active (model.train()), 0: eval                        */
  float dropout_p;   /* one p for every dropout site, as in the reference                 */
  float ln_eps;      /* 1e-5                                                              */
  float pe_timescales[RD_D_PE / 2]; /* max_len ** linspace(0,1,8) computed in fp64 on host,
                                       cast to fp32 (code/models_rd.py:31,34)             */
  int32_t d_pe;        /* width of the positional encoding concatenated to the encoder input; 0 = 16 (Raindrop_v2,
                          code/models_rd.py:215).  Legacy Raindrop v1 uses 36 (code/models_rd.py:68); only the
                          rd_encoder_head_* entry points accept values other than 16                              */
  int32_t emb_dim;     /* width of emb = Linear(d_static, emb_dim): 0 = N (Raindrop_v2, code/models_rd.py:224);
                          d_model for legacy Raindrop v1 (code/models_rd.py:98)                                    */
  int32_t obprop_mode; /* arithmetic of the two observation-propagation GEMMs on the tensor cores:
                          0 = automatic: error-compensated 3xTF32 (fp32-level, gradients match the fp32 reference
                              to ~1e-3) while 2*B*N*C^2 <= 2 GFLOP per layer, i.e. where the layer is launch-latency
                              bound anyway; single-pass TF32 (operands rounded to TF32, forward error ~3e-4) above,
                              where it is what reaches the HBM / tensor roofline
                          1 = always single-pass TF32        2 = always 3xTF32                          */
} rd_dims;

/* Parameters that take part in the live path (SURVEY.md 8a18).  Names = state-dict keys. */
typedef struct rd_encoder_layer_params {
  const float* in_proj_weight;  /* [3D, D] */
  const float* in_proj_bias;    /* [3D]    */
  const float* out_proj_weight; /* [D, D]  */
  const float* out_proj_bias;   /* [D]     */
  const float* linear1_weight;  /* [nhid, D] */
  const float* linear1_bias;    /* [nhid]  */
  const float* linear2_weight;  /* [D, nhid] */
  const float* linear2_bias;    /* [D]     */
  const float* norm1_weight;    /* [D] */
  const float* norm1_bias;
  const float* norm2_weight;
  const float* norm2_bias;
} rd_encoder_layer_params;

typedef struct rd_params {
  const float* R_u;             /* [1, N*d_ob]  plain tensor, code/models_rd.py:241          */
  const float* emb_weight;      /* [N, d_static] or NULL                                     */
  const float* emb_bias;        /* [N] or NULL                                               */
  const float* ob1_value_weight;/* ob_propagation.lin_value.weight        [C, C], C=T*d_ob   */
  const float* ob1_value_bias;  /* [C] */
  const float* ob2_value_weight;/* ob_propagation_layer2.lin_value.weight [C, C]             */
  const float* ob2_value_bias;
  const float* mlp0_weight;     /* mlp_static.0.weight [Df, Df], Df = D + (static ? N : 0)   */
  const float* mlp0_bias;
  const float* mlp2_weight;     /* mlp_static.2.weight [n_classes, Df]                       */
  const float* mlp2_bias;
  rd_encoder_layer_params layer[RD_MAX_LAYERS];
} rd_params;

/* Same members, writable: gradients (written, not accumulated).  R_u gets no gradient. */
typedef struct rd_encoder_layer_grads {
  float* in_proj_weight; float* in_proj_bias; float* out_proj_weight; float* out_proj_bias;
  float* linear1_weight; float* linear1_bias; float* linear2_weight; float* linear2_bias;
  float* norm1_weight; float* norm1_bias; float* norm2_weight; float* norm2_bias;
} rd_encoder_layer_grads;

typedef struct rd_grads {
  float* emb_weight; float* emb_bias;
  float* ob1_value_weight; float* ob1_value_bias;
  float* ob2_value_weight; float* ob2_value_bias;
  float* mlp0_weight; float* mlp0_bias; float* mlp2_weight; float* mlp2_bias;
  rd_encoder_layer_grads layer[RD_MAX_LAYERS];
} rd_grads;

/* Named views into the activation workspace written by rd_raindrop_v2_fwd (for parity tests). */
enum rd_ws_buffer {
  RD_WS_X0 = 0,    /* lifted input   [B*N, C]  (code/models_rd.py:290-296,326-327)          */
  RD_WS_H1 = 1,    /* layer-1 output [B*N, C]  (code/models_rd.py:329-330)                  */
  RD_WS_ENC_IN = 2,/* cat(obs, pe)   [T, B, D] (code/models_rd.py:341,354)                  */
  RD_WS_ENC_OUT = 3,/* r_out         [T, B, D] (code/models_rd.py:358)                      */
  RD_WS_FEAT = 4,  /* cat(pooled, emb) [B, Df] (code/models_rd.py:379,384)                  */
  RD_WS_RNG = 5,   /* 2 x uint64 (seed, step counter) captured by this forward              */
  RD_WS_HEAD_HIDDEN = 6,/* relu(mlp_static.0(feat)) [B, Df] (code/models_rd.py:385)         */
  RD_WS_FFN = 7    /* RD_WS_FFN + l, l < nlayers: dropout(relu(linear1)) of encoder layer l
                      [T*B, nhid], token-major rows t*B + b                                 */
};

int rd_abi_version(void);
const char* rd_last_error_string(void);
/* number of kernels this library has launched so far in this process (host-side counter; a
 * CUDA-graph replay re-runs captured launches without passing through here) */
uint64_t rd_launch_count(void);

/* ---- graph prologue --------------------------------------------------------------------
 * s[n] = sum_{e: tgt[e]==n} softmax_{e->n}(w)   with PyG's  exp(w-max)/(sum+1e-16).
 * Replaces `softmax(gamma, index)` + `scatter(..., reduce='add')` of
 * code/Ob_propagation.py:195,226-228 for the live path where the message depends on the
 * target only (code/Ob_propagation.py:200).  edge_tgt = edge_index[1] (code/models_rd.py:310). */
int rd_node_scale(const int64_t* edge_tgt, const float* edge_w, int32_t E, int32_t N,
                  float* node_scale, void* stream);

/* ---- one observation-propagation layer (operator level) -----------------------------------
 * out[r, :] = relu(x[r, :] . W^T + b) * node_scale[r % scale_mod]      x, out: [rows, C]
 * Replaces Observation_progation.forward with use_beta=False (code/Ob_propagation.py:94-132,
 * 157-160,187-211,213-228) for `rows / N` samples at once (code/models_rd.py:322-336).
 * The tensor cores take TF32 operands: x and weight are first rounded (RN) into `scratch`
 * (rd_obprop_fwd_scratch_bytes(rows, C) bytes); accumulation is fp32.  scratch == NULL promises that
 * x and weight are already TF32-representable (low 13 mantissa bits zero): no rounding pass. */
size_t rd_obprop_fwd_scratch_bytes(int64_t rows, int32_t C);
int rd_obprop_fwd(const float* x, const float* weight, const float* bias, const float* node_scale,
                  int32_t scale_mod, int64_t rows, int32_t C, float* out, void* scratch, void* stream);

/* Backward of the above.  d_out, out: [rows, C].  Writes d_x (may be NULL), d_weight, d_bias.
 * scratch: rd_obprop_bwd_scratch_bytes(rows, C) bytes. */
size_t rd_obprop_bwd_scratch_bytes(int64_t rows, int32_t C);
int rd_obprop_bwd(const float* x, const float* out, const float* d_out, const float* weight,
                  const float* node_scale, int32_t scale_mod, int64_t rows, int32_t C,
                  float* d_x, float* d_weight, float* d_bias, void* scratch, void* stream);

/* Observation_progation.forward with use_beta=True (code/Ob_propagation.py:161-186,191,195-228; dormant in
 * Raindrop_v2, code/models_rd.py:317, but part of the operator's API).  One sample: x [N, C=T*d_ob],
 * p_t [T, 16].  Keeps the K = E/2 edges with the highest mean gamma (in that order), regroups them by
 * SOURCE for the per-channel segment softmax and scatters to the source (as the reference does).
 * Outputs: out [N, C]; pruned edge list edge_src_out/edge_tgt_out [K]; alpha_out [K].  Needs E >= 2 (K >= 1): the
 * forward, the backward and both scratch-size queries (which return 0) refuse fewer. */
size_t rd_obprop_beta_scratch_bytes(int32_t N, int32_t T, int32_t d_ob, int32_t E);
int rd_obprop_beta_fwd(const float* x, const float* p_t, const int64_t* edge_src, const int64_t* edge_tgt,
                       const float* edge_w, int32_t E, int32_t N, int32_t T, int32_t d_ob,
                       const float* increase_dim_w, const float* increase_dim_b, const float* map_weights,
                       const float* value_w, const float* value_b, float* out, int64_t* edge_src_out,
                       int64_t* edge_tgt_out, float* alpha_out, void* scratch, void* stream);

/* Backward of rd_obprop_beta_fwd (same inputs; the forward is recomputed; the top-K edge selection is piecewise
 * constant and carries no gradient).  d_out [N, C]; d_alpha [K] or NULL = gradient w.r.t. the returned alpha (mean
 * gamma of the kept edges, which becomes layer 2's edge weights in code/models_rd.py:332-336).  Writes d_x [N, C]
 * (may be NULL), d_edge_w [E], d_p_t [T, 16] (may be NULL), d_increase_dim_{w [8C, C], b [8C]}, d_map_weights [N, 16],
 * d_value_{w [C, C], b [C]} -- the tensors autograd reaches through code/Ob_propagation.py:161-211.
 * scratch: rd_obprop_beta_bwd_scratch_bytes(N, T, d_ob, E) bytes. */
size_t rd_obprop_beta_bwd_scratch_bytes(int32_t N, int32_t T, int32_t d_ob, int32_t E);
int rd_obprop_beta_bwd(const float* x, const float* p_t, const int64_t* edge_src, const int64_t* edge_tgt,
                       const float* edge_w, int32_t E, int32_t N, int32_t T, int32_t d_ob,
                       const float* increase_dim_w, const float* increase_dim_b, const float* map_weights,
                       const float* value_w, const float* value_b, const float* d_out, const float* d_alpha,
                       float* d_x, float* d_edge_w, float* d_p_t, float* d_increase_dim_w, float* d_increase_dim_b,
                       float* d_map_weights, float* d_value_w, float* d_value_b, void* scratch, void* stream);

/* ---- whole Raindrop_v2 forward / backward ---------------------------------------------------
 * Replaces Raindrop_v2.forward (code/models_rd.py:278-387) for the live configuration
 * (sensor_wise_mask=False, aggreg='mean', use_beta=False) and its autograd backward
 * (code/Raindrop.py:323).
 *   src     [T, B, 2N]   times [T, B]   lengths [B] int64   statics [B, d_static] or NULL
 *   node_scale [N]       from rd_node_scale on the model's graph
 *   rng_state  2 x uint64 on the device: {seed, counter}; the forward copies it into the
 *              workspace and increments the counter (only when training && dropout_p > 0)
 *   workspace  rd_workspace_bytes(dims) bytes, kept by the caller until backward is done
 *   logits  [B, n_classes]
 *   y       optional int64 labels [B]: when given, the head kernel also evaluates
 *           torch.nn.CrossEntropyLoss (mean) -- code/Raindrop.py:322 -- writing the scalar `loss` and
 *           `d_logits` [B, n_classes] = d(loss)/d(logits), ready for rd_raindrop_v2_bwd.  NULL: plain forward
 *           (loss / d_logits ignored).                                                            */
size_t rd_workspace_bytes(const rd_dims* dims);
size_t rd_backward_scratch_bytes(const rd_dims* dims);
/* offset (bytes) and element count of a named buffer inside the workspace; -1 if unknown */
int64_t rd_workspace_offset(const rd_dims* dims, int32_t which, int64_t* n_floats);

int rd_raindrop_v2_fwd(const rd_dims* dims, const rd_params* params, const float* src,
                       const float* statics, const float* times, const int64_t* lengths,
                       const float* node_scale, uint64_t* rng_state, void* workspace,
                       float* logits, const int64_t* y, float* loss, float* d_logits, void* stream);

/* Backward (autograd of the above, code/Raindrop.py:323).  `phases` selects what one call does so that a
 * data-parallel caller can start reducing the first gradient bucket while the rest is still being computed
 * (SURVEY.md 8e):
 *   RD_BWD_ENCODER  head + temporal-attention encoder: every gradient except the two lin_value pairs is final
 *                   when the call's work completes; d(loss)/d(encoder input) stays in `scratch`
 *   RD_BWD_OBPROP   observation propagation: ob1/ob2 lin_value gradients (needs the same scratch, after ENCODER)
 *   both (3)        whole backward, weight gradients in one grouped tensor-core launch
 * grads == NULL (frozen parameters, e.g. attribution with model.requires_grad_(False)): only the data-gradient chain
 * runs -- no weight-gradient GEMMs, column sums or head outer products -- and `scratch` is left holding the same
 * activation gradients, ready for rd_raindrop_v2_input_grad.                                               */
#define RD_BWD_ENCODER 1
#define RD_BWD_OBPROP 2
#define RD_BWD_ALL 3
int rd_raindrop_v2_bwd(const rd_dims* dims, const rd_params* params, const float* statics,
                       const int64_t* lengths, const float* node_scale, const void* workspace,
                       const float* d_logits, const rd_grads* grads, void* scratch, int32_t phases,
                       void* stream);

/* ---- temporal encoder + pooling + head on a caller-provided encoder input ------------------------------------
 * The second half of Raindrop_v2.forward (code/models_rd.py:354-385) and all of legacy Raindrop v1 after its
 * per-sample TransformerConv (code/models_rd.py:168-191): nn.TransformerEncoder with key-padding mask, masked mean
 * (divisor lengths + 1), concat emb(static), mlp_static.  The caller writes the encoder input cat(features, pe)
 * [T, B, D = N*d_ob + d_pe] into the workspace buffer RD_WS_ENC_IN first (rd_workspace_offset), then calls _fwd;
 * _bwd fills every encoder / emb / mlp_static gradient of `grads` (the ob-prop members are ignored) and writes
 * d(loss)/d(encoder input) to d_enc_in [T, B, D].  Same workspace / scratch sizes and rng protocol as
 * rd_raindrop_v2_fwd / _bwd; grads may be NULL as there.  As there, a training forward with Df = D + emb_dim > 722 (the
 * head backward's limit) is refused before it writes anything or advances the rng counter. */
int rd_encoder_head_fwd(const rd_dims* dims, const rd_params* params, const float* statics, const int64_t* lengths,
                        uint64_t* rng_state, void* workspace, float* logits, const int64_t* y, float* loss,
                        float* d_logits, void* stream);
int rd_encoder_head_bwd(const rd_dims* dims, const rd_params* params, const float* statics, const int64_t* lengths,
                        const void* workspace, const float* d_logits, const rd_grads* grads, void* scratch,
                        float* d_enc_in, void* stream);
/* ---- gradients with respect to the inputs src, static and times ----------------------------------------------
 * For saliency maps, integrated gradients and other attribution methods, and for adversarial examples (the batched
 * attack is rd_raindrop_v2_pgd).  Call it
 * after rd_raindrop_v2_bwd (phases including RD_BWD_OBPROP) or rd_encoder_head_bwd, on the same stream, with the
 * same dims / params, the forward's workspace and the backward's scratch `bwd_scratch` untouched in between: the
 * backward leaves d(loss)/d(encoder input), d(loss)/d(layer-1 pre-activation) and d(loss)/d(cat(pooled, emb)) there,
 * and this call finishes the chain through the first ob-prop layer, the lift (code/models_rd.py:285-296,323-327),
 * the positional encoding (:28-37) and emb = Linear(d_static, N) (:293-294).  Outputs (written, not accumulated;
 * each may be NULL, which skips its part):
 *   d_src     [T, B, 2N]  value half d(loss)/d(src[..., :N]); the mask half is unused on the live path and written
 *                         as 0; 0 wherever the value is 0 (relu'(0) = 0).  Train mode replays the forward's lift
 *                         dropout mask.  Needs `scratch` (rd_input_grad_scratch_bytes(dims) bytes) and `src`.
 *   d_times   [T, B]      0 on padded rows t >= lengths[b] (lengths may be NULL: no forced zeros).
 *   d_statics [B, d_static]
 * d_src and d_times need the Raindrop_v2 workspace; after rd_encoder_head_bwd only d_statics is available (the
 * encoder input gradient went to the caller's d_enc_in).  `scratch` may be NULL when d_src is NULL. */
size_t rd_input_grad_scratch_bytes(const rd_dims* dims);
int rd_raindrop_v2_input_grad(const rd_dims* dims, const rd_params* params, const float* src, const float* times,
                              const int64_t* lengths, const void* workspace, const void* bwd_scratch, void* scratch,
                              float* d_src, float* d_times, float* d_statics, void* stream);

/* ---- integrated gradients (IG) attribution of Raindrop_v2, in one call ------------------------------------------
 * For F = logits[b, target[b]] and the straight path x' + alpha (x - x') from the baseline x' to the input x:
 *   attr_src[t,b,n]     = (x - x')[t,b,n] . sum_k weights[k] dF/dsrc[t,b,n] at alpha = alphas[k]     (value half)
 *   attr_statics[b,j]   = (s - s')[b,j]   . sum_k weights[k] dF/dstatic[b,j] at alphas[k]
 * alphas / weights [n_steps] are the quadrature nodes and weights on [0, 1] (device fp32; any rule).  Only the value
 * half of src and the statics are interpolated: the mask half is taken from src, times and lengths are held fixed
 * (attribution over times is not provided; use rd_raindrop_v2_input_grad).  Eval arithmetic: dims->training must be 0,
 * no dropout, the rng state is neither read nor advanced and no parameter gradient is written.
 *   baseline_src     [T, B, 2N] (only the value half is read);  baseline_statics [B, d_static] or NULL when d_static == 0
 *   target           [B] int64 class per sample, or NULL = argmax of the logits at x (read on the device)
 *   attr_src         [T, B, 2N], the mask half written as 0;  attr_statics [B, d_static] or NULL (skipped)
 *   endpoint_logits  [2, B, n_classes]: logits at the baseline ([0]) and at the input ([1]), for the completeness check
 *                    sum(attr) ~ F(x) - F(x')
 * Work: one forward on 2B rows for the endpoints, then chunks of `steps_per_chunk` steps on B*steps_per_chunk rows
 * (step-major) -- inputs expanded in one launch, forward, frozen-parameter backward, dX0 GEMM, and one accumulation
 * launch that adds the chunk's weighted lift / static-embedding backward to running sums in fp32, in a fixed order
 * (deterministic, no atomics).  dims->obprop_mode 0 is resolved once from B*steps_per_chunk rows, so the endpoint
 * forward and every chunk, including a shorter last one, use the same arithmetic.
 * scratch: rd_integrated_gradients_scratch_bytes(dims, steps_per_chunk) bytes (dims->B = samples, training = 0). */
size_t rd_integrated_gradients_scratch_bytes(const rd_dims* dims, int32_t steps_per_chunk);
int rd_raindrop_v2_integrated_gradients(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                        const float* times, const int64_t* lengths, const float* node_scale,
                                        const float* baseline_src, const float* baseline_statics, const int64_t* target,
                                        const float* alphas, const float* weights, int32_t n_steps, int32_t steps_per_chunk,
                                        void* scratch, float* attr_src, float* attr_statics, float* endpoint_logits,
                                        void* stream);

/* ---- coalition attribution of Raindrop_v2: Shapley-value sampling and leave-one-out ablation, in one call ---------
 * Players: sensor groups 0..G-1 (sensor_player [N], device int32, values in [0, G), every group non-empty) and, when
 * d_static > 0, the static vector as player G; n_players = P = G + (d_static > 0).  Removing a player replaces the value
 * columns src[:, b, n] of its sensors by baseline_src[:, b, n] (the static player: statics[b] by baseline_statics[b]);
 * the mask half, times and lengths are never changed.  F(S) = logits[b, target[b]] of the eval-mode model on the input
 * whose players outside S are removed; x = all players kept, x' = all removed (with the cell entry point below, the cells
 * of no player keep x in x' too).
 *   RD_ATTR_SHAPLEY   attr[b, g] = (1/m) sum_p [F(S_pg + g) - F(S_pg)], S_pg = the players ahead of g in orders[p, :]
 *                     (orders [m, P] device int32, each row a permutation of 0..P-1, shared by the batch); sum_g attr[b, g]
 *                     = F(x) - F(x') up to rounding
 *   RD_ATTR_ABLATION  attr[b, g] = F(x) - F(x without player g)   (orders may be NULL, m is ignored)
 * Eval arithmetic: dims->training must be 0, the rng state is neither read nor advanced, no gradient is computed.
 *   baseline_src     [T, B, 2N] (only the value half is read);  baseline_statics [B, d_static] or NULL when d_static == 0
 *   target           [B] int64 class per sample, or NULL = argmax of the logits at x (read on the device)
 *   attr             [B, P] fp32
 *   endpoint_logits  [2, B, n_classes]: logits at x' ([0]) and at x ([1])
 * Work: one forward on 2B rows for the endpoints, then the coalitions -- m*(P-1) for Shapley (the first k = 1..P-1
 * players of each permutation; k = 0 and k = P are the endpoints), P for ablation (all but g) -- in chunks of
 * `coalitions_per_chunk` coalitions on B*coalitions_per_chunk rows (coalition-major): the inputs expanded in one launch,
 * the eval forward, and one launch that adds each coalition's F into fp64 running sums per (b, player) in a fixed order
 * (deterministic, no atomics, independent of the chunking; a player whose removal changes no input bit gets exactly 0).
 * dims->obprop_mode 0 is resolved once from B*coalitions_per_chunk rows, so the endpoint forward and every chunk use the
 * same arithmetic.  scratch: rd_coalition_attribution_scratch_bytes(dims, n_players, coalitions_per_chunk) bytes
 * (dims->B = samples, training = 0). */
#define RD_ATTR_SHAPLEY 0
#define RD_ATTR_ABLATION 1
size_t rd_coalition_attribution_scratch_bytes(const rd_dims* dims, int32_t n_players, int32_t coalitions_per_chunk);
int rd_raindrop_v2_coalition_attribution(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                         const float* times, const int64_t* lengths, const float* node_scale,
                                         const float* baseline_src, const float* baseline_statics, const int64_t* target,
                                         const int32_t* sensor_player, int32_t n_players, const int32_t* orders, int32_t m,
                                         int32_t method, int32_t coalitions_per_chunk, void* scratch, float* attr,
                                         float* endpoint_logits, void* stream);

/* ---- coalition attribution of Raindrop_v2 over value cells: (sensor, time window) players and any other map ---------
 * As rd_raindrop_v2_coalition_attribution, with a player per value cell instead of per sensor: cell (t, b, n) of the
 * value half belongs to player cell_player[t*player_stride_t + b*player_stride_b + n] (device int32).  Ids 0..G-1 are
 * players of the value cells, G = n_players - (d_static > 0), and when d_static > 0 the static vector is player G.  Any
 * other id (negative, or >= G) belongs to no player: that cell always keeps x.  A player with no cell in sample b gets
 * exactly 0 there; G may exceed N.  Strides select the map's layout (both >= 0):
 *   (0, 0)     per sensor [N]  (rd_raindrop_v2_coalition_attribution's sensor_player)
 *   (N, 0)     shared by the batch [T, N]
 *   (B*N, N)   per sample [T, B, N]
 * Removing a player writes the baseline into its cells of the value half; the mask half, times and lengths never
 * change.  Methods, formulas, fp64 sums, chunking, endpoint_logits and scratch (rd_coalition_attribution_scratch_bytes
 * with the same n_players) are those of rd_raindrop_v2_coalition_attribution; both entry points run the same code.  The
 * kept-player test of a cell costs O(1) whatever P: for Shapley one launch per chunk fills the chunk's keep table
 * [cc, P] (in scratch) before the expansion reads it; ablation and the endpoints need no table. */
int rd_raindrop_v2_cell_coalition_attribution(const rd_dims* dims, const rd_params* params, const float* src,
                                              const float* statics, const float* times, const int64_t* lengths,
                                              const float* node_scale, const float* baseline_src,
                                              const float* baseline_statics, const int64_t* target,
                                              const int32_t* cell_player, int64_t player_stride_t, int64_t player_stride_b,
                                              int32_t n_players, const int32_t* orders, int32_t m, int32_t method,
                                              int32_t coalitions_per_chunk, void* scratch, float* attr,
                                              float* endpoint_logits, void* stream);

/* ---- KernelSHAP of Raindrop_v2 over value-cell players, in one call -------------------------------------------------
 * Players, removal, cell_player and its strides ((0, 0): one player per sensor), target, baselines, endpoint_logits and
 * eval arithmetic as for rd_raindrop_v2_cell_coalition_attribution.  With v_b(S) = F(S) of sample b and the caller's
 * coalitions z_j (coalitions [M, P] device uint8, nonzero = player kept) and weights w_j (weights [M] device fp64),
 *   r_b[g]     = sum_j w_j z_j[g] (v_b(z_j) - v_b(empty))                          (fp64, per sample)
 *   attr[b, g] = sum_h K[g, h] r_b[h] + k[g] (v_b(all) - v_b(empty))               (fp64, rounded to fp32)
 * where solve = [K | k] [P, P+1] (device fp64, row-major) is the first P rows of pinv([[A, 1], [1^T, 0]]),
 * A = sum_j w_j z_j z_j^T: the efficiency-constrained weighted least-squares fit of the coalition values.  The operator
 * depends on the coalitions only and is computed by the caller (raindrop_b200.attribution computes it with numpy);
 * with all 2^P - 2 proper non-empty coalitions and the Shapley-kernel weights the result is the exact Shapley values.
 * 1 <= n_players <= RD_KERNEL_SHAP_MAX_PLAYERS; n_coalitions = M >= 0 (M = 0: attr = k (v(all) - v(empty))).
 * Work: the endpoint forward on 2B rows, then the M coalitions in chunks of coalitions_per_chunk on B*coalitions_per_chunk
 * rows (coalition-major): the inputs expanded in one launch that reads the chunk's rows of `coalitions` as its keep
 * table, the eval forward, and one launch that adds the chunk into fp64 sums r [B, P] in coalition order (deterministic,
 * no atomics, independent of the chunking); finally one launch of one CTA per sample applies [K | k].  dims->obprop_mode
 * 0 is resolved once from B*coalitions_per_chunk rows.  scratch: rd_coalition_attribution_scratch_bytes(dims, n_players,
 * coalitions_per_chunk) bytes.  Stream-ordered, allocation- and sync-free, CUDA-graph capturable. */
#define RD_KERNEL_SHAP_MAX_PLAYERS 4096
int rd_raindrop_v2_kernel_shap(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                               const float* times, const int64_t* lengths, const float* node_scale, const float* baseline_src,
                               const float* baseline_statics, const int64_t* target, const int32_t* cell_player,
                               int64_t player_stride_t, int64_t player_stride_b, int32_t n_players, const uint8_t* coalitions,
                               const double* weights, int32_t n_coalitions, const double* solve, int32_t coalitions_per_chunk,
                               void* scratch, float* attr, float* endpoint_logits, void* stream);

/* ---- faithfulness of attributions by removal: deletion / insertion curves and infidelity, in one call each ----------
 * Players, removal, cell_player and its strides ((0, 0): one player per sensor), target, baselines and eval arithmetic
 * as for rd_raindrop_v2_kernel_shap; n_players = P = G + (d_static > 0), 1 <= P <= RD_REMOVAL_MAX_PLAYERS.
 * attributions [B, P] (device fp32) are the scores phi under test, the static player last.  F = logits[b, target[b]].
 *
 * rd_raindrop_v2_removal_curves: rank [B, P] (int32) = the position of player g when sample b's players are sorted by
 * `order` (RD_REMOVAL_DESCENDING: phi high to low; _ASCENDING: low to high; _ABSOLUTE: |phi| high to low), ties to the
 * lower index, -0 as +0, NaN after every number.  counts [K] (device int32, strictly increasing in [0, P]; not checked
 * on the device) are the removal counts.  Deletion point (k, b) removes the players with rank < counts[k]; insertion
 * point (k, b) removes all others.  Outputs:
 *   curve_logits     [2, K, B, n_classes]: deletion ([0]) and insertion ([1]) logits
 *   endpoint_logits  [2, B, n_classes]: logits at x' ([0]) and at x ([1])
 *   values           [2, B, K]: F of the curve points;  target_out [B] int64: the class F reads
 *   summaries        [B, RD_REMOVAL_SUMMARIES] fp64: deletion AUC, insertion AUC, AOPC of the logit F, then the same of
 *                    softmax(logits)[target] (fp64 softmax of the fp32 logits).  AUC: trapezoid rule over
 *                    x_k = counts[k] / P;  AOPC = (1/K) sum_k (F(x) - deletion F at k).
 * Work: the endpoint forward on 2B rows, one rank launch (one CTA per sample, the keys sorted in shared memory), then
 * the 2K (curve, count) pairs in chunks of pairs_per_chunk on B*pairs_per_chunk rows (pair-major): one launch writes
 * the chunk's per-row keep table [nc*B, P] into scratch, one expands the rows, and one eval forward writes its logits
 * straight into curve_logits; finally one summary launch.  scratch: rd_removal_curves_scratch_bytes(dims, n_players,
 * pairs_per_chunk) bytes.
 *
 * rd_raindrop_v2_removal_infidelity: replicate m = 0 .. n_samples-1 removes from sample b the set S_mb of players g
 * whose Philox word b*P + g (word idx & 3 of the block idx >> 2) at site 107 under key {rng[0], rng[1] + m} (rng device
 * uint64[2] = {seed, step}) is below floor(p_remove 2^32), 0 < p_remove <= 1 (1: every player).  With
 * a = sum_{g in S} phi[b, g] and d = F(x) - F(x with S removed), both fp64, moments [B, RD_REMOVAL_MOMENTS] (fp64) =
 * [sum 1, sum a, sum d, sum a^2, sum a d, sum d^2] over the replicates, added in replicate order; clean_logits
 * [B, n_classes] are the logits at x and target_out [B] (may be NULL) the class F reads.  Work: one forward on the B rows
 * of x, then chunks of replicates_per_chunk replicates on B*replicates_per_chunk rows: the keep-table launch, the
 * expansion, the eval forward and one launch adding the chunk to the moments (one CTA per sample).  scratch:
 * rd_removal_infidelity_scratch_bytes(dims, n_players, replicates_per_chunk) bytes.
 *
 * rd_debug_removal_inputs: the keep-table and expansion launches of one chunk, nc pairs or replicates from q0: curve
 * pairs when rank is given (pair q < K: deletion at counts[q], else insertion at counts[q - K]), else infidelity
 * replicates from rng and p_remove.  Writes keep_table [nc*B, P] (uint8, nonzero = kept) and the rows src_e
 * [T, nc*B, 2N], statics_e [nc*B, d_static] (when d_static > 0), times_e [T, nc*B] and lengths_e [nc*B].
 *
 * dims->obprop_mode 0 is resolved once from the full chunk's row count, so every forward of a call uses the same
 * arithmetic; with it pinned the results are bitwise independent of the chunk size.  Every sum is in a fixed order, no
 * atomics.  Stream-ordered, allocation- and sync-free, CUDA-graph capturable. */
#define RD_REMOVAL_MAX_PLAYERS 16384
#define RD_REMOVAL_DESCENDING 0
#define RD_REMOVAL_ASCENDING 1
#define RD_REMOVAL_ABSOLUTE 2
#define RD_REMOVAL_SUMMARIES 6
#define RD_REMOVAL_MOMENTS 6
size_t rd_removal_curves_scratch_bytes(const rd_dims* dims, int32_t n_players, int32_t pairs_per_chunk);
int rd_raindrop_v2_removal_curves(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                  const float* times, const int64_t* lengths, const float* node_scale,
                                  const float* baseline_src, const float* baseline_statics, const int64_t* target,
                                  const int32_t* cell_player, int64_t player_stride_t, int64_t player_stride_b,
                                  int32_t n_players, const float* attributions, int32_t order, const int32_t* counts,
                                  int32_t n_counts, int32_t pairs_per_chunk, void* scratch, int32_t* rank,
                                  float* curve_logits, float* endpoint_logits, float* values, double* summaries,
                                  int64_t* target_out, void* stream);
size_t rd_removal_infidelity_scratch_bytes(const rd_dims* dims, int32_t n_players, int32_t replicates_per_chunk);
int rd_raindrop_v2_removal_infidelity(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                      const float* times, const int64_t* lengths, const float* node_scale,
                                      const float* baseline_src, const float* baseline_statics, const int64_t* target,
                                      const int32_t* cell_player, int64_t player_stride_t, int64_t player_stride_b,
                                      int32_t n_players, const float* attributions, const uint64_t* rng, double p_remove,
                                      int32_t n_samples, int32_t replicates_per_chunk, void* scratch, float* clean_logits,
                                      double* moments, int64_t* target_out, void* stream);
int rd_debug_removal_inputs(const rd_dims* dims, const float* src, const float* statics, const float* times,
                            const int64_t* lengths, const float* baseline_src, const float* baseline_statics,
                            const int32_t* cell_player, int64_t player_stride_t, int64_t player_stride_b,
                            int32_t n_players, const int32_t* rank, const int32_t* counts, int32_t n_counts,
                            const uint64_t* rng, double p_remove, int64_t q0, int32_t nc, uint8_t* keep_table,
                            float* src_e, float* statics_e, float* times_e, int64_t* lengths_e, void* stream);

/* ---- Monte Carlo dropout predictive uncertainty of Raindrop_v2, in one call ------------------------------------------
 * Replicate m = 0 .. n_samples-1 is exactly the training-mode forward of the B-row batch with the dropout stream at
 * {seed, step + m}, rng = {seed, step} (device uint64[2]; read, never written -- the model's own counter is not
 * advanced).  dims->training is not read: every replicate is a training-mode forward at dims->dropout_p.  With
 * p_m = softmax(logits_m) in fp64:
 *   mean_probs [B, C] = mean_m p_m;  variance [B, C] = sample variance over m of p_m (divisor M - 1, 0 when M = 1);
 *   entropies [3, B]  = (H(mean p), mean_m H(p_m), their difference = the mutual information), natural log, 0 log 0 = 0;
 *   samples [M, B, C] (optional, may be NULL) = the replicates' logits.
 * Work: chunks of replicates_per_chunk replicates, each ONE training forward on B*replicates_per_chunk replicate-major
 * rows (row j = m*B + b) in which every dropout site draws for row j the words the B-row forward at step + m draws for
 * row b, and one launch that adds the chunk into fp64 sums in replicate order (no atomics: the result is bitwise
 * independent of the chunking).  dims->obprop_mode 0 is resolved once from B*replicates_per_chunk rows.
 * scratch: rd_mc_dropout_scratch_bytes(dims, replicates_per_chunk) bytes.  Stream-ordered, allocation- and sync-free,
 * CUDA-graph capturable. */
size_t rd_mc_dropout_scratch_bytes(const rd_dims* dims, int32_t replicates_per_chunk);
int rd_raindrop_v2_mc_dropout(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                              const float* times, const int64_t* lengths, const float* node_scale, const uint64_t* rng,
                              int32_t n_samples, int32_t replicates_per_chunk, void* scratch, float* mean_probs,
                              float* variance, float* entropies, float* samples, void* stream);

/* ---- PGD adversarial examples of Raindrop_v2, in one call ------------------------------------------------------------
 * Untargeted projected gradient descent (Madry et al. 2018) on each sample's own cross-entropy CE(logits_b, y_b) (y NULL:
 * the argmax class of logits_clean), so a sample's result depends on neither B nor the chunking.
 * Threat model: only the value half of src is perturbed, and only at observed cells (src[t, b, N + n] > 0; padded rows
 * have mask 0) of sensors with sensor_perturbable[n] != 0 (NULL: every sensor) of samples with sample_attacked[b] != 0
 * (NULL: every sample); with perturb_static also the statics of those samples.  These elements form S_b.  The mask half,
 * times and lengths never change.  eps is in the units the model sees (per-feature standard deviations after
 * normalisation).  norm RD_PGD_LINF: |delta| <= eps per element; RD_PGD_L2: ||delta_b||_2 <= eps over S_b.
 * Iterates x_k = x + delta_k (an element with delta == 0 keeps x bit for bit):
 *   start   delta_0 = 0; random_start: linf delta_0 ~ U(-eps, eps) per element, l2 uniform in the ball
 *           eps r^(1/d) z / ||z|| (z ~ N(0, I) over S_b, r ~ U(0, 1), d = |S_b|), drawn from Philox4x32-10 at site 98
 *           under rng = {seed, step} (device uint64[2], read only): element e of sample b (e = t*N + n for value cells,
 *           T*N + j for statics) at index b*(T*N + d_static + 1) + e, r at b*(T*N + d_static + 1) + T*N + d_static; the
 *           word of index i is word i & 3 of the block at counter i >> 2 (as for dropout), uniforms (word >> 8) 2^-24,
 *           normals by Box-Muller on the block's word pairs as rd_dp_add_noise draws them
 *   step k  g = d CE(logits_b, y_b) / d x at x_k; linf: delta = clip(delta + alpha sign(g), -eps, eps) (fp32);
 *           l2: delta += alpha g / ||g|| (no step when ||g|| = 0), delta *= min(1, eps / ||delta||) (norms in fp64)
 * Returned per sample: the iterate of highest loss among x_0 .. x_{n_steps} (ties: the earliest), so without a random
 * start loss_adv >= CE at x.  FGSM is n_steps = 1, alpha = eps, random_start = 0.  The lift relu(v R_u) has gradient 0 at
 * a cell whose d_ob channels are all inactive (d_ob = 1: every value of the wrong sign), so such a cell does not move
 * from delta_0 = 0; random_start avoids that.
 *   src_adv      [T, B, 2N]: the returned input (the mask half and every element outside S_b copied bit for bit)
 *   statics_adv  [B, d_static] or NULL (skipped)
 *   logits_adv   [B, n_classes] at src_adv;  loss_adv [B] its cross-entropy (fp64 rounded to fp32)
 *   logits_clean [B, n_classes] at x
 * Eval arithmetic (dims->training must be 0): no dropout, the model's rng state is neither read nor advanced, no
 * parameter gradient is written.  Work: chunks of samples_per_chunk samples; per chunk the inputs expanded in one
 * launch, the forward at x, with random_start one launch drawing x_0 and its forward, then per step the
 * frozen-parameter backward, the dX0 GEMM, one step launch and the next forward, and after every forward one launch
 * that takes the loss and keeps the best iterate: n_steps + 1 (+1 with random_start) forwards and n_steps backwards.
 * Per-sample kernels are one CTA per sample with fixed-order fp64 sums (no atomics): bitwise independent of the
 * chunking.  dims->obprop_mode 0 is resolved once from samples_per_chunk rows, so a shorter last chunk uses the same
 * arithmetic.  scratch: rd_pgd_scratch_bytes(dims, samples_per_chunk) bytes.  Stream-ordered, allocation- and
 * sync-free, CUDA-graph capturable. */
#define RD_PGD_LINF 0
#define RD_PGD_L2 1
size_t rd_pgd_scratch_bytes(const rd_dims* dims, int32_t samples_per_chunk);
int rd_raindrop_v2_pgd(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                       const float* times, const int64_t* lengths, const float* node_scale, const int64_t* y,
                       const uint8_t* sensor_perturbable, const uint8_t* sample_attacked, int32_t perturb_static,
                       int32_t norm, float eps, float alpha, int32_t n_steps, int32_t random_start, const uint64_t* rng,
                       int32_t samples_per_chunk, void* scratch, float* src_adv, float* statics_adv, float* logits_adv,
                       float* logits_clean, float* loss_adv, void* stream);

/* ---- counterfactual explanations of Raindrop_v2, in one call --------------------------------------------------------
 * For each sample b and target class t_b (target NULL: the clean prediction's runner-up, the first argmax over
 * c != the first argmax of logits_clean), a sparse, bounded change delta of the recorded values that makes the model
 * predict t_b (Wachter et al. 2017; the elastic-net form of Dhurandhar et al. 2018).
 * Mutable set S_b (the threat model of rd_raindrop_v2_pgd): the value cells with src[t, b, N + n] > 0 of sensors with
 * sensor_mutable[n] != 0 (NULL: every sensor), plus the statics when opt->perturb_static.  The mask half, times and
 * lengths never change; an element with delta == 0 is written as x bit for bit.
 * Per element, given per sensor n (then per static column j at index N + j, read when perturb_static): a weight
 * w > 0 (weights NULL: 1) and a box [lower, upper] (NULL: -inf / +inf), in normalised units.  The effective box is
 * [min(lower, x), max(upper, x)], so delta = 0 is always feasible; clip_box clips to it.
 * Objective over delta supported on S_b:  c_b max(0, kappa - m(x + delta)) + beta ||w delta||_1 + ||w delta||_2^2, with
 * the logit margin m = z_t - max_{c != t} z_c (first index c* on ties).  The hinge is active when m <= kappa; its logit
 * gradient c_b (e_{c*} - e_t) seeds the frozen-parameter backward.
 * Round s = 0 .. n_search-1 of replica r restarts FISTA at the replica's start point (x_0 = y_0), then for
 * k = 0 .. n_steps-1:  forward at y_k and track;  g = c grad(hinge)(y_k) + 2 w^2 y_k;
 *   x_{k+1} = clip_box(S(y_k - alpha g, alpha beta w))  (S the soft-threshold);
 *   y_{k+1} = clip_box(x_{k+1} + k/(k+3) (x_{k+1} - x_k));
 * and a last forward and track at y_{n_steps}: n_steps + 1 forwards and n_steps backwards per round.  Element arithmetic
 * is fp32 (the iterate the model reads is x + delta clamped to the box); per-sample sums, the distance and c are fp64.
 * A point is valid when m > 0 and m >= kappa; its distance is d = beta ||w delta||_1 + ||w delta||_2^2 (fp64).  The
 * result of sample b is the valid evaluated point of smallest d over all rounds, steps and replicas; ties go to the
 * earliest (round, step), then the lowest replica.  Without a valid point: src_cf is x bit for bit, logits_cf =
 * logits_clean, distance = +inf, valid = 0.
 * Bisection per (sample, replica), lo = 0, hi = +inf, c = c_init; after each round (fp64):
 *   the round found a valid point: hi = min(hi, c), c = (lo + hi) / 2;  else lo = max(lo, c), c = (lo + hi) / 2 if
 *   hi < inf, else 10 c.
 * Restarts: n_restarts = R independent replicas per sample, each with its own c.  Replica 0 starts at delta = 0; replica
 * r >= 1 at clip_box(init_scale (2u - 1)) on S_b, u = (word >> 8) 2^-24 drawn from Philox4x32-10 at site 103 (96: DP
 * noise, 97: Fisher labels, 98: PGD start, 99: Laplace, 100: smoothing, 101: ablation, 102: SWAG) under rng =
 * {seed, step} (device uint64[2], read only; may be NULL when R = 1), element e (t*N + n for value cells, T*N + j for
 * statics) at index (b*R + r)*(T*N + d_static) + e, the word of index i being word i & 3 of the block at counter i >> 2.
 * A replica's search depends on (b, r) alone: replica 0 of an R-replica call is the R = 1 call.
 *   src_cf       [T, B, 2N]: the returned input;  statics_cf [B, d_static] or NULL (skipped)
 *   logits_cf    [B, n_classes] at it;  logits_clean [B, n_classes] at x;  target_out [B] int64
 *   valid        [B] uint8;  distance [B] fp64
 *   c_final      [B, R] fp64: c after the last round's update;  round_valid [B, R, n_search] uint8
 * Eval arithmetic (dims->training must be 0): no dropout, the model's rng state is neither read nor advanced, no
 * parameter gradient is written.  Work: chunks of samples_per_chunk samples on samples_per_chunk*R rows (sample-major);
 * per chunk one launch expanding the inputs, the forward at x and one launch taking the clean logits and target, then
 * per round one start launch and the steps (frozen-parameter backward, dX0 GEMM, one step launch, forward, one track
 * launch), and one bisection launch.  Per-row and per-sample kernels are one CTA each with fixed-order fp64 sums (no
 * atomics): bitwise independent of the chunking once dims->obprop_mode is pinned (mode 0 is resolved once from
 * samples_per_chunk*R rows).  scratch: rd_counterfactual_scratch_bytes(dims, samples_per_chunk, n_restarts) bytes.
 * Stream-ordered, allocation- and sync-free, CUDA-graph capturable. */
typedef struct rd_cf_options {
  double kappa;          /* margin the target must win by, >= 0 */
  double c_init;         /* the hinge's first loss weight, > 0 */
  float beta;            /* L1 weight, >= 0 */
  float step_size;       /* FISTA step alpha, > 0 */
  float init_scale;      /* half-width of the restarts' uniform start, >= 0 */
  int32_t n_search;      /* bisection rounds, >= 1 */
  int32_t n_steps;       /* FISTA steps per round, >= 0 */
  int32_t n_restarts;    /* replicas per sample, >= 1 */
  int32_t perturb_static;
} rd_cf_options;
size_t rd_counterfactual_scratch_bytes(const rd_dims* dims, int32_t samples_per_chunk, int32_t n_restarts);
int rd_raindrop_v2_counterfactual(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                  const float* times, const int64_t* lengths, const float* node_scale,
                                  const int64_t* target, const uint8_t* sensor_mutable, const float* weights,
                                  const float* lower, const float* upper, const rd_cf_options* opt, const uint64_t* rng,
                                  int32_t samples_per_chunk, void* scratch, float* src_cf, float* statics_cf,
                                  float* logits_cf, float* logits_clean, int64_t* target_out, uint8_t* valid,
                                  double* distance, double* c_final, uint8_t* round_valid, void* stream);

/* ---- randomized smoothing of Raindrop_v2: Monte Carlo class votes, in one call --------------------------------------
 * The smoothed classifier g(x) = argmax_c P(f(x + sigma z) = c) (Cohen, Rosenfeld & Kolter 2019) of the eval-mode model
 * f, estimated by counting the argmax classes of n_samples noisy replicates of every sample.
 * Perturbable set S_b (the threat model of rd_raindrop_v2_pgd): the value cells with src[t, b, N + n] > 0 of sensors with
 * sensor_perturbable[n] != 0 (NULL: every sensor), plus the statics when perturb_static.  The mask half, times and
 * lengths are copied bit for bit, and so is every element outside S_b.
 * Noise: replicate m = 0 .. n_samples-1 is x + sigma z, z ~ N(0, I) on S_b and 0 elsewhere (an element whose noise is 0
 * keeps x bit for bit), in normalised units.  z is drawn from Philox4x32-10 at site 100 (96: DP noise, 97: Fisher
 * labels, 98: PGD start, 99: Laplace) under key {seed, step + m}, rng = {seed, step} (device uint64[2], read only):
 * element e of sample b (e = t*N + n for value cells, T*N + j for statics) at index b*(T*N + d_static) + e, counter
 * index >> 2, Box-Muller on the block's word pairs as rd_dp_add_noise draws them.  A replicate depends on
 * (seed, step + m, b) alone, not on B or the chunking.
 *   counts [B, n_classes] int64 = per sample, how many replicates' logits have their (first) maximum at each class.  A
 *          replicate with a non-finite logit votes for no class, so counts.sum(1) <= n_samples.
 * Eval arithmetic (dims->training must be 0): no dropout, the model's rng state is neither read nor advanced, no
 * parameter gradient is written.  Work: chunks of replicates_per_chunk replicates; per chunk one launch expanding the
 * noisy replicate-major rows (row j = m*B + b), ONE eval forward on B*replicates_per_chunk rows and one launch adding
 * the rows' votes (integers: exact, independent of the chunking once dims->obprop_mode is pinned; mode 0 is resolved
 * once from B*replicates_per_chunk rows).  scratch: rd_smooth_scratch_bytes(dims, replicates_per_chunk) bytes.
 * Stream-ordered, allocation- and sync-free, CUDA-graph capturable. */
size_t rd_smooth_scratch_bytes(const rd_dims* dims, int32_t replicates_per_chunk);
int rd_raindrop_v2_smooth_counts(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                 const float* times, const int64_t* lengths, const float* node_scale,
                                 const uint8_t* sensor_perturbable, int32_t perturb_static, float sigma,
                                 const uint64_t* rng, int32_t n_samples, int32_t replicates_per_chunk, void* scratch,
                                 int64_t* counts, void* stream);

/* ---- randomized ablation of Raindrop_v2: class votes over random sensor subsets, in one call -----------------------
 * The ablation-smoothed classifier g(x) = argmax_c P(f(ablate(x, S)) = c) over uniform k-subsets S of the players
 * (Levine & Feizi 2020) of the eval-mode model f, estimated (sampled) or computed exactly (exhaustive) by counting the
 * argmax classes of n_samples ablated replicates of every sample.
 * Players: the sensors n with sensor_player[n] != 0 (NULL: every sensor) in increasing n, then the static vector when
 * ablate_static (last).  n_players = P must be their number (1 <= P <= RD_ABLATION_MAX_PLAYERS); a sensor past the
 * first P - ablate_static players counts as no player.  Sensors that are not players are always kept.
 * Ablating a player writes +0.0 into its value column src[:, b, n] at every time step, also into its mask column
 * src[:, b, N + n] when ablate_mask, and into every static for the static player.  Everything else (kept players, the
 * other sensors, times, lengths) is copied bit for bit.
 * Replicate m = 0 .. n_samples-1 keeps keep = k players (1 <= k <= P), rng = {seed, step} (device uint64[2], read only):
 *   sampled (exhaustive = 0): the first k positions of a partial Fisher-Yates shuffle of 0 .. P-1 (position i swaps
 *     with i + U(P - i), i < k), U(r) Lemire's unbiased bounded integer with rejection, over the 32-bit Philox4x32-10
 *     words of key {seed, step + m} at site 101: word j of sample b at index (b << 32) + j, word index & 3 of the block
 *     at counter index >> 2.  An exactly uniform k-subset; a replicate depends on (seed, step + m, b) alone.
 *   exhaustive (exhaustive = 1): the subset of lexicographic rank step + m among the J = C(P, k) <= 2^31 - 1 subsets
 *     (itertools.combinations order); the seed is ignored and a rank >= J keeps no player.
 *   counts [B, n_classes] int64 = per sample, how many replicates' logits have their (first) maximum at each class; a
 *          replicate with a non-finite logit votes for no class.
 * Eval arithmetic (dims->training must be 0), as rd_raindrop_v2_smooth_counts: per chunk of replicates_per_chunk
 * replicates a keep-table launch, an expansion launch, ONE eval forward on B*replicates_per_chunk rows and one vote
 * launch (exact, independent of the chunking once dims->obprop_mode is pinned).
 * scratch: rd_ablation_scratch_bytes(dims, n_players, replicates_per_chunk) bytes (0: invalid arguments).
 * Stream-ordered, allocation- and sync-free, CUDA-graph capturable. */
#define RD_ABLATION_MAX_PLAYERS 4096
size_t rd_ablation_scratch_bytes(const rd_dims* dims, int32_t n_players, int32_t replicates_per_chunk);
int rd_raindrop_v2_ablation_counts(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                   const float* times, const int64_t* lengths, const float* node_scale,
                                   const uint8_t* sensor_player, int32_t n_players, int32_t ablate_static,
                                   int32_t ablate_mask, int32_t keep, int32_t exhaustive, const uint64_t* rng,
                                   int32_t n_samples, int32_t replicates_per_chunk, void* scratch, int64_t* counts,
                                   void* stream);

/* ---- worst-case sensor removal of Raindrop_v2: the fewest missing players that flip a prediction, in one call --------
 * Players and removal as rd_raindrop_v2_ablation_counts (sensor_player, n_players = P, remove_static, remove_mask):
 * removing a player writes +0.0 into its value column (and mask column when remove_mask, every static for the static
 * player); times and lengths are copied bit for bit.
 * Score of the eval-mode logits z of a row against the reference class: untargeted (target NULL) y = y[b], or the
 * clean prediction (first argmax) when y is NULL, s = z_y - max_{c != y} z_c, success when the first argmax of z is not
 * y; targeted, s = max_{c != t} z_c - z_t with t = target[b], success when the first argmax is t.  fp32; a row with a
 * non-finite logit has s = +inf and never succeeds.  Candidates are ordered by (s, sorted tuple of removed players).
 * Round 0 evaluates the empty set (the clean forward, clean_logits [B, n_classes]).  Round r = 1 .. R = max_removed:
 *   beam (exhaustive = 0): every set S of the beam extended by every player p not in S, W_r * P rows per sample with
 *     W_r = min(W, C(P, r-1)) (rows whose p is in S or whose beam slot is empty are evaluated and ignored); the next
 *     beam is the W = beam_width smallest distinct candidates.  W = 1 is the greedy attack.
 *   exhaustive (exhaustive = 1): every one of the C(P, r) sets of r players; sum_{r <= R} C(P, r) <= 2^31 - 1.
 *   best_score [B, R+1]: the smallest score of each round.  In the first round r with a success, n_removed [B] = r and
 *   the result is the smallest successful candidate of that round; with none by round R, n_removed = -1 and the result
 *   is the smallest candidate of round R.  removed [B, P] (uint8, 1 = removed), logits [B, n_classes] and score [B]
 *   describe the result.
 * 1 <= W <= RD_SENSOR_ATTACK_MAX_BEAM, 1 <= R <= min(P, RD_SENSOR_ATTACK_MAX_REMOVED); y and target are device int64
 * [B] class indices (at most one of them).  Eval arithmetic (dims->training must be 0).  Work: chunks of
 * candidates_per_chunk candidates of a round; per chunk a keep-table launch (beam rounds) or ablation's unranking launch
 * (round 0 and exhaustive rounds), the expansion launch, ONE eval forward on B*candidates_per_chunk rows and one
 * selection launch (one CTA per sample, fixed order, no atomics).  Bitwise independent of the chunking once
 * dims->obprop_mode is pinned.  scratch: rd_sensor_attack_scratch_bytes(dims, n_players, beam_width, max_removed,
 * candidates_per_chunk) bytes (0: invalid arguments).  Stream-ordered, allocation- and sync-free, CUDA-graph
 * capturable. */
#define RD_SENSOR_ATTACK_MAX_BEAM 32
#define RD_SENSOR_ATTACK_MAX_REMOVED 32
size_t rd_sensor_attack_scratch_bytes(const rd_dims* dims, int32_t n_players, int32_t beam_width, int32_t max_removed,
                                      int32_t candidates_per_chunk);
int rd_raindrop_v2_sensor_attack(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                 const float* times, const int64_t* lengths, const float* node_scale,
                                 const uint8_t* sensor_player, int32_t n_players, int32_t remove_static,
                                 int32_t remove_mask, const int64_t* y, const int64_t* target, int32_t beam_width,
                                 int32_t max_removed, int32_t exhaustive, int32_t candidates_per_chunk, void* scratch,
                                 uint8_t* removed, int64_t* n_removed, float* logits, float* clean_logits, float* score,
                                 float* best_score, void* stream);

/* ---- early prediction of Raindrop_v2: the logits of every prefix of every record, in one call ------------------------
 * Prefix r of sample b (0 <= r <= T) is the record cut after row r: rows t < r bit for bit, +0.0 in both halves of src
 * and in times at rows t >= r (how a shorter record is padded), the statics unchanged, and the length lengths[b] when
 * r >= T (the input itself), else min(lengths[b], #{t < r : times[t, b] > 0}) -- the rule lengths follow (one count of
 * times > 0 per sample) applied to the truncated record; it also keeps the quirk of records whose first time is 0.
 * Prefix k = 0 .. n_prefixes-1 is given either
 *   by row count: rows [K] (device int32), r = rows[k] clipped to [0, T], or
 *   by horizon:   horizons [K] (device fp32, in the units of times), r = the number of leading rows with times <= h,
 *                 counted up to the first row whose time exceeds h (a prefix even for unsorted times; padding rows have
 *                 time 0 and count, which changes nothing they hold).
 * Exactly one of the two is given.  A prefix of length 0 is computed as the model computes any length-0 sample: finite,
 * and outside the reference's envelope.
 *   logits  [K, B, n_classes]: the eval-mode logits of prefix k of sample b at [k, b, :]
 *   cutoffs [K, B] int32: r of each (prefix, sample), or NULL (not written)
 *   prefix_lengths [K, B] int64: the prefix's length, or NULL (not written)
 * Eval arithmetic (dims->training must be 0): no dropout, the model's rng state is neither read nor advanced, no
 * parameter gradient is written.  Work: chunks of prefixes_per_chunk prefixes; per chunk one launch computing the
 * cutoffs and lengths (one thread per (prefix, sample)), one launch expanding the prefix-major rows (row j = m*B + b)
 * and ONE eval forward on B*prefixes_per_chunk rows that writes the chunk's logits into its slice of `logits`.  Bitwise
 * the forward on those rows, independent of the chunking once dims->obprop_mode is pinned (mode 0 is resolved once from
 * B*prefixes_per_chunk rows).  scratch: rd_prefix_scratch_bytes(dims, prefixes_per_chunk) bytes (0: invalid
 * arguments).  Stream-ordered, allocation- and sync-free, CUDA-graph capturable. */
size_t rd_prefix_scratch_bytes(const rd_dims* dims, int32_t prefixes_per_chunk);
int rd_raindrop_v2_prefix_logits(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                 const float* times, const int64_t* lengths, const float* node_scale,
                                 const float* horizons, const int32_t* rows, int32_t n_prefixes,
                                 int32_t prefixes_per_chunk, void* scratch, float* logits, int32_t* cutoffs,
                                 int64_t* prefix_lengths, void* stream);

/* ---- out-of-distribution detection for Raindrop_v2: penultimate features, their moments, and per-sample scores -------
 * Post-hoc detectors on the features of a trained eval-mode model (Lee et al. 2018, Mahalanobis; Sun et al. 2022, deep
 * k-nearest neighbours; Hendrycks & Gimpel 2017, maximum softmax probability; Liu et al. 2020, energy).  Every score is
 * oriented so that larger means more likely out of distribution.  Features f [B, Df] of one of two layers:
 *   RD_OOD_POOLED: cat(pooled, emb(static)), the workspace view RD_WS_FEAT;
 *   RD_OOD_HIDDEN: relu(mlp_static.0(f_pooled)), the view RD_WS_HEAD_HIDDEN (the penultimate activation).
 * Fp = Df rounded up to a multiple of 4: the device copies of query rows, the bank and W^T carry zero columns up to Fp
 * (the tensor-core GEMM takes K % 4 == 0), which add exact zeros to every dot product. */
enum rd_ood_layer { RD_OOD_POOLED = 0, RD_OOD_HIDDEN = 1 };
#define RD_OOD_MAX_K 256
#define RD_OOD_SEL_EXTRA 32      /* candidates the kNN selection keeps per query beyond k (rd_raindrop_v2_ood_scores) */

/* features [B, Df] fp32 of `layer` and logits [B, n_classes] (either may be NULL: skipped), copied out of the workspace
 * of eval forwards over chunks of samples_per_chunk samples (the chunk's inputs are copied out of the batch when a
 * chunk does not cover it; the ob-prop arithmetic of mode 0 is resolved from samples_per_chunk rows).  Bitwise the
 * rows the forward writes; independent of the chunking once dims->obprop_mode is pinned.  dims->training must be 0.
 * scratch: rd_ood_features_scratch_bytes(dims, samples_per_chunk) bytes (0: invalid arguments).  Stream-ordered,
 * allocation- and sync-free, CUDA-graph capturable. */
size_t rd_ood_features_scratch_bytes(const rd_dims* dims, int32_t samples_per_chunk);
int rd_raindrop_v2_features(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                            const float* times, const int64_t* lengths, const float* node_scale, int32_t layer,
                            int32_t samples_per_chunk, void* scratch, float* features, float* logits, void* stream);

/* The moments of n feature rows feats [n, F] (fp32, contiguous) with labels [n] (int64), in float64:
 *   class_sums [n_classes, F] = sum of the rows of each class, class_counts [n_classes] int64 = class sizes (labels
 *   outside [0, n_classes) count nowhere; class_sums NULL skips both), gram [F, F] = sum_b f_b f_b^T (NULL: skipped).
 * accumulate != 0 adds to the values already there, else they are overwritten.  Every entry adds the samples one at a
 * time in index order (the products of two fp32 values are exact in fp64, so each step rounds once): the result is
 * bitwise independent of the launch configuration and of how a data set is split across accumulating calls.  One pass
 * over a training set gives the class means and the tied covariance S = gram - sum_c n_c mu_c mu_c^T (on the host).
 * Stream-ordered, allocation- and sync-free, CUDA-graph capturable. */
int rd_feature_moments(const float* feats, const int64_t* labels, int64_t n, int32_t F, int32_t n_classes,
                       int32_t accumulate, double* class_sums, int64_t* class_counts, double* gram, void* stream);

/* The kNN bank of n feature rows feats [n, F]: bank [n, ld] = the L2-normalised rows f / max(||f||_2, 1e-12) (norm in
 * fp64, as F.normalize divides) with zero columns F .. ld-1, and bank_lo = bank - trunc19(bank), the remainder the
 * error-compensated GEMM reads.  ld a multiple of 4, both 16-byte aligned.  rd_raindrop_v2_ood_scores reads the bank
 * with round_up(n, 4) rows: the caller allocates those (their values are never used). */
int rd_ood_prepare_bank(const float* feats, int64_t n, int32_t F, int32_t ld, float* bank, float* bank_lo, void* stream);

/* Per-sample OOD scores of a batch, per chunk of samples_per_chunk samples: ONE eval forward, then
 *   logits [B, C] (a copy of the forward's), msp [B] = -max_c softmax(logits)_c and energy [B] = -T logsumexp(logits/T),
 *   T = temperature > 0 (both in fp64 from the fp32 logits);
 *   Mahalanobis: Z = (f - mean) W on the tensor cores (3xTF32, mean [Df] fp64 subtracted before rounding to fp32),
 *     W^T = w_t [rp, Fp] (rp = r rounded up to 4; zero rows past r and zero columns past Df), then per class
 *     d_c = ||Z - class_proj[c]||^2 in fp64 over rp columns (class_proj [n_classes, rp] = (mu_c - mean) W):
 *     mahalanobis_per_class [B, C], mahalanobis [B] = min_c d_c over the d_c that are numbers and
 *     mahalanobis_class [B] = its first argmin (NaN and class 0 when none is).
 *     With W = V_r Lambda_r^-1/2 from the tied covariance this is min_c (f - mu_c)^T Sigma^+ (f - mu_c);
 *   kNN: the L2-normalised rows q [B, Fp] against the bank [round_up(n_bank, 4), Fp] (rd_ood_prepare_bank) on the
 *     tensor cores (3xTF32, one full-K dot per pair, so a similarity depends on neither the chunking nor the bank
 *     slicing), in slices whose similarities fit in 64 MiB, each merged by a selection launch into a running list of
 *     the ks = min(k + RD_OOD_SEL_EXTRA, n_bank) largest; the last launch recomputes those ks similarities as fp64
 *     dots of the fp32 rows (NaN, from non-finite features, ranks last) and keeps the k largest of them:
 *     knn_index [B, k] int64 = their bank rows (ties: the lower index first) and knn [B] = 2 - 2 s_(k), the squared
 *     distance to the k-th neighbour.  A 3xTF32 similarity is within delta = (6 ceil(Fp/8) + 48) 2^-24 of exact (unit
 *     rows), so the result is the top k of the fp64 dots whenever fewer than RD_OOD_SEL_EXTRA + 1 bank rows have dots
 *     within 2 delta below the k-th.  1 <= k <= min(RD_OOD_MAX_K, n_bank).
 * Any output may be NULL: Mahalanobis runs when one of its three outputs is given (then mean, w_t, class_proj and
 * r >= 1 are needed), kNN when one of its two is (then bank, bank_lo and n_bank >= 1).  Eval arithmetic (dims->training
 * must be 0); every output is bitwise independent of the chunking once dims->obprop_mode is pinned.  scratch:
 * rd_ood_scores_scratch_bytes(dims, r, n_bank, k, samples_per_chunk) bytes, with r = 0 / n_bank = 0 for a call without
 * Mahalanobis / kNN (0: invalid arguments).  Stream-ordered, allocation- and sync-free, CUDA-graph capturable. */
size_t rd_ood_scores_scratch_bytes(const rd_dims* dims, int32_t r, int64_t n_bank, int32_t k, int32_t samples_per_chunk);
int rd_raindrop_v2_ood_scores(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                              const float* times, const int64_t* lengths, const float* node_scale, int32_t layer,
                              const double* mean, const float* w_t, const float* class_proj, int32_t r, const float* bank,
                              const float* bank_lo, int64_t n_bank, int32_t k, float temperature,
                              int32_t samples_per_chunk, void* scratch, float* logits, float* msp, float* energy,
                              float* mahalanobis, int64_t* mahalanobis_class, float* mahalanobis_per_class, float* knn,
                              int64_t* knn_index, void* stream);

/* y[i] = x[i] * keep(site, i) / (1 - p): nn.Dropout driven by the library's counter-based stream (rng_captured =
 * {seed, counter} on the device).  The same call on a gradient is its backward. */
int rd_dropout(const float* x, int64_t n, float p, const uint64_t* rng_captured, uint32_t site, float* y, void* stream);

/* ---- pieces exposed on their own (module-level drop-ins and tests) -------------------------
 * pe[t,b,:] = [sin(times/ts_k), cos(times/ts_k)], k < d_pe/2 (d_pe <= 64)  -> out[(t*B+b)*ld + col0 + 0..d_pe-1]
 * Replaces PositionalEncodingTF.getPE (code/models_rd.py:28-37) without the host round trip. */
int rd_positional_encoding(const float* times, int64_t n_tokens, const float* timescales_host, int32_t d_pe,
                           float* out, int64_t ld, int32_t col0, void* stream);
/* Its backward: d_times[tok] = sum_k d_pe[tok*ld + col0 + k] cos(times/ts_k)/ts_k - d_pe[tok*ld + col0 + d_pe_width/2 + k]
 * sin(times/ts_k)/ts_k, k < d_pe_width/2 (the module-level PositionalEncodingTF is differentiable in times). */
int rd_positional_encoding_bwd(const float* times, const float* d_pe, int64_t n_tokens, const float* timescales_host,
                               int32_t d_pe_width, int64_t ld, int32_t col0, float* d_times, void* stream);

/* out[rows, out_f] = [relu](x[rows, in_f] . weight[out_f, in_f]^T + bias): the encoder's projection
 * GEMM on its own (torch.nn.Linear inside nn.TransformerEncoderLayer, code/models_rd.py:232-237).
 * Error-compensated TF32 on the tensor cores (fp32-level accuracy) when in_f % 4 == out_f % 4 == 0,
 * CUDA cores otherwise.  scratch: rd_linear_scratch_bytes(in_f, out_f) bytes (weight remainder). */
size_t rd_linear_scratch_bytes(int32_t in_features, int32_t out_features);
int rd_linear_fwd(const float* x, const float* weight, const float* bias, int64_t rows, int32_t in_features,
                  int32_t out_features, int32_t relu, float* out, void* scratch, void* stream);

/* Temporal self-attention core of nn.TransformerEncoderLayer.self_attn (code/models_rd.py:232-237,358) for one
 * packed projection qkv [T, B, 3*H*hd] (seq-first, as F.multi_head_attention_forward lays it out):
 *   ctx[t, b, h*hd:(h+1)*hd] = dropout(softmax_j(q_t . k_j / sqrt(hd), keys j >= lengths[b] masked)) . v
 * and its backward d_qkv [T, B, 3*H*hd] from d_ctx [T, B, H*hd] (probabilities are recomputed, nothing T x T is
 * stored).  rng_captured = 2 x uint64 {seed, counter} on the device (ignored when drop_p == 0); `site` selects the
 * dropout stream (16 + layer inside the model).  impl: 0 = automatic, 1 = tensor-core kernels
 * (T <= 64, hd <= 96, hd % 4 == 0), 2 = CUDA-core kernels (T <= 64, hd <= 96).  Longer sequences are handled inside
 * rd_raindrop_v2_fwd/_bwd (they need workspace). */
int rd_temporal_attention_fwd(const float* qkv, const int64_t* lengths, int32_t B, int32_t H, int32_t T, int32_t hd,
                              float drop_p, const uint64_t* rng_captured, uint32_t site, int32_t impl, float* ctx,
                              void* stream);
int rd_temporal_attention_bwd(const float* qkv, const float* d_ctx, const int64_t* lengths, int32_t B, int32_t H,
                              int32_t T, int32_t hd, float drop_p, const uint64_t* rng_captured, uint32_t site,
                              int32_t impl, float* d_qkv, void* stream);

/* Weight/bias gradients of up to 12 torch.nn.Linear layers in ONE grouped tensor-core launch (+ one reduction
 * launch): d_weight[out_f, in_f] = d_out[rows, out_f]^T . x[rows, in_f], d_bias[out_f] = column sums of d_out.
 * This is what autograd computes for every Linear on the path (code/Raindrop.py:323); a training step has ten of
 * them (8 encoder weights + the two lin_value).  Error-compensated TF32 (fp32-level accuracy), deterministic.
 * `partial`: rd_linear_wgrad_partial_bytes(rows, out_f, in_f) bytes of scratch per problem, 16-byte aligned. */
typedef struct rd_wgrad_item {
  const float* d_out; const float* x; int64_t rows; int32_t out_features; int32_t in_features;
  float* d_weight; float* d_bias; void* partial;
} rd_wgrad_item;
size_t rd_linear_wgrad_partial_bytes(int64_t rows, int32_t out_features, int32_t in_features);
int rd_linear_wgrad_group(const rd_wgrad_item* items, int32_t n, void* stream);

/* TransformerConv.forward (code/transformer_conv.py:139-207), concat=True, root_weight=True, beta=False, no edge
 * features -- and its backward.  Batched over `n_graphs` independent graphs that share ONE edge list (legacy Raindrop v1
 * applies the layer to every sample of a batch, code/models_rd.py:158-166): the row of node i of graph g in x / out is
 * i * node_stride + g * graph_stride (single graph: n_graphs = 1, node_stride = 1, graph_stride = 0).  The rows must
 * tile [0, n_nodes * n_graphs) densely: (node_stride, graph_stride) = (n_graphs, 1) or (1, n_nodes); anything else is
 * refused.
 *   x [rows, in];  weights [H*F, in];  edge_w [E] or NULL (then the logits are q_i.k_j / sqrt(F));
 *   out [rows, H*F];  alpha [n_graphs, E, H] (post-softmax, as returned by the reference).
 * Backward: writes d_x (may be NULL), d_w* / d_b* (written, not accumulated; with edge_w the q/k projections take no
 * part in the output, code/transformer_conv.py:199-200, so their gradients are zeros) and d_edge_w [E] (optional,
 * only with edge_w).  scratch: rd_transformer_conv_scratch_bytes(..., backward) bytes. */
size_t rd_transformer_conv_scratch_bytes(int32_t n_nodes, int32_t n_graphs, int32_t in_ch, int32_t heads,
                                         int32_t out_ch, int32_t E, int32_t backward);
int rd_transformer_conv_fwd(const float* x, int32_t n_nodes, int32_t n_graphs, int64_t node_stride,
                            int64_t graph_stride, int32_t in_ch, int32_t heads, int32_t out_ch,
                            const int64_t* edge_src, const int64_t* edge_tgt, const float* edge_w, int32_t E,
                            const float* wq, const float* bq, const float* wk, const float* bk, const float* wv,
                            const float* bv, const float* ws, const float* bs, float* out, float* alpha,
                            void* scratch, void* stream);
int rd_transformer_conv_bwd(const float* x, int32_t n_nodes, int32_t n_graphs, int64_t node_stride,
                            int64_t graph_stride, int32_t in_ch, int32_t heads, int32_t out_ch,
                            const int64_t* edge_src, const int64_t* edge_tgt, const float* edge_w, int32_t E,
                            const float* wq, const float* bq, const float* wk, const float* bk, const float* wv,
                            const float* bv, const float* ws, const float* alpha, const float* d_out, float* d_x,
                            float* d_wq, float* d_bq, float* d_wk, float* d_bk, float* d_wv, float* d_bv,
                            float* d_ws, float* d_bs, float* d_edge_w, void* scratch, void* stream);

/* ---- device-side batch assembly (SURVEY.md 8f2) ---------------------------------------------------
 * out[t, j, :] = src[t, idx[j], :] for t < T, j < B: selects a batch out of a training set that stays
 * resident in HBM, replacing the host-side `Ptrain_tensor[:, idx, :].cuda()` copies of
 * code/Raindrop.py:311-315 (T = 1 for the [n, d_static] statics and labels viewed as float rows). */
int rd_gather_batch(const float* src, const int64_t* idx, int64_t T, int64_t n_total, int32_t width, int32_t B,
                    float* out, void* stream);

/* Whole-batch assembly in ONE launch: for j < B copies sample idx[j] of the resident tensors P [T, n_total, width],
 * Ptime [T, n_total], Pstatic [n_total, d_static] (may be NULL), y [n_total] (may be NULL) into the batch buffers and
 * writes lengths[j] = #(Ptime[:, idx[j]] > 0)  (code/Raindrop.py:311-317). */
int rd_assemble_batch(const float* P, const float* Ptime, const float* Pstatic, const int64_t* y, const int64_t* idx,
                      int32_t T, int64_t n_total, int32_t width, int32_t d_static, int32_t B, float* src, float* times,
                      float* statics, int64_t* y_out, int64_t* lengths, void* stream);

/* Per-feature statistics of the OBSERVED entries (value > 0) of raw [n, T, F]: mean and population standard deviation
 * (floored at 1e-7), accumulated in double -- getStats, code/utils_rd.py:149-161.
 * scratch: rd_feature_stats_scratch_bytes(n, T, F) bytes. */
size_t rd_feature_stats_scratch_bytes(int64_t n, int32_t T, int32_t F);
int rd_feature_stats(const float* raw, int64_t n, int32_t T, int32_t F, float* mean, float* std, void* scratch,
                     void* stream);
/* mask_normalize (code/utils_rd.py:164-175) fused with the concat of the observation mask and the permute to the
 * training layout (code/Raindrop.py:233): raw [n, T, F] -> out [T, n, 2F] with
 *   out[t, i, f] = raw > 0 ? (raw - mean_f) / (std_f + 1e-18) : 0      out[t, i, F + f] = raw > 0
 * minutes (optional) [n, T] -> times_out [T, n] = minutes / 60 (code/utils_rd.py:235). */
int rd_mask_normalize(const float* raw, const float* mean, const float* std, int64_t n, int32_t T, int32_t F,
                      float* out, const float* minutes, float* times_out, void* stream);
/* Leave-sensors-out masking of a batch P [T, B, width = 2F] (code/Raindrop.py:214-231): zero the VALUE columns
 * idx[k], k < K; per_sample != 0: idx is [B, K] (feature_removal_level 'sample'), else [K] ('set').  The mask columns
 * are left untouched, exactly as in the reference. */
int rd_zero_features(float* P, int64_t T, int32_t B, int32_t width, const int64_t* idx, int32_t K, int32_t per_sample,
                     void* stream);

/* ---- training-step helpers (the caller-side ops of code/Raindrop.py:321-324) ----------------
 * mean cross entropy + d(loss)/d(logits), torch.nn.CrossEntropyLoss semantics. */
int rd_cross_entropy_fwd_bwd(const float* logits, const int64_t* y, int32_t B, int32_t n_classes,
                             float* loss, float* d_logits, void* stream);
/* torch.optim.Adam (no weight decay, no amsgrad) on flat buffers, ONE launch.  `step` is int64[2] on the
 * device: step[0] = number of updates so far (incremented by the call, by the last CTA to finish),
 * step[1] = ticket word that must be 0 on entry (the call leaves it 0).  grad is multiplied by grad_scale
 * first (1/world_size after a sum all-reduce).  lr_dev: optional device scalar that overrides `lr`, so a
 * captured CUDA graph follows a scheduler (ReduceLROnPlateau, code/Raindrop.py:257-259) without re-capture. */
int rd_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n,
                 float lr, const float* lr_dev, float beta1, float beta2, float eps, float grad_scale,
                 int64_t* step, void* stream);

/* ---- differentially private training (DP-SGD, Abadi et al. 2016) ---------------------------------------------------
 * theta = the trained tensors of Raindrop_v2 in flat-bucket order (raindrop_b200.functional.used_param_fields): the
 * head (emb weight and bias when d_static > 0, mlp_static.0 weight and bias, mlp_static.2 weight and bias), 12 per
 * encoder layer (in_proj weight, bias, out_proj weight, bias, linear1 weight, bias, linear2 weight, bias, norm1 weight,
 * bias, norm2 weight, bias), then ob_propagation.lin_value weight, bias and ob_propagation_layer2.lin_value weight,
 * bias: n_fields = (d_static > 0 ? 6 : 4) + 12 nlayers + 4.  l_b = CrossEntropy(logits_b, y_b) of the forward in the
 * workspace (training mode: with its dropout masks), g_b = grad_theta l_b.  A DP step:
 *   1. rd_raindrop_v2_fwd with labels: d_logits = (softmax - onehot) / B;
 *   2. rd_raindrop_v2_per_sample_grad_sqnorms: the per-sample squared norms of the gradient of l_b / B;
 *   3. rd_dp_clip_scale: d_logits row b *= w_b c_b B / L with c_b = min(1, C / (||g_b|| + 1e-6));
 *   4. rd_raindrop_v2_bwd(RD_BWD_ALL) on the same workspace: grads = sum_b w_b c_b g_b / L;
 *   5. rd_dp_add_noise: grads += (sigma C / L) xi, xi ~ N(0, I) over the used elements of the bucket;
 *   6. rd_adam_step. */

/* Scratch of rd_raindrop_v2_per_sample_grad_sqnorms: a backward scratch and the norm pass's partial sums. */
size_t rd_dp_scratch_bytes(const rd_dims* dims);
/* sqnorms [B, n_fields] (fp64, device) = the squared L2 norm of each sample's gradient per trained tensor, for the
 * gradient the backward would compute from d_logits (after step 1: of l_b / B).  Runs the data-gradient chain of the
 * backward (grads == NULL, as rd_raindrop_v2_bwd); per linear layer the sample's rows (encoder: t*B + b, ob-prop:
 * b*N + n) give the norm in the cheaper of the ghost form sum_{r,r'} (y_r.y_r')(x_r.x_r' + 1) and the explicit form
 * ||sum_r y_r [x_r, 1]^T||^2 (chosen from the shape alone); LayerNorm gamma / beta from the recomputed normalised input;
 * the head from its one row per sample.  Every entry is written by one thread in a fixed order, without atomics: the
 * result is bitwise reproducible.  The workspace and the backward's arithmetic mode are those of the forward (dims as
 * passed to it).  scratch: rd_dp_scratch_bytes(dims) bytes.  Stream-ordered, sync-free, CUDA-graph capturable. */
int rd_raindrop_v2_per_sample_grad_sqnorms(const rd_dims* dims, const rd_params* params, const float* statics,
                                           const int64_t* lengths, const float* node_scale, const void* workspace,
                                           const float* d_logits, void* scratch, double* sqnorms, void* stream);
/* Clipping, in place on d_logits [B, n_classes] of step 1: n_b = B sqrt(sum_f sqnorms[b, f]) (fp64),
 * c_b = min(1, max_grad_norm / (n_b + 1e-6)) -> clip_factors[b]; row b *= w_b c_b B / expected_batch_size, weight [B]
 * in {0, 1}; loss = sum_b w_b l_b / sum_b w_b (0 when every weight is 0) from the forward's per-sample losses in the
 * workspace.  One launch. */
int rd_dp_clip_scale(const rd_dims* dims, const void* workspace, const double* sqnorms, const float* weight,
                     float max_grad_norm, float expected_batch_size, float* d_logits, float* clip_factors, float* loss,
                     void* stream);
/* grad[i] += noise_std * xi_i for i in the used ranges [field_offsets[f], + field_numel[f]) of the flat bucket grad [n]
 * (host arrays, ascending, offsets % 4 == 0, n % 4 == 0, 1 <= n_fields <= 128); padding is not touched.  xi_i is drawn
 * from the Philox4x32-10 stream of the dropout masks with key {seed, step} = key[0], key[1] (device uint64[3]; key[2]
 * is a ticket word, 0 on entry), site 96, counter i >> 2, and Box-Muller on the block's word pairs:
 * u1 = ((w0 >> 8) + 1) 2^-24, u2 = (w1 >> 8) 2^-24, xi = sqrt(-2 ln u1) (cos, sin)(2 pi u2) in fp64, rounded to fp32.
 * The launch advances key[1] by one, so CUDA-graph replays draw fresh noise.  Philox is not a cryptographically secure
 * generator.  One 128-bit grid-stride launch. */
int rd_dp_add_noise(float* grad, int64_t n, const int64_t* field_offsets, const int64_t* field_numel, int32_t n_fields,
                    float noise_std, uint64_t* key, void* stream);

/* ---- training-data influence (TracIn, Pruthi et al. 2020) -----------------------------------------------------------
 * influence(z_q, z_t) = sum_c lr_c < g_q(theta_c), g_t(theta_c) >, g = the per-sample gradients of the DP-SGD section
 * above, materialised as rows of the flat bucket and contracted on the tensor cores. */

/* Scratch of rd_raindrop_v2_per_sample_grads: a backward scratch. */
size_t rd_per_sample_grads_scratch_bytes(const rd_dims* dims);
/* G [B, ldg] (fp32, device, 16-byte aligned): row b = g_b = grad_theta CrossEntropy(logits_b, y_b), the gradient of l_b
 * (not of l_b / B), in the layout of TrainStep's flat gradient bucket: the trained tensors in the order of the DP-SGD
 * section, each at an offset rounded up to 4 floats, padding columns written as 0, ldg = the bucket length (anything
 * else is refused).  d_logits: as rd_raindrop_v2_fwd writes it with labels (the gradient of l_b / B; every row is
 * scaled by B).  Runs the data-gradient chain of the backward (grads == NULL) and, where the training path queues a
 * weight-gradient item, writes sample b's [Nout, Kin + 1] tile of dY_b^T [X_b | 1] (the bias as the ones column;
 * encoder rows t*B + b, ob-prop rows b*N + n) on the CUDA cores, fp32 slices of 16 rows summed in fp64; LayerNorm
 * gamma / beta from the recomputed normalised input; the head from its one row per sample.  Every value is scaled and
 * rounded to fp32 once, written by one thread, without atomics: bitwise reproducible.  scratch:
 * rd_per_sample_grads_scratch_bytes(dims) bytes.  Stream-ordered, sync-free, CUDA-graph capturable. */
int rd_raindrop_v2_per_sample_grads(const rd_dims* dims, const rd_params* params, const float* statics, const int64_t* lengths,
                                    const float* node_scale, const void* workspace, const float* d_logits, void* scratch,
                                    float* G, int64_t ldg, void* stream);

/* Longest segment of rd_per_sample_grad_dot, in columns: each segment's inner product is one fp32 sum of at most this
 * many error-compensated products. */
#define RD_GRAD_DOT_SEGMENT 4096
/* Scratch of rd_per_sample_grad_dot: the remainder image of Gq [Bq, ldg], the segment table and fp32 partial sums
 * [n_seg, Bq, Bt]. */
size_t rd_per_sample_grad_dot_scratch_bytes(int32_t Bq, int32_t Bt, int64_t ldg, int32_t n_seg);
/* scores[q * lds + t] += alpha * sum_s < Gq[q, seg_s], Gt[t, seg_s] > for q < Bq, t < Bt (fp64, device).  Gq [Bq, ldg]
 * and Gt [Bt, ldg]: fp32 rows, device, 16-byte aligned, ldg % 4 == 0.  Segment s = columns [seg_off[s], + seg_len[s])
 * (host arrays, n_seg <= 65535, offsets % 4 == 0, 1 <= length <= RD_GRAD_DOT_SEGMENT, inside the row).  Precondition:
 * a segment runs in 32-column blocks from its offset, and its last block may reach past its end (into the next field,
 * or past ldg, where nothing is read).  Gt's columns there are replaced by 0, but Gq's are read and multiplied by that
 * 0, so they must be finite: a NaN or Inf in Gq[q, seg_off[s] + seg_len[s] .. seg_off[s] + 32 ceil(seg_len[s] / 32))
 * makes every score of query q NaN (0 * Inf is NaN).  Columns further from every segment are never multiplied into a
 * score.  One psg_lo launch (the remainder image), one launch of wgmma 3xTF32 tiles over (64 queries, 128 train rows, segment), each segment summed in
 * fp32, and one reduce launch adding the segments in order in fp64: every score is the same product sequence whatever
 * Bq, Bt and the segment count, hence bitwise reproducible across query blockings and train chunkings.  Stream-ordered;
 * the segment table is copied from the host (not CUDA-graph capturable). */
int rd_per_sample_grad_dot(const float* Gq, int32_t Bq, const float* Gt, int32_t Bt, int64_t ldg, const int64_t* seg_off,
                           const int64_t* seg_len, int32_t n_seg, double alpha, double* scores, int64_t lds, void* scratch,
                           void* stream);

/* Random projection of gradient rows (TracIn-RP, Pruthi et al. 2020): phi = g Omega / sqrt(dim), E[phi_q . phi_t] =
 * g_q . g_t.  Omega [ldg, dim] is +-1 and never stored: Omega(seed, j, m) for absolute column j and dimension m is
 * bit (j & 31) of word ((j >> 5) & 3) of Philox4x32-10 with key (seed & 0xffffffff, seed >> 32) and counter
 * (jb & 0xffffffff, jb >> 32, m, 0), jb = j >> 7 (words and bits numbered from 0, bits from the least significant);
 * bit 0 -> +1, bit 1 -> -1.  A column has the same signs whatever the fields, the segments or the rows.  dim: a multiple
 * of 128 in [128, 32768]. */
/* Scratch of rd_grad_projection: the remainder image of G [rows, ldg], the segment table and fp32 partial sums
 * [n_seg, rows, dim]; 0 for sizes rd_grad_projection refuses. */
size_t rd_grad_projection_scratch_bytes(int32_t rows, int64_t ldg, int32_t dim, int32_t n_seg);
/* out[r * ldo + m] = (1/sqrt(dim)) sum_s sum_{j in seg_s} G[r, j] Omega(seed, j, m) for r < rows, m < dim (fp32,
 * device).  G [rows, ldg]: fp32 rows, device, 16-byte aligned, ldg % 4 == 0.  Segments as for rd_per_sample_grad_dot
 * (host arrays, n_seg <= 65535, offsets % 4 == 0, 1 <= length <= RD_GRAD_DOT_SEGMENT, inside the row); the k-blocks
 * run over whole 32-column blocks, so columns next to a segment are read and multiplied by 0 and the rows must be
 * finite.  One psg_lo launch (the remainder image), one launch of wgmma TF32 tiles over (128 dimensions, 64 rows,
 * segment) with Omega drawn in registers and two passes (Omega.G_lo, Omega.G_hi; Omega is exact in TF32), each segment
 * summed in fp32, and one reduce launch adding the segments in order in fp64 and rounding to fp32 once.  A row's output
 * is bitwise the same whatever the other rows of the launch and `rows`.  Stream-ordered, sync-free; the segment table
 * is copied from the host (not CUDA-graph capturable). */
int rd_grad_projection(const float* G, int32_t rows, int64_t ldg, const int64_t* seg_off, const int64_t* seg_len,
                       int32_t n_seg, int32_t dim, uint64_t seed, float* out, int64_t ldo, void* scratch, void* stream);

/* ---- EK-FAC influence functions (George et al. 2018; Grosse et al. 2023) ----------------------------------------------
 * score(q, t) = sum_j G~_q[j] G~_t[j] / (Lambda_j + lambda), G~ = the gradient rows rotated into the Kronecker eigenbasis
 * of each linear layer's Fisher block A (x) S:  G~_b = Q_S^T G_b Q_A = sum_r (Q_S^T dy_r)(Q_A^T x~_r)^T, x~ = [x | 1].
 * Blocks, in bucket order: per encoder layer in_proj [3D, D], out_proj [D, D], linear1 [nhid, D], linear2 [D, nhid],
 * then the lin_value of ob-prop layers 1 and 2 [C, C] ([Nout, Kin] each).  Every block covers its weight and bias.
 * factors (fp64): per block A [(Kin + 1)^2] then S [Nout^2], row-major, packed (rd_kfac_factors_doubles(dims) in all).
 * bases (fp32): per block Q_S^T [Nout, Nout] (padded to 4 floats), Q_A[:Kin]^T [Np, Kin] and Q_A[Kin] [Np], Np = Kin + 1
 * rounded up to 4, rows / entries past Kin + 1 zero (rd_ekfac_bases_floats(dims) in all). */
int64_t rd_kfac_factors_doubles(const rd_dims* dims);
int64_t rd_ekfac_bases_floats(const rd_dims* dims);
/* Scratch of rd_raindrop_v2_kfac_factors: a backward scratch, the fp32 factor sums of every block and their partial
 * buffers. */
size_t rd_kfac_factors_scratch_bytes(const rd_dims* dims);
/* factors += this batch's K-FAC sums, per block A += sum_rows x~ x~^T over [X | 1] and S += sum_rows (B dy)(B dy)^T
 * (d_logits as rd_raindrop_v2_fwd writes it with labels, the gradient of l_b / B; scaled to l_b as the rows are), over
 * the rows of each queued item (encoder t*B + b for all T, ob-prop b*N + n).  Runs the data-gradient chain of the backward
 * (grads == NULL); each item becomes two weight-gradient problems (X, X) and (dY, dY) of the grouped tensor-core launch
 * (CUDA cores for shapes it does not take), flushed with the phase; one small launch per block then adds the fp32 sums
 * into the fp64 factors (the last row and column of A from the bias column and the row count).  No atomics: bitwise
 * reproducible.  The caller divides by the sample count.  Stream-ordered, sync-free. */
int rd_raindrop_v2_kfac_factors(const rd_dims* dims, const rd_params* params, const float* statics, const int64_t* lengths,
                                const float* node_scale, const void* workspace, const float* d_logits, void* scratch,
                                double* factors, void* stream);
/* Scratch of rd_raindrop_v2_ekfac_rows: a backward scratch, the remainder image of the bases and the rotated operands
 * of the larger backward phase. */
size_t rd_ekfac_rows_scratch_bytes(const rd_dims* dims);
/* As rd_raindrop_v2_per_sample_grads, but the linear layers' fields hold the rotated G~_b: each queued item's operands
 * are first rotated, Y^ = dY Q_S and X^ = [X | 1] Q_A (the error-compensated tensor-core GEMM of rd_linear_fwd, the
 * last row of Q_A as its bias), and sample b's tile Y^_b^T X^_b goes to the weight field (columns < Kin) and the bias
 * field (column Kin).  LayerNorm and head fields are the plain gradient (identity basis).  bases: 16-byte aligned. */
int rd_raindrop_v2_ekfac_rows(const rd_dims* dims, const rd_params* params, const float* statics, const int64_t* lengths,
                              const float* node_scale, const void* workspace, const float* d_logits, const float* bases,
                              void* scratch, float* G, int64_t ldg, void* stream);
/* lam[j] += sum_{r < rows} G[r * ldg + j]^2 (fp64, rows in order, one thread per column, no atomics) for the columns of
 * the segments (host arrays; segments separated by bucket padding only are launched as one run). */
int rd_ekfac_accumulate_sq(const float* G, int32_t rows, int64_t ldg, const int64_t* seg_off, const int64_t* seg_len,
                           int32_t n_seg, double* lam, void* stream);
/* G[r * ldg + j] *= w[j] (fp32) for r < rows and the columns of the segments. */
int rd_ekfac_scale_rows(float* G, int32_t rows, int64_t ldg, const int64_t* seg_off, const int64_t* seg_len,
                        int32_t n_seg, const float* w, void* stream);
/* Labels of the true Fisher: y[b] = the first class c with u_b sum_c' p_c' < sum_{c'' <= c} p_c'' (fp64, p_c =
 * exp(logits[b, c] - max_c logits[b, c]), classes in order; the last class if none), u_b = U(seed, index0 + b).
 * U(seed, i) = ((w0 >> 5) 2^26 + (w1 >> 6)) / 2^53 with (w0, w1, w2, w3) = Philox4x32-10 with key (seed & 0xffffffff,
 * seed >> 32) and counter (i & 0xffffffff, i >> 32, 97, 0): site 97, past the dropout sites 1-96.  A sample's label
 * depends on (seed, its global index, its logits) alone. */
int rd_fisher_labels(const float* logits, int32_t B, int32_t n_classes, uint64_t seed, uint64_t index0, int64_t* y,
                     void* stream);
/* debug: out[i] = U(seed, index0 + i) (fp64, device) for i < n. */
int rd_debug_fisher_uniforms(uint64_t seed, uint64_t index0, int32_t n, double* out, void* stream);

/* ---- TRAK (Park et al. 2023) ------------------------------------------------------------------------------------------
 * tau(q, i) = [(1/M) sum_k sum_j w_kj (phi_k(q) v_kj)(phi_k(z_i) v_kj)] [(1/M) sum_k Q_k(i)], phi = the projected margin
 * gradient rows (rd_grad_projection of rows seeded by rd_trak_margin_seed), K = Phi^T Phi = V diag(lambda) V^T over the
 * training set, w = 1 / (lambda + damping), Q = sigmoid(-margin).  dim: a multiple of 128 in [128, RD_TRAK_DIM_MAX]. */
#define RD_TRAK_DIM_MAX 8192
/* The margin seed: for each b < B, with m_b = z_y - log sum_{c != y} exp(z_c) (z = logits[b], y = y[b]),
 * d_logits[b, y] = 1 / B and d_logits[b, c] = -exp(z_c - M) / S / B for c != y (M = max_{c != y} z_c, S =
 * sum_{c != y} exp(z_c - M)), the gradient of m_b / B as rd_raindrop_v2_fwd writes the loss's, so that
 * rd_raindrop_v2_per_sample_grads on an eval forward without labels gives grad_theta m_b; Q[b] = sigmoid(-m_b) (fp64).
 * Everything in fp64, d_logits rounded to fp32 once: saturated rows stay finite and Q >= 0 without cancellation.
 * n_classes >= 2; labels outside [0, n_classes) give NaN rows.  Stream-ordered, sync-free. */
int rd_trak_margin_seed(const float* logits, int32_t B, int32_t n_classes, const int64_t* y, float* d_logits, double* Q,
                        void* stream);
/* K[i, j] += sum_{r < n} Phi[r, i] Phi[r, j] for i, j < dim (fp64, device, [dim, dim] row-major).  Phi [n, dim]: fp32,
 * device, 16-byte aligned.  One launch of 64 x 64 tiles over the upper triangle, mma.sync m16n8k16 f64 (the products of
 * fp32 inputs are exact in fp64) summed over 32-row k-blocks in row order; each tile is added at (bi, bj) and its
 * transpose at (bj, bi), a diagonal tile's upper triangle on both sides, so K stays exactly symmetric when it was.  The
 * order of every sum is fixed by (n, dim) alone and there are no atomics: bitwise reproducible.  Stream-ordered,
 * sync-free. */
int rd_trak_gram(const float* Phi, int64_t n, int32_t dim, double* K, void* stream);
/* out[r, j] = fp32(sum_k Phi[r, k] V[k, j]) for r < n, j < dim.  Phi [n, dim] fp32, V [dim, dim] fp64 row-major, out
 * [n, dim] fp32 (device, 16-byte aligned, n <= 65535 * 64).  mma.sync m16n8k16 f64 over 32-column k-blocks in order,
 * rounded once: a row's output depends on its row of Phi and on V alone, whatever the other rows of the launch.
 * Stream-ordered, sync-free. */
int rd_trak_rotate(const float* Phi, int64_t n, int32_t dim, const double* V, float* out, void* stream);

/* ---- Batch active learning: BatchBALD (Kirsch et al. 2019) and BADGE (Ash et al. 2020) --------------------------------
 * Both pick k points of an unlabelled pool of N, greedily, in one stream-ordered call whose loop has no host
 * synchronisation (the argmax and the CDF search run on the device), so it can be captured in a CUDA graph.  Random
 * draws are Philox4x32-10 with key (seed & 0xffffffff, (seed >> 32) ^ (step >> 32)) and counter (c0, c1, site,
 * step & 0xffffffff), word 0 (and 1): sites 105 (BatchBALD) and 106 (BADGE), past every dropout and sampling site. */
#define RD_ACTIVE_MAX_CLASSES 8
#define RD_ACTIVE_MAX_REPLICATES 1024
#define RD_ACTIVE_MAX_CONFIGS 65536
/* Bytes of scratch rd_batch_bald needs (0 for sizes it refuses).  chunk: candidates per joint-entropy launch. */
size_t rd_batch_bald_scratch_bytes(int64_t N, int32_t M, int32_t C, int32_t n_configs, int64_t chunk);
/* Greedy BatchBALD over logits [M, N, C] (fp32, device; replicate-major).  Step i, with the chosen set A (|A| = i), picks
 * the unchosen n maximising H(y_A, y_n) - sum_{a in A u {n}} E_m H(y_a | theta_m), ties to the lowest index.  The joint
 * entropy is exact while C^i <= n_configs (the C^i configurations of A as mixed-radix rows), otherwise Kirsch's
 * importance-weighted estimate over n_configs configurations drawn from the mixture: configuration s draws its
 * replicate m_s = (w M) >> 32 from w = word 0 at counter (s, 0), and its label for the pick of step j as
 * min{c : (w >> 8) 2^-24 < fp32 cumsum_c p[m_s, a_j, c]} from w = word 0 at counter (s, j + 1) (the largest class with
 * p > 0 if none).  Rows of configurations are kept scaled to max 1 with their log-scale in fp64.  The products
 * Q = P_A . p run on the tensor cores in 3xTF32 with the entropy in the epilogue (fp32 logarithm, fp64 sums).  Outputs
 * (device): indices [k] int64, scores [k] fp64 (the joint mutual information of the batch after each pick), exact [k]
 * (1 where the pick enumerated), bald [N] fp64 (the single-point mutual information).  Every sum has an order fixed
 * by (N, M, C, n_configs): the result is bitwise independent of `chunk`.  2 <= C <= RD_ACTIVE_MAX_CLASSES, 1 <= M <=
 * RD_ACTIVE_MAX_REPLICATES, 1 <= n_configs <= RD_ACTIVE_MAX_CONFIGS, 1 <= k <= N; scratch 256-byte aligned. */
int rd_batch_bald(const float* logits, int64_t N, int32_t M, int32_t C, int32_t k, int32_t n_configs, uint64_t seed,
                  uint64_t step, int64_t chunk, void* scratch, int64_t* indices, double* scores, uint8_t* exact,
                  double* bald, void* stream);
/* Bytes of scratch rd_badge needs (0 for sizes it refuses). */
size_t rd_badge_scratch_bytes(int64_t N, int32_t F, int32_t C);
/* BADGE's k-means++ seeding over g_n = (p_n - e_yhat_n) (x) [h_n; 1], hidden [N, F] and logits [N, C] (fp32, device),
 * p = softmax, yhat = argmax (ties to the lowest class).  Distances use the factorised form |a_i|^2 |h~_i|^2 +
 * |a_c|^2 |h~_c|^2 - 2 (a_i . a_c)(h~_i . h~_c) (fp32 products in fp64, fp64 sums, clamped at 0): the embedding is never
 * formed.  The first centre has the largest norm (ties to the lowest index); pick i >= 1 draws U = ((w0 >> 5) 2^26 +
 * (w1 >> 6)) 2^-53 at counter (i, 0) and takes the first point whose running sum of D^2, in tiles of 256 points in
 * index order, exceeds U sum D^2 (the lowest unchosen index when every D^2 is 0).  Outputs (device): indices [k] int64
 * and d2 [k] fp64, D^2 at pick time (inf for the first).  2 <= C <= RD_ACTIVE_MAX_CLASSES, 1 <= k <= N. */
int rd_badge(const float* hidden, const float* logits, int64_t N, int32_t F, int32_t C, int32_t k, uint64_t seed,
             uint64_t step, void* scratch, int64_t* indices, double* d2, void* stream);

/* ---- KNN-Shapley data valuation (Jia et al., VLDB 2019) ----------------------------------------------------------------
 * The exact Shapley value of every training record under the utility of a K-nearest-neighbour classifier, per query:
 * U(S) = (1/K) #{the min(K, |S|) records of S most similar to q that carry q's label}.  Similarity = the fp64 dot of two
 * L2-normalised fp32 rows (rd_ood_prepare_bank); the N candidates are ranked by similarity descending, ties to the lower
 * index (alpha_1 .. alpha_N).  With m_r = 1[y_train(alpha_r) = y_q] and c_r = min(K, r) / (r K), the record at rank r
 * gets s_r = m_r c_r - sum_{j = max(r, K) + 1}^{N} m_j / (j (j - 1)), which is Theorem 1's recursion s_r = s_{r+1} +
 * (m_r - m_{r+1}) c_r from s_N = m_N c_N, exact for K > N too; sum_r s_r = U(all). */
/* Bytes of scratch rd_knn_shapley needs for chunks of queries_per_chunk queries (0 for sizes it refuses). */
size_t rd_knn_shapley_scratch_bytes(int64_t n_train, int32_t ld, int32_t queries_per_chunk);
/* values [n_train] (+)= sum_q s^(q) (fp64, device), the queries added one at a time in query index order, so the result
 * is bitwise independent of queries_per_chunk and of how a query set is split across accumulating calls (accumulate != 0
 * adds to the values stored, else they are overwritten).  per_query [n_query, n_train] (fp64; NULL: skipped) = s^(q) in
 * record order; utility [n_query] (fp64; NULL: skipped) = U_q(all).  bank [n_train, ld] and queries [n_query, ld]: the
 * normalised fp32 rows with zero columns up to ld (a multiple of 4; both 16-byte aligned); y_train [n_train] and y_query
 * [n_query] int64 labels.  self_offset >= 0: query q is training record self_offset + q and is left out of its own
 * ranking (N = n_train - 1, s = 0 at its own record); -1: no exclusion (N = n_train).  Per chunk: one DMMA launch of the
 * similarities as descending-order 64-bit keys (every element over the same k-order, so identical rows get identical
 * similarities), one CTA per query for a stable LSD radix sort (eight 8-bit passes through scratch, the index as payload)
 * and the suffix sums in a fixed order, then one thread per record adds the chunk's rows in order.  Refused with -2
 * before any launch: k < 1, n_train outside [1, 2^31), fewer than 2 records with self_offset >= 0, a self range outside
 * the bank, a NULL required pointer, misaligned pointers (scratch 256-byte aligned).  Non-finite rows rank after every
 * number (the Python layer refuses them).  Stream-ordered, allocation- and sync-free, CUDA-graph capturable. */
int rd_knn_shapley(const float* bank, int64_t n_train, int32_t ld, const int64_t* y_train, const float* queries,
                   int64_t n_query, const int64_t* y_query, int32_t k, int64_t self_offset, int32_t queries_per_chunk,
                   int32_t accumulate, void* scratch, double* values, double* per_query, double* utility, void* stream);
/* debug: the ranking of rd_knn_shapley as one chunk of n_query queries (scratch: rd_knn_shapley_scratch_bytes(n_train,
 * ld, n_query)): order [n_query, n_train] int64 = the records in ranked order (with self_offset >= 0 the query's own
 * record last), sim [n_query, n_train] fp64 = each record's similarity, read back from its sort key (NaN at the query's
 * own record). */
int rd_debug_knn_rank(const float* bank, int64_t n_train, int32_t ld, const float* queries, int64_t n_query,
                      int64_t self_offset, void* scratch, double* sim, int64_t* order, void* stream);

/* ---- Laplace approximation (MacKay 1992; Ritter et al. 2018; Daxberger et al. 2021) ----------------------------------
 * Posterior N(theta*, H^-1), H = n F + delta I with F the EK-FAC Fisher above: diagonal in the Kronecker eigenbasis,
 * n Lambda_j + delta.  The linearised predictive of sample b is f ~ N(f(x_b; theta*), Sigma_b) over its logits, with
 *   Sigma_b[c, c'] = sum_j w_j J~_{b,c,j} J~_{b,c',j},   w_j = 1 / (n Lambda_j + delta) (0 off the selected fields),
 * J~_{b,c} = the rotated gradient row of logit c (rd_raindrop_v2_ekfac_rows seeded with d_logits = e_c / B).
 * At most RD_LAPLACE_MAX_CLASSES classes. */
#define RD_LAPLACE_MAX_CLASSES 8
/* Scratch of rd_raindrop_v2_laplace_logit_cov: the rows scratch of rd_raindrop_v2_ekfac_rows, the seed d_logits [B, C],
 * the rows [C, B, bucket] fp32 and the Gram's fp64 slab partials [B, ceil(bucket / 16384), C (C + 1) / 2]; 0 for dims
 * it refuses. */
size_t rd_laplace_logit_cov_scratch_bytes(const rd_dims* dims);
/* cov [B, C, C] (fp64, device) = Sigma_b of every sample of the batch whose eval rd_raindrop_v2_fwd (without labels) left
 * `workspace`.  Per class c: one seed launch (d_logits = e_c / B on the device), the rotated rows of
 * rd_raindrop_v2_ekfac_rows into the scratch (bases as there); then one Gram launch over (16384-column slab, sample)
 * CTAs, products w_j J~_cj in fp32 times J~_c'j in fp32, summed in fp64 per thread in column order, across the CTA in a
 * fixed tree, and one launch adding the slabs in order: no atomics, so a sample's Sigma_b is bitwise reproducible and
 * depends on its own rows only.  w: fp32 [bucket] on the device, 16-byte aligned (0 outside the selected fields and on
 * padding).  Stream-ordered, allocation- and sync-free, CUDA-graph capturable. */
int rd_raindrop_v2_laplace_logit_cov(const rd_dims* dims, const rd_params* params, const float* statics,
                                     const int64_t* lengths, const float* node_scale, const void* workspace,
                                     const float* bases, const float* w, void* scratch, double* cov, void* stream);
/* Relative pivot tolerance of the predictive's Cholesky factor: a pivot <= RD_LAPLACE_PIVOT_TOL * trace(Sigma_b) counts
 * as 0 and its column of L_b is zeroed, so positive semi-definite Sigma_b (a class whose logit has no gradient in the
 * selected fields, or an all-zero Sigma_b) is factorised without NaN. */
#define RD_LAPLACE_PIVOT_TOL 1e-12
/* Scratch of rd_laplace_predictive_mc: L_b [B, C, C] fp64, the fp64 sums of mc_dropout's reduction and one chunk's
 * logits [samples_per_chunk, B, C] fp32; 0 for sizes it refuses. */
size_t rd_laplace_sample_scratch_bytes(int32_t B, int32_t n_classes, int32_t samples_per_chunk);
/* Monte Carlo predictive of the linearised Laplace posterior: replicate m = 0 .. n_samples-1 draws for every sample b
 *   f_{m,b} = mean_logits[b] + L_b eps_{m,b}   (fp64, rounded to fp32 once)
 * with L_b the lower Cholesky factor of cov[b] (fp64, pivots as RD_LAPLACE_PIVOT_TOL says) and eps_{m,b,k} a standard
 * normal from the Philox4x32-10 stream of the dropout masks with key {seed, step + m} (rng = {seed, step}, device
 * uint64[2], read only), site 99 (96: DP noise, 97: Fisher labels, 98: PGD start), element index e = b*C + k: counter
 * e >> 2, Box-Muller on the block's word pairs as rd_dp_add_noise (e & 3 in {0, 1}: words (x, y), {2, 3}: (z, w); even e
 * takes the cosine, odd e the sine).  A draw depends on (seed, step + m, b, k) alone, not on B or the chunking.  The
 * replicates are reduced as rd_raindrop_v2_mc_dropout reduces its replicates (the same launch): mean_probs [B, C],
 * variance [B, C], entropies [3, B], samples [M, B, C] (optional, may be NULL).  Work: one Cholesky launch, then per
 * chunk of samples_per_chunk replicates one draw launch and one reduction launch (fp64 sums in replicate order, bitwise
 * independent of the chunking).  mean_logits [B, C] fp32, cov [B, C, C] fp64, scratch
 * rd_laplace_sample_scratch_bytes(B, C, samples_per_chunk) bytes, 16-byte aligned.  Stream-ordered, allocation- and
 * sync-free, CUDA-graph capturable. */
int rd_laplace_predictive_mc(const float* mean_logits, const double* cov, int32_t B, int32_t n_classes, const uint64_t* rng,
                             int32_t n_samples, int32_t samples_per_chunk, void* scratch, float* mean_probs,
                             float* variance, float* entropies, float* samples, void* stream);

/* ---- SWA / SWAG of Raindrop_v2 (Izmailov et al. 2018; Maddox et al. 2019; MultiSWAG, Wilson & Izmailov 2020) ---------
 * theta is a flat fp32 parameter bucket of n floats (n % 4 == 0; TrainStep's layout, padding lanes 0).  A SWAG posterior
 * is the fp64 running moments mean [n], sq_mean [n] of the snapshots collected so far and up to `rank` deviation
 * columns dev [rank, n] fp32 (slot-major: each column is contiguous); with c snapshots, k = min(c, rank) columns hold
 * data.  Every fp64 operation is rounded on its own (no FMA contraction), so a float64 restatement matches bit for bit.
 * Buffers are 16-byte aligned. */
#define RD_SWAG_MAX_RANK 1024
/* Folds snapshot c = n_collected into the moments:
 *   mean' = (c mean + theta) / (c + 1),  sq_mean' = (c sq_mean + theta^2) / (c + 1)   (fp64)
 * and, when rank > 0, writes slot c % rank of dev = fp32(theta - mean') (fp64 difference).  rank = 0 keeps the moments
 * only (SWAG-diagonal; dev may be NULL).  One launch; theta is only read. */
int rd_swag_collect(const float* theta, int64_t n, int64_t n_collected, int32_t rank, double* mean, double* sq_mean,
                    float* dev, void* stream);
/* Draws one weight vector of the posterior (fp64, the slot sum in slot order j = 0 .. k-1):
 *   theta_out = fp32(mean + sqrt(scale) (sqrt(max(sq_mean - mean^2, 0)) z1 + [k >= 2] sum_{j<k} dev[j] z2_j / sqrt(k - 1)))
 * scale = 0.5 is Maddox et al.'s 1/sqrt(2) on both terms; scale = 0 returns fp32(mean).  z is a standard normal of the
 * Philox4x32-10 stream of the dropout masks with key {seed, step + replicate} (rng = {seed, step}, device uint64[2], read
 * only), site 102 (96: DP noise, 97: Fisher labels, 98: PGD start, 99: Laplace, 100: smoothing, 101: ablation): element
 * index i for z1[i] (i < n) and n + j for z2_j, counter index >> 2, Box-Muller on the block's word pairs as
 * rd_dp_add_noise draws them.  Lanes where mean, sq_mean and dev are 0 (the bucket's padding) come out as +0.
 * 0 <= k <= RD_SWAG_MAX_RANK (dev may be NULL when k < 2), scale finite and >= 0, replicate >= 0.  One launch. */
int rd_swag_sample(const double* mean, const double* sq_mean, const float* dev, int64_t n, int32_t k, double scale,
                   const uint64_t* rng, int64_t replicate, float* theta_out, void* stream);
/* One member of a (Multi)SWAG predictive: a posterior as rd_swag_sample reads it. */
typedef struct rd_swag_member {
  const double* mean;
  const double* sq_mean;
  const float* dev;
  int32_t k;
} rd_swag_member;
/* Scratch of rd_raindrop_v2_swag_predictive: the forward workspace and inputs of rows_per_chunk samples, the fp64 sums
 * of mc_dropout's reduction and one replicate's logits [B, C]; 0 for arguments it refuses. */
size_t rd_swag_predictive_scratch_bytes(const rd_dims* dims, int32_t rows_per_chunk);
/* The Bayesian model average of the batch over sampled weights.  Replicate r = member * n_samples + s (M = n_members *
 * n_samples in all) is the eval forward of the batch with the weights theta_s = rd_swag_sample(members[member], scale,
 * rng, replicate = r): one sample launch into theta_s [n], then the eval forward over chunks of rows_per_chunk samples
 * with `params`, whose trained pointers lie in theta_s (R_u and the untrained tensors are the model's), writing the
 * replicate's logits [B, C], then one reduction launch of rd_raindrop_v2_mc_dropout (replicate offset r, total M):
 * mean_probs [B, C], variance [B, C], entropies [3, B] and samples [M, B, C] (optional, may be NULL), defined as there.
 * scale = 0 with n_samples = 1 is the deep ensemble of the members' mean weights.  Eval arithmetic: dims->training must
 * be 0; the model's rng is neither read nor written.  dims->obprop_mode 0 is resolved once from rows_per_chunk rows, so
 * the result is bitwise independent of the chunking.  `members` is a host array of n_members >= 1 entries, read during
 * the call.  scratch: rd_swag_predictive_scratch_bytes(dims, rows_per_chunk) bytes.  Stream-ordered, allocation- and
 * sync-free, CUDA-graph capturable. */
int rd_raindrop_v2_swag_predictive(const rd_dims* dims, const rd_params* params, const float* src, const float* statics,
                                   const float* times, const int64_t* lengths, const float* node_scale,
                                   const rd_swag_member* members, int32_t n_members, double scale, const uint64_t* rng,
                                   int32_t n_samples, float* theta_s, int64_t n, int32_t rows_per_chunk, void* scratch,
                                   float* mean_probs, float* variance, float* entropies, float* samples, void* stream);

/* debug: when `buffer` is non-NULL ([n_ctas][16] uint64 on the device), the tensor-core attention kernels write the
 * SM clock (clock64) of each CTA's start into slot 0 and of its end into slot 12; NULL switches it off. */
int rd_debug_attention_timing(uint64_t* buffer);
/* same for the tensor-core GEMM kernel (rd_linear_fwd, the encoder and ob-prop GEMMs): [n_ctas][8] uint64,
 * %globaltimer at the CTA's entry (slot 5), after its grid dependency wait (0), at the first full stage seen by MMA
 * thread 0 (1), at that thread's last wgmma retired (2), at the epilogue end of MMA warpgroup 0 / 1 (3 / 4) and at the
 * end of thread 0 (7) */
int rd_debug_gemm_timing(uint64_t* buffer);
/* same for the grouped weight-gradient kernel (rd_linear_wgrad_group and the training backward): [n_ctas][16] uint64
 * per launch CTA (at most one per SM), clock64 at the CTA's start (slot 0) and end (1); summed cycles of the producer
 * waiting for an empty stage (2), for its X tile (3), transposing and storing it (4); of MMA thread 0 waiting for a full
 * stage (5) and in its epilogue (6); %globaltimer ns from start to end (7); k-blocks produced (8); the producer's end
 * (9); the producer's cycles issuing the loads of a released stage (10).  Each launch overwrites the buffer. */
int rd_debug_wgrad_timing(uint64_t* buffer);

/* debug: materialise the dropout keep/scale mask (0 or 1/(1-p)) of one dropout site, so tests can
 * replay train-mode forward/backward in the oracle with identical masks.  `site` ids in DESIGN.md. */
int rd_debug_dropout_mask(const uint64_t* rng_captured, uint32_t site, int64_t n, float p, float* out,
                          void* stream);

/* debug: materialise the block out[c * dim + m] = Omega(seed, col0 + c, m) (+1.0f / -1.0f) of rd_grad_projection's
 * projection, c < n_cols, m < dim, so tests can compare it with a host restatement of the mapping. */
int rd_debug_projection_signs(uint64_t seed, int64_t col0, int32_t n_cols, int32_t dim, float* out, void* stream);

/* debug: the noisy inputs of replicates m0 .. m0+nc-1 of rd_raindrop_v2_smooth_counts (same launch, same stream) in its
 * replicate-major layout, row j = (m - m0)*B + b: src_e [T, nc*B, 2N], statics_e [nc*B, d_static] (d_static > 0),
 * times_e [T, nc*B] and lengths_e [nc*B] (each of these two may be NULL: skipped).  Only dims' B, T, N (d_inp) and
 * d_static are read.  With nc = 1 and m0 = 0 it is one Gaussian-augmented copy of the batch at key rng, which is how
 * SmoothingTrainStep draws its noisy batch. */
int rd_debug_smoothing_inputs(const rd_dims* dims, const float* src, const float* statics, const float* times,
                              const int64_t* lengths, const uint8_t* sensor_perturbable, int32_t perturb_static,
                              float sigma, const uint64_t* rng, int64_t m0, int32_t nc, float* src_e, float* statics_e,
                              float* times_e, int64_t* lengths_e, void* stream);

/* debug: the keep table and ablated inputs of replicates m0 .. m0+nc-1 of rd_raindrop_v2_ablation_counts (the same two
 * launches, same stream): keep_table [nc*B, n_players] uint8 (1 = kept; row j = (m - m0)*B + b), src_e, statics_e,
 * times_e and lengths_e as rd_debug_smoothing_inputs lays them out (times_e / lengths_e may be NULL: skipped).  Only
 * dims' B, T, N (d_inp) and d_static are read.  With nc = 1 and m0 = 0 it is one ablated copy of the batch at key rng,
 * which is how AblationTrainStep draws its batch. */
int rd_debug_ablation_inputs(const rd_dims* dims, const float* src, const float* statics, const float* times,
                             const int64_t* lengths, const uint8_t* sensor_player, int32_t n_players, int32_t ablate_static,
                             int32_t ablate_mask, int32_t keep, int32_t exhaustive, const uint64_t* rng, int64_t m0,
                             int32_t nc, uint8_t* keep_table, float* src_e, float* statics_e, float* times_e,
                             int64_t* lengths_e, void* stream);

/* debug: the prefix inputs of rd_raindrop_v2_prefix_logits (the same two launches, same stream) for all n_prefixes = K
 * prefixes at once: cutoffs [K, B] int32, src_e [T, K*B, 2N], statics_e [K*B, d_static] (NULL: skipped), times_e
 * [T, K*B] and lengths_e [K*B], prefix-major (row k*B + b).  rng NULL: the prefixes given by horizons or rows as there.
 * rng = {seed, step} (device uint64[2]): K = 1 and one cutoff per slot drawn on the device from Philox4x32-10 at site
 * 104 (96: DP noise, 97: Fisher labels, 98: PGD start, 99: Laplace, 100: smoothing, 101: ablation, 102: SWAG, 103:
 * counterfactual starts), the 32-bit words (b << 32) + j of key {seed, step}, word index & 3 of the block at counter
 * index >> 2.  With R_b = 1 + the last row with times > 0 (0 if none: the slot keeps its record) and f_b the first: the
 * first word keeps the whole record when it is < floor(p_full 2^32); otherwise r = lo_b + U(R_b - lo_b + 1), U Lemire's
 * unbiased bounded integer with rejection over the next words and lo_b = max(f_b + 1, ceil(min_fraction R_b)), so a
 * drawn prefix keeps row f_b.  rows (optional, [B] int32 in this mode): a slot with rows[b] >= 0 takes cutoff
 * min(rows[b], T) instead.  p_full and min_fraction lie in [0, 1].  Only dims' B, T, N (d_inp) and d_static are read.
 * With K = 1 it is one truncated copy of the batch, which is how PrefixTrainStep draws its batch. */
int rd_debug_prefix_inputs(const rd_dims* dims, const float* src, const float* statics, const float* times,
                           const int64_t* lengths, const float* horizons, const int32_t* rows, int32_t n_prefixes,
                           const uint64_t* rng, double p_full, double min_fraction, int32_t* cutoffs, float* src_e,
                           float* statics_e, float* times_e, int64_t* lengths_e, void* stream);

/* ---- the forward GEMM engines on their own (debug: operator-level tests) -------------------------------------------
 * Fields are grouped by size (pointers, 64-bit, 32-bit) so the layout has no interior padding. */
/* One tc_nt_kernel launch: C[M, N] = epi(A[M, K] . B[N, K]^T), A with row stride lda, B (and B_lo) with row stride K,
 * C with row stride N.  B_lo = B - trunc19(B) selects the error-compensated mode (3xTF32); NULL selects single-pass TF32
 * on operands the caller keeps TF32-representable.  epi = +bias[col] -> relu -> *scale[row % scale_mod] ->
 * *(gate[row * gate_ld + col] > 0 ? gate_scale : 0) -> dropout (site drop_site, index row * N + col, or through the
 * replicate rows rep_B / rep_Bc; keep bits to drop_mask[row * drop_mask_ld + col / 32], bit col % 32, the bits past N of
 * the row's last word zeroed) -> +resid[row * resid_ld + col] -> RN to TF32 (round_out); perm != 0 stores row b*pN + n,
 * col t*4 + k to C[(t*pB + b)*pD + n*4 + k].  Only the epilogue combinations the model uses are instantiated; others are
 * refused.  BN = 0 or n_tiles = 0: the plan of tc_nt_plan, written back into the struct. */
typedef struct rd_debug_tc_nt_args {
  const float* A; const float* B; const float* B_lo; float* C;
  const float* bias; const float* scale; const float* gate; const uint64_t* rng; uint32_t* drop_mask; const float* resid;
  int64_t lda, M, gate_ld, resid_ld;
  int32_t N, K, BN, n_tiles;
  int32_t relu, scale_mod; float gate_scale;
  float drop_p; uint32_t drop_site; int32_t rep_B, rep_Bc, drop_mask_ld;
  int32_t round_out;
  int32_t perm, pB, pN, pD;
} rd_debug_tc_nt_args;
int rd_debug_tc_nt(rd_debug_tc_nt_args* args, void* stream);
/* One call of the CUDA-core GEMM (rd_gemm.cu): C(i, j) = epi(alpha * sum_k A(i, k) B(k, j)) with element strides
 * (ta: A(i, k) = A[k*sAk + i], else A[i*sAi + k]; tb: B(k, j) = B[j*sBj + k], else B[k*sBk + j]), batched over
 * z = zo * nz_inner + zi (offsets s?zo, s?zi), C(i, j) at C[i*sCi + j*sCj].  epi = +bias[j] -> relu ->
 * *rowscale[i % rowscale_mod] -> *(gate[i*gate_ld + j] > 0 ? gate_scale : 0) -> dropout (site drop_site, index i*N + j,
 * or through the replicate rows rep_B / rep_Bc) -> +resid[i*resid_ld + j] -> store (perm != 0: row b*pN + n, col
 * t*pdob + k to C[(t*pB + b)*pD + n*pdob + k]).  asum (optional): asum[i] = sum_k A(i, k).  Split-K (nz = 1): nsplit
 * partial products in `partial` (partial_floats floats), summed in split order; it takes alpha and asum but no other
 * epilogue field and a contiguous C (sCi = N, sCj = 1).  nsplit = 0: the count of gemm_splitk_plan, written back with
 * partial_floats (0 when it is 1); with no `partial` for a plan that needs one the call is refused after the write-back. */
typedef struct rd_debug_gemm_args {
  const float* A; const float* B; float* C; float* asum;
  const float* bias; const float* rowscale; const float* gate; const uint64_t* rng; const float* resid;
  int64_t sAi, sAk, sBk, sBj, sCi, sCj;
  int64_t sAzo, sAzi, sBzo, sBzi, sCzo, sCzi;
  int64_t gate_ld, resid_ld, partial_floats;
  int32_t M, N, K, ta, tb, nz, nz_inner, nsplit;
  float alpha; int32_t relu, rowscale_mod; float gate_scale;
  float drop_p; uint32_t drop_site; int32_t rep_B, rep_Bc;
  int32_t perm, pB, pN, pdob, pD;
} rd_debug_gemm_args;
int rd_debug_gemm_f32(rd_debug_gemm_args* args, float* partial, void* stream);
/* One item of the per-step weight split (split_weights): for w [rows, cols], lo = w - trunc19(w), t = w^T, t_lo =
 * w^T - trunc19(w^T), rn = RN_tf32(w) (ties away from zero), rn_t = rn^T.  Every output but w may be NULL (t and t_lo
 * together). */
int rd_debug_split_weights(const float* w, int32_t rows, int32_t cols, float* lo, float* t, float* t_lo, float* rn,
                           float* rn_t, void* stream);
/* out[j] = sum_{i < rows} x[i*ld + j], j < cols: per chunk of 32 rows in row order, then the chunks in order.
 * scratch: ceil(rows / 32) * cols floats. */
int rd_debug_colsum(const float* x, int64_t rows, int32_t cols, int64_t ld, float* out, float* scratch, void* stream);

/* ---- the weight-gradient launch on its own (debug: operator-level tests) ----------------------------------------------
 * One grouped weight-gradient launch exactly as the training backward issues it: one tc_wgrad_kernel launch over the
 * n <= 12 problems (none when n = 0) and one reduce launch that sums their row splits and the ncs <= 36 column sums.
 * items[i].d_bias may be NULL (no bias gradient); partial_bytes[i] is the size of items[i].partial, which must be at
 * least rd_linear_wgrad_partial_bytes(rows, out_features, in_features) and 16-byte aligned.  A problem the tensor-core
 * kernel does not take (out_features or in_features not a multiple of 4 or below 16, d_out / x not 16-byte aligned, or
 * the tensor-core path switched off with RD_TC_WGRAD=0) is refused: there is no CUDA-core fallback here.
 * RD_TC_WGRAD_BN=<width> forces the tile width as it does for every grouped launch. */
typedef struct rd_debug_colsum_item {          /* out[c] = sum_{s < nsplit} partial[s*stride + c], c < ncols */
  const float* partial; float* out;
  int64_t stride;
  int32_t nsplit, ncols;
} rd_debug_colsum_item;
/* The plan the launch ran: the tile width (0 when n = 0), the group's rows target, and per problem in the caller's
 * order the row split count and the rows per split (a multiple of 32; the last split holds the remainder). */
typedef struct rd_debug_wgrad_plan {
  int32_t BN, rows_target;
  int32_t nsplit[12], rows_per_split[12];
} rd_debug_wgrad_plan;
int rd_debug_wgrad_group(const rd_wgrad_item* items, const uint64_t* partial_bytes, int32_t n,
                         const rd_debug_colsum_item* cs, int32_t ncs, rd_debug_wgrad_plan* plan, void* stream);

/* ---- the per-sample gradient tiles of the linear layers on their own (debug: operator-level tests) --------------------
 * One group of 1 <= n <= 32 linear items exactly as the backward's per-sample modes issue it.  Item i's sample b has the
 * R rows r = b*sstride + t*rstride (t < R) of d_out [., ld_out] (first out_features columns read) and x [., ld_x];
 * its gradient is the [out_features, in_features + 1] product d_out_b^T [x_b | 1].
 *   RD_PS_SQNORMS  one dp_norm_tile_kernel and one dp_norm_finalize_kernel launch: sqnorms[b*nf + fw] = the squared
 *                  Frobenius norm of the weight part, sqnorms[b*nf + fb] = that of the bias column (fp64, device), in
 *                  the item's form: -1 the backward's choice (ghost iff R (out + in + 1) < out (in + 1)), 0 explicit
 *                  (64 x 64 tiles of the product), 1 ghost (64 x 64 tiles of the R x R Gram triangle).  partial: 16
 *                  bytes per CTA, at least 16 * B * (sum over the items of ntiles) bytes (partial_bytes, checked).
 *   RD_PS_ROWS     one psg_tile_kernel launch: G[b*ldg + gw + m*in_features + n] = scale * product[m, n] and
 *                  G[b*ldg + gb + m] = scale * product[m, in_features], each value rounded to fp32 once; no other
 *                  column of G is written (the padding between fields is left as it was).
 *   RD_PS_ROTATED  the same launch with x holding in_features + 1 columns that already include the bias column (the
 *                  EK-FAC rotated [x | 1] Q_A): product = d_out_b^T x_b, no ones column appended.
 * fw / fb / form are read in sqnorms mode only, gw / gb in the rows modes only.  Refused: a NULL pointer, n out of
 * range, an unknown mode or form, B, R, a width or a stride below 1, ld_out below out_features or ld_x below the columns
 * read, field indices outside [0, nf), fields that leave the row of ldg floats, and an undersized partial buffer.  The
 * plan that ran is written back per item: the form (1 ghost), tm, tn and the tiles per sample. */
#define RD_PS_SQNORMS 0
#define RD_PS_ROWS 1
#define RD_PS_ROTATED 2
typedef struct rd_debug_per_sample_item {
  const float* d_out; const float* x;
  int64_t ld_out, ld_x, sstride, rstride;
  int64_t gw, gb;                                  /* rows modes: bucket offsets of the weight and bias fields */
  int32_t R, out_features, in_features;
  int32_t fw, fb, form;                            /* sqnorms mode: field indices and the form */
} rd_debug_per_sample_item;
typedef struct rd_debug_per_sample_plan {
  int32_t ghost, tm, tn, ntiles;
} rd_debug_per_sample_plan;
int rd_debug_per_sample_linear(const rd_debug_per_sample_item* items, int32_t n, int32_t B, int32_t mode, double* sqnorms,
                               int32_t nf, double* partial, uint64_t partial_bytes, float* G, int64_t ldg, float scale,
                               rd_debug_per_sample_plan* plan, void* stream);

/* ---- the encoder's LayerNorm on its own (debug: operator-level tests) -------------------------------------------------
 * Forward (forward != 0): one layernorm_fwd call, y [rows, D] = (x - mean) rstd gamma + beta, stats [rows][2] = {mean,
 * rstd}, rstd = 1 / sqrt(var + eps).  Backward (backward != 0): one layernorm_bwd call on x, stats (the forward's when
 * both run, else the caller's), gamma and dy [rows, D]: dx, and when drop_p > 0 dx_drop = dx times the dropout mask of
 * `site` (keep_bits [rows][keep_ld] words when given, bit j % 32 of word j / 32, read by the fused kernel only; else
 * Philox at index row * D + j with key rng = {seed, step}); its per-CTA partial rows land in scratch [chunks][2][D] and
 * are reduced into dgamma and dbeta [D] by one tc_wgrad_group launch with two column sums and no weight problems, as
 * the training backward's gradient consumer folds them.  Written back: the classes that ran (fwd_class: RD_LN_GENERIC
 * or the vector kernel's float4 per lane RD_LN_VEC1 / 2 / 5; bwd_class: the fused kernel's RD_LN_VEC1 / 2 / 5 or
 * RD_LN_SPLIT_VEC / RD_LN_SPLIT_SCALAR), chunks (the partial rows) and keep_source (RD_LN_KEEP_*, the mask dx_drop
 * took).  Refused: a NULL pointer a half needs, neither half, rows or D below 1, scratch_floats below
 * rd_debug_layernorm_scratch_floats(rows, D), keep_bits with keep_ld below ceil(D / 32), drop_p outside [0, 1), and
 * drop_p > 0 without rng or dx_drop. */
#define RD_LN_GENERIC 0
#define RD_LN_VEC1 1
#define RD_LN_VEC2 2
#define RD_LN_VEC5 5
#define RD_LN_SPLIT_VEC 16
#define RD_LN_SPLIT_SCALAR 17
#define RD_LN_KEEP_NONE 0
#define RD_LN_KEEP_PHILOX 1
#define RD_LN_KEEP_BITS 2
typedef struct rd_debug_layernorm_args {
  const float* x; const float* gamma; const float* beta; float* y; float* stats;
  const float* dy; float* dx; float* dx_drop; const uint64_t* rng; const uint32_t* keep_bits;
  float* scratch; float* dgamma; float* dbeta;
  int64_t rows, scratch_floats;
  int32_t D, keep_ld; float eps, drop_p; uint32_t site;
  int32_t forward, backward;
  int32_t fwd_class, bwd_class, chunks, keep_source;      /* written back */
} rd_debug_layernorm_args;
int64_t rd_debug_layernorm_scratch_floats(int64_t rows, int32_t D);
int rd_debug_layernorm(rd_debug_layernorm_args* args, void* stream);
/* One per-sample LayerNorm launch exactly as the backward's gradient consumer issues it, over the T*B rows r = t*B + b of
 * x, stats and dy (the encoder layout): sample b's gamma gradient is sum_t dy_r (x_r - mean_r) rstd_r, its beta gradient
 * sum_t dy_r.  RD_PS_SQNORMS: one dp_ln_sqnorm_kernel launch, sqnorms[b*nf + fw] and [b*nf + fb] = their squared norms
 * (fp64).  RD_PS_ROWS: one psg_ln_kernel launch, G[b*ldg + gw + d] and G[b*ldg + gb + d] = scale times them, rounded to
 * fp32 once (the rotated modes of the consumer issue the same launch: LayerNorms are not rotated); nothing else of G is
 * written.  Refused: a NULL pointer, an unknown mode, T, B or D below 1, fields outside [0, nf), fields that leave the
 * row of ldg floats. */
int rd_debug_per_sample_layernorm(int32_t mode, const float* x, const float* stats, const float* dy, int32_t T, int32_t B,
                                  int32_t D, double* sqnorms, int32_t nf, int32_t fw, int32_t fb, float* G, int64_t ldg,
                                  int64_t gw, int64_t gb, float scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RAINDROP_B200_H */
