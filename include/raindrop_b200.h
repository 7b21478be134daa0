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
 * For saliency maps, integrated gradients and other attribution methods, and for adversarial training.  Call it
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
 * (host arrays, n_seg <= 65535, offsets % 4 == 0, 1 <= length <= RD_GRAD_DOT_SEGMENT, inside the row).  A segment's
 * last 32-column block may reach past its end: those columns of Gq are read and multiplied by 0, so the rows must be
 * finite.  One psg_lo launch (the remainder image), one launch of wgmma 3xTF32 tiles over (64 queries, 128 train rows, segment), each segment summed in
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

/* debug: when `buffer` is non-NULL ([n_ctas][16] uint64 on the device), the tensor-core attention kernels write the
 * SM clock (clock64) of each CTA's start into slot 0 and of its end into slot 12; NULL switches it off. */
int rd_debug_attention_timing(uint64_t* buffer);
/* same for the tensor-core GEMM kernel (rd_linear_fwd, the encoder and ob-prop GEMMs): [n_ctas][8] uint64,
 * %globaltimer at the CTA's start (slot 0) and end (slot 7) */
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

#ifdef __cplusplus
}
#endif
#endif /* RAINDROP_B200_H */
