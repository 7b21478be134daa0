"""ctypes binding of librd_b200.so (the C ABI declared in include/raindrop_b200.h).

The library is built in-tree by `raindrop_b200/csrc/build.sh` (see __graft_entry__.build) and is
the ONLY compute path: if it is missing or a call fails, we raise -- there is no CPU fallback.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "librd_b200.so")

RD_MAX_LAYERS = 8
ABI_VERSION = 2
BWD_ENCODER, BWD_OBPROP, BWD_ALL = 1, 2, 3
RD_D_PE = 16
GRAD_DOT_SEGMENT = 4096     # RD_GRAD_DOT_SEGMENT
LAPLACE_MAX_CLASSES = 8     # RD_LAPLACE_MAX_CLASSES
LAPLACE_PIVOT_TOL = 1e-12   # RD_LAPLACE_PIVOT_TOL
ABLATION_MAX_PLAYERS = 4096  # RD_ABLATION_MAX_PLAYERS
SENSOR_ATTACK_MAX_BEAM = 32  # RD_SENSOR_ATTACK_MAX_BEAM
SENSOR_ATTACK_MAX_REMOVED = 32  # RD_SENSOR_ATTACK_MAX_REMOVED
OOD_MAX_K = 256             # RD_OOD_MAX_K
OOD_POOLED, OOD_HIDDEN = 0, 1   # enum rd_ood_layer
SWAG_MAX_RANK = 1024        # RD_SWAG_MAX_RANK
TRAK_DIM_MAX = 8192         # RD_TRAK_DIM_MAX
ACTIVE_MAX_CLASSES = 8      # RD_ACTIVE_MAX_CLASSES
ACTIVE_MAX_REPLICATES = 1024  # RD_ACTIVE_MAX_REPLICATES
ACTIVE_MAX_CONFIGS = 65536  # RD_ACTIVE_MAX_CONFIGS
REMOVAL_MAX_PLAYERS = 16384  # RD_REMOVAL_MAX_PLAYERS
REMOVAL_DESCENDING, REMOVAL_ASCENDING, REMOVAL_ABSOLUTE = 0, 1, 2   # RD_REMOVAL_*
REMOVAL_SUMMARIES = REMOVAL_MOMENTS = 6   # RD_REMOVAL_SUMMARIES, RD_REMOVAL_MOMENTS

# enum rd_ws_buffer
WS_X0, WS_H1, WS_ENC_IN, WS_ENC_OUT, WS_FEAT, WS_RNG, WS_HEAD_HIDDEN = range(7)
WS_FFN = 7                  # + layer index: one view per encoder layer

# dropout site ids (rd_common.cuh: DropSite)
SITE_LIFT, SITE_ATTN, SITE_RESID1, SITE_FFN, SITE_RESID2 = 1, 16, 32, 48, 64

c_float_p = C.c_void_p  # device pointers travel as integers


class RdDims(C.Structure):
    _fields_ = [("B", C.c_int32), ("T", C.c_int32), ("N", C.c_int32), ("d_ob", C.c_int32),
                ("nhead", C.c_int32), ("nhid", C.c_int32), ("nlayers", C.c_int32),
                ("d_static", C.c_int32), ("n_classes", C.c_int32), ("training", C.c_int32),
                ("dropout_p", C.c_float), ("ln_eps", C.c_float),
                ("pe_timescales", C.c_float * (RD_D_PE // 2)), ("d_pe", C.c_int32), ("emb_dim", C.c_int32),
                ("obprop_mode", C.c_int32)]


_LAYER_FIELDS = ["in_proj_weight", "in_proj_bias", "out_proj_weight", "out_proj_bias",
                 "linear1_weight", "linear1_bias", "linear2_weight", "linear2_bias",
                 "norm1_weight", "norm1_bias", "norm2_weight", "norm2_bias"]


class RdLayer(C.Structure):
    _fields_ = [(f, C.c_void_p) for f in _LAYER_FIELDS]


class RdParams(C.Structure):
    _fields_ = [("R_u", C.c_void_p), ("emb_weight", C.c_void_p), ("emb_bias", C.c_void_p),
                ("ob1_value_weight", C.c_void_p), ("ob1_value_bias", C.c_void_p),
                ("ob2_value_weight", C.c_void_p), ("ob2_value_bias", C.c_void_p),
                ("mlp0_weight", C.c_void_p), ("mlp0_bias", C.c_void_p),
                ("mlp2_weight", C.c_void_p), ("mlp2_bias", C.c_void_p),
                ("layer", RdLayer * RD_MAX_LAYERS)]


class RdGrads(C.Structure):
    _fields_ = [("emb_weight", C.c_void_p), ("emb_bias", C.c_void_p),
                ("ob1_value_weight", C.c_void_p), ("ob1_value_bias", C.c_void_p),
                ("ob2_value_weight", C.c_void_p), ("ob2_value_bias", C.c_void_p),
                ("mlp0_weight", C.c_void_p), ("mlp0_bias", C.c_void_p),
                ("mlp2_weight", C.c_void_p), ("mlp2_bias", C.c_void_p),
                ("layer", RdLayer * RD_MAX_LAYERS)]


class RdWgradItem(C.Structure):
    _fields_ = [("d_out", C.c_void_p), ("x", C.c_void_p), ("rows", C.c_int64), ("out_features", C.c_int32),
                ("in_features", C.c_int32), ("d_weight", C.c_void_p), ("d_bias", C.c_void_p), ("partial", C.c_void_p)]


class RdSwagMember(C.Structure):
    _fields_ = [("mean", C.c_void_p), ("sq_mean", C.c_void_p), ("dev", C.c_void_p), ("k", C.c_int32)]


class RdCfOptions(C.Structure):
    _fields_ = [("kappa", C.c_double), ("c_init", C.c_double), ("beta", C.c_float), ("step_size", C.c_float),
                ("init_scale", C.c_float), ("n_search", C.c_int32), ("n_steps", C.c_int32), ("n_restarts", C.c_int32),
                ("perturb_static", C.c_int32)]


class RdDebugTcNtArgs(C.Structure):
    _fields_ = ([(f, C.c_void_p) for f in ("A", "B", "B_lo", "C", "bias", "scale", "gate", "rng", "drop_mask", "resid")] +
                [(f, C.c_int64) for f in ("lda", "M", "gate_ld", "resid_ld")] +
                [(f, C.c_int32) for f in ("N", "K", "BN", "n_tiles", "relu", "scale_mod")] +
                [("gate_scale", C.c_float), ("drop_p", C.c_float), ("drop_site", C.c_uint32)] +
                [(f, C.c_int32) for f in ("rep_B", "rep_Bc", "drop_mask_ld", "round_out", "perm", "pB", "pN", "pD")])


class RdDebugGemmArgs(C.Structure):
    _fields_ = ([(f, C.c_void_p) for f in ("A", "B", "C", "asum", "bias", "rowscale", "gate", "rng", "resid")] +
                [(f, C.c_int64) for f in ("sAi", "sAk", "sBk", "sBj", "sCi", "sCj", "sAzo", "sAzi", "sBzo", "sBzi", "sCzo",
                                          "sCzi", "gate_ld", "resid_ld", "partial_floats")] +
                [(f, C.c_int32) for f in ("M", "N", "K", "ta", "tb", "nz", "nz_inner", "nsplit")] +
                [("alpha", C.c_float), ("relu", C.c_int32), ("rowscale_mod", C.c_int32), ("gate_scale", C.c_float),
                 ("drop_p", C.c_float), ("drop_site", C.c_uint32)] +
                [(f, C.c_int32) for f in ("rep_B", "rep_Bc", "perm", "pB", "pN", "pdob", "pD")])


class RdDebugColsumItem(C.Structure):
    _fields_ = [("partial", C.c_void_p), ("out", C.c_void_p), ("stride", C.c_int64), ("nsplit", C.c_int32),
                ("ncols", C.c_int32)]


class RdDebugWgradPlan(C.Structure):
    _fields_ = [("BN", C.c_int32), ("rows_target", C.c_int32), ("nsplit", C.c_int32 * 12),
                ("rows_per_split", C.c_int32 * 12)]


class RdDebugPerSampleItem(C.Structure):
    _fields_ = ([("d_out", C.c_void_p), ("x", C.c_void_p)] +
                [(f, C.c_int64) for f in ("ld_out", "ld_x", "sstride", "rstride", "gw", "gb")] +
                [(f, C.c_int32) for f in ("R", "out_features", "in_features", "fw", "fb", "form")])


class RdDebugPerSamplePlan(C.Structure):
    _fields_ = [(f, C.c_int32) for f in ("ghost", "tm", "tn", "ntiles")]


RD_PS_SQNORMS, RD_PS_ROWS, RD_PS_ROTATED = 0, 1, 2


class RdDebugLayernormArgs(C.Structure):
    _fields_ = ([(f, C.c_void_p) for f in ("x", "gamma", "beta", "y", "stats", "dy", "dx", "dx_drop", "rng", "keep_bits",
                                           "scratch", "dgamma", "dbeta")] +
                [("rows", C.c_int64), ("scratch_floats", C.c_int64), ("D", C.c_int32), ("keep_ld", C.c_int32),
                 ("eps", C.c_float), ("drop_p", C.c_float), ("site", C.c_uint32)] +
                [(f, C.c_int32) for f in ("forward", "backward", "fwd_class", "bwd_class", "chunks", "keep_source")])


RD_LN_GENERIC, RD_LN_VEC1, RD_LN_VEC2, RD_LN_VEC5, RD_LN_SPLIT_VEC, RD_LN_SPLIT_SCALAR = 0, 1, 2, 5, 16, 17
RD_LN_KEEP_NONE, RD_LN_KEEP_PHILOX, RD_LN_KEEP_BITS = 0, 1, 2


# name -> (restype, argtypes); every symbol include/raindrop_b200.h declares
SIGNATURES = {
    "rd_abi_version": (C.c_int, []),
    "rd_last_error_string": (C.c_char_p, []),
    "rd_launch_count": (C.c_uint64, []),
    "rd_node_scale": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "rd_obprop_fwd_scratch_bytes": (C.c_size_t, [C.c_int64, C.c_int32]),
    "rd_obprop_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64,
                                C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rd_obprop_bwd_scratch_bytes": (C.c_size_t, [C.c_int64, C.c_int32]),
    "rd_obprop_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p]),
    "rd_obprop_beta_scratch_bytes": (C.c_size_t, [C.c_int32] * 4),
    "rd_obprop_beta_fwd": (C.c_int, [C.c_void_p] * 5 + [C.c_int32] * 4 + [C.c_void_p] * 11),
    "rd_obprop_beta_bwd_scratch_bytes": (C.c_size_t, [C.c_int32] * 4),
    "rd_obprop_beta_bwd": (C.c_int, [C.c_void_p] * 5 + [C.c_int32] * 4 + [C.c_void_p] * 5 + [C.c_void_p] * 2 + [C.c_void_p] * 8 +
                           [C.c_void_p, C.c_void_p]),
    "rd_workspace_bytes": (C.c_size_t, [C.POINTER(RdDims)]),
    "rd_backward_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims)]),
    "rd_workspace_offset": (C.c_int64, [C.POINTER(RdDims), C.c_int32, C.POINTER(C.c_int64)]),
    "rd_raindrop_v2_fwd": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams), C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rd_raindrop_v2_bwd": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams), C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(RdGrads), C.c_void_p,
                                     C.c_int32, C.c_void_p]),
    "rd_positional_encoding": (C.c_int, [C.c_void_p, C.c_int64, C.POINTER(C.c_float), C.c_int32, C.c_void_p,
                                         C.c_int64, C.c_int32, C.c_void_p]),
    "rd_positional_encoding_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_float), C.c_int32,
                                             C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]),
    "rd_input_grad_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims)]),
    "rd_raindrop_v2_input_grad": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 10),
    "rd_integrated_gradients_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims), C.c_int32]),
    "rd_raindrop_v2_integrated_gradients": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 10 +
                                            [C.c_int32, C.c_int32] + [C.c_void_p] * 5),
    "rd_coalition_attribution_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims), C.c_int32, C.c_int32]),
    "rd_raindrop_v2_coalition_attribution": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 9 +
                                             [C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32] + [C.c_void_p] * 4),
    "rd_raindrop_v2_cell_coalition_attribution": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 9 +
                                                  [C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
                                                   C.c_int32] + [C.c_void_p] * 4),
    "rd_raindrop_v2_kernel_shap": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 9 +
                                   [C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                    C.c_int32] + [C.c_void_p] * 4),
    "rd_removal_curves_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims), C.c_int32, C.c_int32]),
    "rd_raindrop_v2_removal_curves": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 9 +
                                      [C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                       C.c_int32] + [C.c_void_p] * 8),
    "rd_removal_infidelity_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims), C.c_int32, C.c_int32]),
    "rd_raindrop_v2_removal_infidelity": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 9 +
                                          [C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_double,
                                           C.c_int32, C.c_int32] + [C.c_void_p] * 5),
    "rd_debug_removal_inputs": (C.c_int, [C.POINTER(RdDims)] + [C.c_void_p] * 7 + [C.c_int64, C.c_int64, C.c_int32] +
                                [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_double, C.c_int64, C.c_int32] +
                                [C.c_void_p] * 6),
    "rd_mc_dropout_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims), C.c_int32]),
    "rd_raindrop_v2_mc_dropout": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 6 +
                                  [C.c_int32, C.c_int32] + [C.c_void_p] * 6),
    "rd_pgd_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims), C.c_int32]),
    "rd_raindrop_v2_pgd": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 8 +
                           [C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_int32, C.c_int32, C.c_void_p, C.c_int32] +
                           [C.c_void_p] * 7),
    "rd_counterfactual_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims), C.c_int32, C.c_int32]),
    "rd_raindrop_v2_counterfactual": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 10 +
                                      [C.POINTER(RdCfOptions), C.c_void_p, C.c_int32] + [C.c_void_p] * 11),
    "rd_smooth_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims), C.c_int32]),
    "rd_raindrop_v2_smooth_counts": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 6 +
                                     [C.c_int32, C.c_float, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                      C.c_void_p]),
    "rd_debug_smoothing_inputs": (C.c_int, [C.POINTER(RdDims)] + [C.c_void_p] * 5 + [C.c_int32, C.c_float, C.c_void_p,
                                                                                       C.c_int64, C.c_int32] +
                                  [C.c_void_p] * 5),
    "rd_ablation_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims), C.c_int32, C.c_int32]),
    "rd_raindrop_v2_ablation_counts": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 6 +
                                       [C.c_int32] * 5 + [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                                          C.c_void_p]),
    "rd_debug_ablation_inputs": (C.c_int, [C.POINTER(RdDims)] + [C.c_void_p] * 5 + [C.c_int32] * 5 +
                                 [C.c_void_p, C.c_int64, C.c_int32] + [C.c_void_p] * 6),
    "rd_sensor_attack_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims)] + [C.c_int32] * 4),
    "rd_raindrop_v2_sensor_attack": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 6 +
                                     [C.c_int32] * 3 + [C.c_void_p] * 2 + [C.c_int32] * 4 + [C.c_void_p] * 8),
    "rd_prefix_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims), C.c_int32]),
    "rd_raindrop_v2_prefix_logits": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 7 +
                                     [C.c_int32, C.c_int32] + [C.c_void_p] * 5),
    "rd_debug_prefix_inputs": (C.c_int, [C.POINTER(RdDims)] + [C.c_void_p] * 6 + [C.c_int32, C.c_void_p, C.c_double,
                                                                                    C.c_double] + [C.c_void_p] * 6),
    "rd_ood_features_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims), C.c_int32]),
    "rd_raindrop_v2_features": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 5 +
                                [C.c_int32, C.c_int32] + [C.c_void_p] * 4),
    "rd_feature_moments": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32] +
                           [C.c_void_p] * 4),
    "rd_ood_prepare_bank": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rd_ood_scores_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims), C.c_int32, C.c_int64, C.c_int32, C.c_int32]),
    "rd_raindrop_v2_ood_scores": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 5 + [C.c_int32] +
                                  [C.c_void_p] * 3 + [C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_float,
                                                      C.c_int32] + [C.c_void_p] * 10),
    "rd_encoder_head_fwd": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 9),
    "rd_encoder_head_bwd": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.POINTER(RdGrads), C.c_void_p, C.c_void_p, C.c_void_p]),
    "rd_dropout": (C.c_int, [C.c_void_p, C.c_int64, C.c_float, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]),
    "rd_linear_scratch_bytes": (C.c_size_t, [C.c_int32, C.c_int32]),
    "rd_linear_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                C.c_void_p, C.c_void_p, C.c_void_p]),
    "rd_temporal_attention_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float,
                                            C.c_void_p, C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p]),
    "rd_temporal_attention_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                            C.c_float, C.c_void_p, C.c_uint32, C.c_int32, C.c_void_p, C.c_void_p]),
    "rd_linear_wgrad_partial_bytes": (C.c_size_t, [C.c_int64, C.c_int32, C.c_int32]),
    "rd_linear_wgrad_group": (C.c_int, [C.POINTER(RdWgradItem), C.c_int32, C.c_void_p]),
    "rd_transformer_conv_scratch_bytes": (C.c_size_t, [C.c_int32] * 7),
    "rd_transformer_conv_fwd": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32] + [C.c_void_p] * 8 +
                                [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rd_transformer_conv_bwd": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32] + [C.c_void_p] * 7 +
                                [C.c_void_p] * 2 + [C.c_void_p] * 10 + [C.c_void_p, C.c_void_p]),
    "rd_gather_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_void_p,
                                  C.c_void_p]),
    "rd_assemble_batch": (C.c_int, [C.c_void_p] * 5 + [C.c_int32, C.c_int64, C.c_int32, C.c_int32, C.c_int32] + [C.c_void_p] * 6),
    "rd_feature_stats_scratch_bytes": (C.c_size_t, [C.c_int64, C.c_int32, C.c_int32]),
    "rd_feature_stats": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rd_mask_normalize": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p]),
    "rd_zero_features": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "rd_cross_entropy_fwd_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                           C.c_void_p, C.c_void_p]),
    "rd_adam_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_void_p,
                               C.c_float, C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_void_p]),
    "rd_dp_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims)]),
    "rd_raindrop_v2_per_sample_grad_sqnorms": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 8),
    "rd_dp_clip_scale": (C.c_int, [C.POINTER(RdDims), C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_float] +
                         [C.c_void_p] * 4),
    "rd_dp_add_noise": (C.c_int, [C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_int32, C.c_float,
                                  C.c_void_p, C.c_void_p]),
    "rd_per_sample_grads_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims)]),
    "rd_raindrop_v2_per_sample_grads": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 7 +
                                        [C.c_int64, C.c_void_p]),
    "rd_per_sample_grad_dot_scratch_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int64, C.c_int32]),
    "rd_per_sample_grad_dot": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int64, C.POINTER(C.c_int64),
                                         C.POINTER(C.c_int64), C.c_int32, C.c_double, C.c_void_p, C.c_int64, C.c_void_p,
                                         C.c_void_p]),
    "rd_grad_projection_scratch_bytes": (C.c_size_t, [C.c_int32, C.c_int64, C.c_int32, C.c_int32]),
    "rd_grad_projection": (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                     C.c_int32, C.c_int32, C.c_uint64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "rd_debug_attention_timing": (C.c_int, [C.c_void_p]),
    "rd_debug_gemm_timing": (C.c_int, [C.c_void_p]),
    "rd_debug_wgrad_timing": (C.c_int, [C.c_void_p]),
    "rd_debug_dropout_mask": (C.c_int, [C.c_void_p, C.c_uint32, C.c_int64, C.c_float, C.c_void_p,
                                        C.c_void_p]),
    "rd_debug_projection_signs": (C.c_int, [C.c_uint64, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "rd_debug_tc_nt": (C.c_int, [C.POINTER(RdDebugTcNtArgs), C.c_void_p]),
    "rd_debug_gemm_f32": (C.c_int, [C.POINTER(RdDebugGemmArgs), C.c_void_p, C.c_void_p]),
    "rd_debug_split_weights": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32] + [C.c_void_p] * 6),
    "rd_debug_colsum": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rd_debug_wgrad_group": (C.c_int, [C.POINTER(RdWgradItem), C.POINTER(C.c_uint64), C.c_int32,
                                       C.POINTER(RdDebugColsumItem), C.c_int32, C.POINTER(RdDebugWgradPlan), C.c_void_p]),
    "rd_debug_per_sample_linear": (C.c_int, [C.POINTER(RdDebugPerSampleItem), C.c_int32, C.c_int32, C.c_int32,
                                             C.c_void_p, C.c_int32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int64,
                                             C.c_float, C.POINTER(RdDebugPerSamplePlan), C.c_void_p]),
    "rd_debug_layernorm_scratch_floats": (C.c_int64, [C.c_int64, C.c_int32]),
    "rd_debug_layernorm": (C.c_int, [C.POINTER(RdDebugLayernormArgs), C.c_void_p]),
    "rd_debug_per_sample_layernorm": (C.c_int, [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                                C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                                C.c_int64, C.c_int64, C.c_int64, C.c_float, C.c_void_p]),
    "rd_kfac_factors_doubles": (C.c_int64, [C.POINTER(RdDims)]),
    "rd_ekfac_bases_floats": (C.c_int64, [C.POINTER(RdDims)]),
    "rd_kfac_factors_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims)]),
    "rd_raindrop_v2_kfac_factors": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 8),
    "rd_ekfac_rows_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims)]),
    "rd_raindrop_v2_ekfac_rows": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 8 +
                                  [C.c_int64, C.c_void_p]),
    "rd_ekfac_accumulate_sq": (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                         C.c_int32, C.c_void_p, C.c_void_p]),
    "rd_ekfac_scale_rows": (C.c_int, [C.c_void_p, C.c_int32, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                      C.c_int32, C.c_void_p, C.c_void_p]),
    "rd_fisher_labels": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p]),
    "rd_debug_fisher_uniforms": (C.c_int, [C.c_uint64, C.c_uint64, C.c_int32, C.c_void_p, C.c_void_p]),
    "rd_trak_margin_seed": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32] + [C.c_void_p] * 4),
    "rd_trak_gram": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]),
    "rd_trak_rotate": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rd_batch_bald_scratch_bytes": (C.c_size_t, [C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int64]),
    "rd_batch_bald": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_uint64,
                                C.c_uint64, C.c_int64] + [C.c_void_p] * 6),
    "rd_badge_scratch_bytes": (C.c_size_t, [C.c_int64, C.c_int32, C.c_int32]),
    "rd_badge": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_uint64, C.c_uint64] +
                 [C.c_void_p] * 4),
    "rd_knn_shapley_scratch_bytes": (C.c_size_t, [C.c_int64, C.c_int32, C.c_int32]),
    "rd_knn_shapley": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                 C.c_int32, C.c_int64, C.c_int32, C.c_int32] + [C.c_void_p] * 5),
    "rd_debug_knn_rank": (C.c_int, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64, C.c_int64] +
                          [C.c_void_p] * 4),
    "rd_laplace_logit_cov_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims)]),
    "rd_raindrop_v2_laplace_logit_cov": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 9),
    "rd_laplace_sample_scratch_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    "rd_laplace_predictive_mc": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32] +
                                 [C.c_void_p] * 6),
    "rd_swag_collect": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p]),
    "rd_swag_sample": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_double, C.c_void_p,
                                 C.c_int64, C.c_void_p, C.c_void_p]),
    "rd_swag_predictive_scratch_bytes": (C.c_size_t, [C.POINTER(RdDims), C.c_int32]),
    "rd_raindrop_v2_swag_predictive": (C.c_int, [C.POINTER(RdDims), C.POINTER(RdParams)] + [C.c_void_p] * 5 +
                                       [C.POINTER(RdSwagMember), C.c_int32, C.c_double, C.c_void_p, C.c_int32,
                                        C.c_void_p, C.c_int64, C.c_int32] + [C.c_void_p] * 6),
}

_lib = None


class RaindropB200Error(RuntimeError):
    pass


def load():
    """Loads librd_b200.so (once).  Raises if it has not been built: there is no fallback path."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise RaindropB200Error(
            "%s is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(raindrop_b200/csrc/build.sh).  raindrop_b200 has no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the header and the library disagree
        fn.restype = res
        fn.argtypes = args
    if lib.rd_abi_version() != ABI_VERSION:
        raise RaindropB200Error("ABI version mismatch: %d" % lib.rd_abi_version())
    _lib = lib
    return lib


def check(rc, what):
    if rc != 0:
        msg = load().rd_last_error_string()
        raise RaindropB200Error("%s failed (rc=%d): %s" % (what, rc, msg.decode() if msg else "?"))


def ptr(t):
    """Device pointer of a tensor (0 for None)."""
    return 0 if t is None else t.data_ptr()


def stream_ptr(device=None):
    """cudaStream_t of torch's current stream on `device` (default: the current device)."""
    import torch
    return torch.cuda.current_stream(device).cuda_stream
