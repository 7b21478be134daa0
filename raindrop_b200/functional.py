"""torch.autograd bindings over the C ABI (librd_b200.so).  PyTorch is plumbing here: it owns the
device memory, the stream and the autograd graph; every number is produced by our CUDA kernels."""
import ctypes as C

import numpy as np
import torch

from . import lib as L

# parameters that take part in the live path, in the order they are passed to the autograd
# Function (state-dict keys of the reference model, SURVEY.md section 8b / 8a18)
_LAYER_KEYS = ["self_attn.in_proj_weight", "self_attn.in_proj_bias", "self_attn.out_proj.weight",
               "self_attn.out_proj.bias", "linear1.weight", "linear1.bias", "linear2.weight",
               "linear2.bias", "norm1.weight", "norm1.bias", "norm2.weight", "norm2.bias"]
_HEAD_FIELDS = [("emb.weight", "emb_weight"), ("emb.bias", "emb_bias"),
                ("mlp_static.0.weight", "mlp0_weight"), ("mlp_static.0.bias", "mlp0_bias"),
                ("mlp_static.2.weight", "mlp2_weight"), ("mlp_static.2.bias", "mlp2_bias")]
_OBPROP_FIELDS = [("ob_propagation.lin_value.weight", "ob1_value_weight"),
                  ("ob_propagation.lin_value.bias", "ob1_value_bias"),
                  ("ob_propagation_layer2.lin_value.weight", "ob2_value_weight"),
                  ("ob_propagation_layer2.lin_value.bias", "ob2_value_bias")]


def used_param_fields(nlayers, static):
    """[(state-dict key, struct field path)] in Function-argument = flat-bucket order.  The order is the order
    in which the backward FINISHES gradients (head, encoder, then the two lin_value pairs), so that the bucket
    splits into a front part that can be all-reduced while the observation-propagation backward still runs
    (SURVEY.md section 8e) and a tail part (`n_obprop_fields` entries)."""
    out = []
    for key, field in _HEAD_FIELDS:
        if not static and key.startswith("emb."):
            continue
        out.append((key, (field,)))
    for l in range(nlayers):
        for k, f in zip(_LAYER_KEYS, L._LAYER_FIELDS):
            out.append(("transformer_encoder.layers.%d.%s" % (l, k), ("layer", l, f)))
    for key, field in _OBPROP_FIELDS:
        out.append((key, (field,)))
    return out


N_OBPROP_FIELDS = len(_OBPROP_FIELDS)


def _set_field(struct, path, value):
    if len(path) == 1:
        setattr(struct, path[0], value)
    else:
        setattr(getattr(struct, path[0])[path[1]], path[2], value)


def pe_timescales(max_len, d_pe=16):
    """max_len ** linspace(0, 1, d_pe/2) in fp64, cast to fp32 (code/models_rd.py:31,34)."""
    return (float(max_len) ** np.linspace(0, 1, d_pe // 2)).astype(np.float32)


class Plan:
    """Everything about one model instance that the kernels need besides the tensors."""

    def __init__(self, d_inp, d_ob, nhead, nhid, nlayers, d_static, n_classes, max_len, dropout, static, d_pe=16, emb_dim=0,
                 obprop=True):
        self.N, self.d_ob, self.nhead, self.nhid, self.nlayers = d_inp, d_ob, nhead, nhid, nlayers
        self.d_pe, self.emb_dim = d_pe, emb_dim
        self.d_static = d_static if static else 0
        self.n_classes, self.T, self.dropout = n_classes, max_len, float(dropout)
        self.static = static
        self.fields = used_param_fields(nlayers, static)
        if not obprop:          # legacy v1: no observation-propagation layers
            self.fields = self.fields[:-N_OBPROP_FIELDS]
        self.timescales = pe_timescales(max_len)
        self.node_scale = None      # [N] device tensor (rd_node_scale)
        self.R_u = None             # [1, N*d_ob] device tensor
        self.rng_state = None       # int64[2] device tensor {seed, counter}
        self.owner = None           # weakref to the module (receives the flat gradient bucket)
        self.obprop_mode = 0        # 0 auto, 1 single-pass TF32, 2 error-compensated 3xTF32 (rd_dims.obprop_mode)
        self.debug_keep_workspace = False   # tests: keep the last forward's workspace for workspace_view()
        self.last_workspace = None
        self.last_dims = None

    def dims(self, B, training):
        key = (B, bool(training), self.obprop_mode)
        cache = self.__dict__.setdefault("_dims_cache", {})
        d = cache.get(key)
        if d is not None:
            return d
        d = cache[key] = self._make_dims(B, training)
        return d

    def _make_dims(self, B, training):
        d = L.RdDims()
        d.B, d.T, d.N, d.d_ob = B, self.T, self.N, self.d_ob
        d.nhead, d.nhid, d.nlayers = self.nhead, self.nhid, self.nlayers
        d.d_static, d.n_classes = self.d_static, self.n_classes
        d.training = 1 if training else 0
        d.dropout_p = self.dropout
        d.ln_eps = 1e-5
        d.obprop_mode = int(self.obprop_mode)
        d.d_pe = 0 if self.d_pe == 16 else int(self.d_pe)
        d.emb_dim = int(self.emb_dim)
        for i, v in enumerate(self.timescales):
            d.pe_timescales[i] = float(v)
        return d


def _as_f32(t):
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


class RaindropV2Function(torch.autograd.Function):
    """logits = Raindrop_v2.forward(...) (code/models_rd.py:278-387) as ONE autograd node:
    rd_raindrop_v2_fwd in forward, rd_raindrop_v2_bwd in backward."""

    @staticmethod
    def forward(ctx, plan, training, src, static, times, lengths, *params):
        lib = L.load()
        if not src.is_cuda:
            raise L.RaindropB200Error("raindrop_b200 runs on CUDA tensors only (no CPU fallback)")
        T, B = src.shape[0], src.shape[1]
        if T != plan.T or src.shape[2] != 2 * plan.N:
            raise ValueError("src must be [max_len=%d, B, 2*d_inp=%d], got %s" % (plan.T, 2 * plan.N, tuple(src.shape)))
        dims = plan.dims(B, training)
        keep = [t if (t.dtype == torch.float32 and t.is_contiguous()) else _as_f32(t) for t in params]
        ptrs = (plan.R_u.data_ptr(),) + tuple(t.data_ptr() for t in keep)
        cached = plan.__dict__.get("_param_struct")
        if cached is not None and cached[0] == ptrs:
            P = cached[1]
        else:
            P = L.RdParams()
            P.R_u = ptrs[0]
            for (key, path), ptr_ in zip(plan.fields, ptrs[1:]):
                _set_field(P, path, ptr_)
            plan.__dict__["_param_struct"] = (ptrs, P)
        sizes = plan.__dict__.setdefault("_ws_bytes", {})
        ws_bytes = sizes.get((B, bool(training), plan.obprop_mode))
        if ws_bytes is None:
            ws_bytes = sizes[(B, bool(training), plan.obprop_mode)] = (lib.rd_workspace_bytes(C.byref(dims)),
                                                     lib.rd_backward_scratch_bytes(C.byref(dims)))
        ws_bytes, sc_bytes = ws_bytes
        if ws_bytes == 0:
            L.check(-2, "rd_workspace_bytes")
        # activation workspace: recycled through a small per-(B, mode) pool (a forward whose backward has not run
        # yet keeps its workspace; everything else reuses the last one instead of a fresh multi-MB allocation)
        pool = plan.__dict__.setdefault("_ws_pool", {}).setdefault((B, bool(training), src.device.index, plan.obprop_mode), [])
        ws = pool.pop() if pool else torch.empty(ws_bytes // 4, dtype=torch.float32, device=src.device)
        logits = torch.empty(B, plan.n_classes, dtype=torch.float32, device=src.device)
        rng = plan.rng_state
        rc = lib.rd_raindrop_v2_fwd(C.byref(dims), C.byref(P), src.data_ptr(), L.ptr(static), times.data_ptr(),
                                    lengths.data_ptr(), plan.node_scale.data_ptr(), L.ptr(rng), ws.data_ptr(),
                                    logits.data_ptr(), None, None, None, L.stream_ptr(src.device))
        L.check(rc, "rd_raindrop_v2_fwd")
        ctx.plan, ctx.dims, ctx.P, ctx.ws, ctx.pool = plan, dims, P, ws, pool
        ctx.keep = (keep, static, lengths, plan.node_scale, plan.R_u)
        ctx.inputs = (src, times) if any(ctx.needs_input_grad[2:5]) else None    # the lift / PE backward read them
        ctx.sc_bytes = sc_bytes
        if plan.debug_keep_workspace:      # parity tests read named activation buffers (workspace_view)
            plan.last_workspace = ws
            plan.last_dims = dims
        elif not any(ctx.needs_input_grad):
            pool.append(ws)                # no backward will come: hand the workspace straight back
            ctx.ws = None
        return logits

    @staticmethod
    def backward(ctx, d_logits):
        lib = L.load()
        plan, dims = ctx.plan, ctx.dims
        if ctx.ws is None:
            raise L.RaindropB200Error("backward called twice (or after a no-grad forward): the activation workspace of "
                                      "this forward has been released; retain_graph is not supported")
        keep, static, lengths, node_scale, _ = ctx.keep
        d_logits = _as_f32(d_logits)
        dev = d_logits.device
        params = keep
        if not any(ctx.needs_input_grad[6:]):
            # frozen parameters (attribution): the data-gradient chain alone, no weight-gradient GEMMs
            scratch = _bwd_scratch(plan, ctx.sc_bytes, dev)
            L.check(lib.rd_raindrop_v2_bwd(C.byref(dims), C.byref(ctx.P), L.ptr(static), lengths.data_ptr(),
                                           node_scale.data_ptr(), ctx.ws.data_ptr(), d_logits.data_ptr(), None,
                                           scratch.data_ptr(), L.BWD_ALL, L.stream_ptr(dev)), "rd_raindrop_v2_bwd")
            d_in = _input_grads(ctx, scratch) if ctx.inputs is not None else (None, None, None)
            _release_workspace(ctx)
            return (None, None) + d_in + (None,) + (None,) * len(params)
        layout = plan.__dict__.get("_grad_layout")
        if layout is None:      # tightly packed flat bucket, one offset per used parameter
            offs, total = [], 0
            for t in params:
                offs.append(total)
                total += t.numel()
            layout = plan.__dict__["_grad_layout"] = (offs, total)
        offs, total = layout
        owner = plan.owner() if plan.owner is not None else None
        flat = torch.empty(total, dtype=torch.float32, device=dev)
        base = flat.data_ptr()
        cachedG = plan.__dict__.get("_grad_struct")
        if cachedG is not None and cachedG[0] == base:
            G = cachedG[1]
        else:
            G = L.RdGrads()
            for (key, path), off in zip(plan.fields, offs):
                _set_field(G, path, base + 4 * off)
            plan.__dict__["_grad_struct"] = (base, G)
        scratch = _bwd_scratch(plan, ctx.sc_bytes, dev)
        rc = lib.rd_raindrop_v2_bwd(C.byref(dims), C.byref(ctx.P), L.ptr(static), lengths.data_ptr(),
                                    node_scale.data_ptr(), ctx.ws.data_ptr(), d_logits.data_ptr(), C.byref(G),
                                    scratch.data_ptr(), L.BWD_ALL, L.stream_ptr(dev))
        L.check(rc, "rd_raindrop_v2_bwd")
        grads = torch._utils._unflatten_dense_tensors(flat, params)      # views, one C++ call
        if owner is not None:
            owner._flat_grad = flat          # the DDP bucket: one all-reduce covers every gradient
        d_in = _input_grads(ctx, scratch) if ctx.inputs is not None else (None, None, None)
        _release_workspace(ctx)
        return (None, None) + d_in + (None,) + tuple(grads)


def _bwd_scratch(plan, sc_bytes, dev):
    scs = plan.__dict__.setdefault("_scratch", {})
    skey = (sc_bytes, dev.index)
    scratch = scs.get(skey)
    if scratch is None:                  # backward scratch holds nothing across calls: one buffer per size
        scratch = scs[skey] = torch.empty(sc_bytes // 4, dtype=torch.float32, device=dev)
    return scratch


def _release_workspace(ctx):
    if not ctx.plan.debug_keep_workspace:
        ctx.pool.append(ctx.ws)
    ctx.ws = None


def _input_grads(ctx, scratch):
    """(d_src, d_static, d_times) for the inputs that need one (rd_raindrop_v2_input_grad, right after the backward
    that left its activation gradients in `scratch`)."""
    lib = L.load()
    plan, dims = ctx.plan, ctx.dims
    src, times = ctx.inputs
    static, lengths = ctx.keep[1], ctx.keep[2]
    need_src, need_static, need_times = ctx.needs_input_grad[2:5]
    dev = src.device
    d_src = torch.empty_like(src) if need_src else None
    d_times = torch.empty_like(times) if need_times else None
    d_static = torch.empty_like(static) if (need_static and static is not None) else None
    ig = None
    if need_src:
        igs = plan.__dict__.setdefault("_ig_scratch", {})
        key = (src.shape[1], dims.obprop_mode, dev.index)
        ig = igs.get(key)
        if ig is None:
            ig = igs[key] = torch.empty(lib.rd_input_grad_scratch_bytes(C.byref(dims)) // 4, dtype=torch.float32, device=dev)
    L.check(lib.rd_raindrop_v2_input_grad(C.byref(dims), C.byref(ctx.P), src.data_ptr(), times.data_ptr(), lengths.data_ptr(),
                                          ctx.ws.data_ptr(), scratch.data_ptr(), L.ptr(ig), L.ptr(d_src), L.ptr(d_times),
                                          L.ptr(d_static), L.stream_ptr(dev)), "rd_raindrop_v2_input_grad")
    return d_src, d_static, d_times


class _StepSlot:
    """Static buffers + captured CUDA graphs of one (batch size, mode, device) for the flat-bucket fast path."""

    def __init__(self, plan, B, training, dev, flat):
        lib = L.load()
        self.B, self.training, self.dev = B, training, dev
        self.dims = plan.dims(B, training)
        f32 = dict(dtype=torch.float32, device=dev)
        self.src = torch.zeros(plan.T, B, 2 * plan.N, **f32)
        self.times = torch.zeros(plan.T, B, **f32)
        self.lengths = torch.ones(B, dtype=torch.int64, device=dev)
        self.static = torch.zeros(B, plan.d_static, **f32) if plan.static else None
        self.logits = torch.zeros(B, plan.n_classes, **f32)
        self.d_logits = torch.zeros(B, plan.n_classes, **f32)
        ws_bytes = lib.rd_workspace_bytes(C.byref(self.dims))
        if ws_bytes == 0:
            L.check(-2, "rd_workspace_bytes")
        self.ws = torch.empty(ws_bytes // 4, **f32)
        self.scratch = None
        self.P, self.G = L.RdParams(), L.RdGrads()
        self.P.R_u = plan.R_u.data_ptr()
        for (key, path), off in zip(plan.fields, flat.offsets):
            _set_field(self.P, path, flat.flat_p.data_ptr() + 4 * off)
            _set_field(self.G, path, flat.flat_g.data_ptr() + 4 * off)
        self.key = (flat.flat_p.data_ptr(), flat.flat_g.data_ptr(), plan.R_u.data_ptr(), plan.node_scale.data_ptr(),
                    plan.rng_state.data_ptr())
        self.fwd_calls = self.bwd_calls = 0
        self.fwd_graph = self.bwd_graph = None
        self.pending = False          # a forward whose backward has not run yet owns the buffers


def _run_or_capture(slot, which, fn):
    """1st call eager (one-time kernel attribute setup must not happen inside a capture), 2nd call captured,
    afterwards one graph launch per call."""
    graph = getattr(slot, which + "_graph")
    if graph is not None:
        graph.replay()
        return
    calls = getattr(slot, which + "_calls")
    setattr(slot, which + "_calls", calls + 1)
    if calls == 0 or not GRAPHS_ENABLED or torch.cuda.is_current_stream_capturing():
        fn()
        return
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    setattr(slot, which + "_graph", g)
    g.replay()


GRAPHS_ENABLED = True


class RaindropV2FlatFunction(torch.autograd.Function):
    """Same arithmetic as RaindropV2Function for a model whose used parameters live in ONE flat leaf tensor
    (raindrop_b200.optim.FlatAdam).  Inputs are staged into static buffers so that the forward and the backward are
    each ONE CUDA-graph launch; the gradient bucket is written in place (flat_p.grad IS the bucket), so autograd
    has a single leaf to visit and nothing to copy."""

    @staticmethod
    def forward(ctx, plan, training, slot, flat, src, static, times, lengths, flat_p):
        lib = L.load()
        slot.src.copy_(src); slot.times.copy_(times); slot.lengths.copy_(lengths)
        if slot.static is not None:
            slot.static.copy_(static)

        def fwd():
            rc = lib.rd_raindrop_v2_fwd(C.byref(slot.dims), C.byref(slot.P), slot.src.data_ptr(), L.ptr(slot.static),
                                        slot.times.data_ptr(), slot.lengths.data_ptr(), plan.node_scale.data_ptr(),
                                        L.ptr(plan.rng_state), slot.ws.data_ptr(), slot.logits.data_ptr(), None, None, None,
                                        L.stream_ptr(slot.dev))
            L.check(rc, "rd_raindrop_v2_fwd")
        _run_or_capture(slot, "fwd", fwd)
        ctx.plan, ctx.slot, ctx.flat = plan, slot, flat
        slot.pending = bool(ctx.needs_input_grad[-1])
        if plan.debug_keep_workspace:
            plan.last_workspace, plan.last_dims = slot.ws, slot.dims
        return slot.logits.clone()

    @staticmethod
    def backward(ctx, d_logits):
        lib = L.load()
        plan, slot, flat = ctx.plan, ctx.slot, ctx.flat
        if not slot.pending:
            raise L.RaindropB200Error("backward called twice for one forward (retain_graph is not supported)")
        slot.d_logits.copy_(d_logits)
        if slot.scratch is None:
            slot.scratch = torch.empty(lib.rd_backward_scratch_bytes(C.byref(slot.dims)) // 4, dtype=torch.float32,
                                       device=slot.dev)

        def bwd():
            rc = lib.rd_raindrop_v2_bwd(C.byref(slot.dims), C.byref(slot.P), L.ptr(slot.static), slot.lengths.data_ptr(),
                                        plan.node_scale.data_ptr(), slot.ws.data_ptr(), slot.d_logits.data_ptr(),
                                        C.byref(slot.G), slot.scratch.data_ptr(), L.BWD_ALL, L.stream_ptr(slot.dev))
            L.check(rc, "rd_raindrop_v2_bwd")
        _run_or_capture(slot, "bwd", bwd)
        slot.pending = False
        flat.grads_ready = True
        owner = plan.owner() if plan.owner is not None else None
        if owner is not None:
            owner._flat_grad = flat.flat_g
        # flat_p.grad already IS flat_g (written in place by the kernels): nothing for autograd to accumulate
        return (None,) * 9


def flat_forward(plan, training, flat, src, static, times, lengths):
    """Entry of the flat-bucket fast path (models_rd.Raindrop_v2.forward when a FlatAdam is bound)."""
    dev = src.device
    B = src.shape[1]
    if src.shape[0] != plan.T or src.shape[2] != 2 * plan.N:
        raise ValueError("src must be [max_len=%d, B, 2*d_inp=%d], got %s" % (plan.T, 2 * plan.N, tuple(src.shape)))
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (src, static, times)):
        # input gradients come through the general path; its parameter gradients accumulate into the .grad windows of
        # the bucket, so the bucket starts from zero (a backward overwrites the gradients, as on the fast path)
        flat.flat_g.zero_()
        flat.grads_ready = False
        return None
    slots = plan.__dict__.setdefault("_slots", {})
    k = (B, bool(training), dev.index)
    slot = slots.get(k)
    if slot is not None and slot.dims.obprop_mode != plan.obprop_mode:
        slot = None                      # arithmetic mode changed: new workspace layout, new graphs
    key = (flat.flat_p.data_ptr(), flat.flat_g.data_ptr(), plan.R_u.data_ptr(), plan.node_scale.data_ptr(),
           plan.rng_state.data_ptr())
    if slot is None or slot.key != key:      # pointers changed (graph / R_u / optimiser re-created): rebuild
        slot = slots[k] = _StepSlot(plan, B, bool(training), dev, flat)
    if slot.pending:
        if torch.is_grad_enabled():
            raise L.RaindropB200Error("a FlatAdam-bound model keeps ONE forward in flight per batch size: call "
                                      "loss.backward() before the next training forward (for gradient accumulation "
                                      "use torch.optim.Adam)")
        return None      # caller falls back to the general path (e.g. a no-grad probe between forward and backward)
    return RaindropV2FlatFunction.apply(plan, training, slot, flat, src, static, times, lengths, flat.flat_p)


class ObPropLayerFunction(torch.autograd.Function):
    """One observation-propagation layer on `rows` node rows at once (rd_obprop_fwd / _bwd)."""

    @staticmethod
    def forward(ctx, x, weight, bias, node_scale, mod):
        lib = L.load()
        x, weight, bias = _as_f32(x), _as_f32(weight), _as_f32(bias)
        rows, Cc = x.shape
        out = torch.empty_like(x)
        sc = torch.empty(lib.rd_obprop_fwd_scratch_bytes(rows, Cc) // 4, dtype=torch.float32, device=x.device)
        rc = lib.rd_obprop_fwd(x.data_ptr(), weight.data_ptr(), bias.data_ptr(), node_scale.data_ptr(), int(mod),
                               rows, Cc, out.data_ptr(), sc.data_ptr(), L.stream_ptr())
        L.check(rc, "rd_obprop_fwd")
        ctx.save_for_backward(x, weight, out, node_scale)
        ctx.mod = int(mod)
        return out

    @staticmethod
    def backward(ctx, d_out):
        lib = L.load()
        x, weight, out, node_scale = ctx.saved_tensors
        d_out = _as_f32(d_out)
        rows, Cc = x.shape
        d_x = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        d_w = torch.empty_like(weight)
        d_b = torch.empty(Cc, dtype=torch.float32, device=x.device)
        sc = torch.empty(lib.rd_obprop_bwd_scratch_bytes(rows, Cc) // 4, dtype=torch.float32, device=x.device)
        rc = lib.rd_obprop_bwd(x.data_ptr(), out.data_ptr(), d_out.data_ptr(), weight.data_ptr(),
                               node_scale.data_ptr(), ctx.mod, rows, Cc, L.ptr(d_x), d_w.data_ptr(), d_b.data_ptr(),
                               sc.data_ptr(), L.stream_ptr())
        L.check(rc, "rd_obprop_bwd")
        return d_x, d_w, d_b, None, None


def _check_edges(who, edge_index, edge_weights):
    """edge_index must be [2, E] int64 and edge_weights (when given) [E]: the kernels index with them unchecked."""
    if not torch.is_tensor(edge_index) or edge_index.dim() != 2 or edge_index.shape[0] != 2 or edge_index.dtype != torch.int64:
        got = "%s %s" % (tuple(edge_index.shape), edge_index.dtype) if torch.is_tensor(edge_index) else type(edge_index).__name__
        raise L.RaindropB200Error("%s: edge_index must be a [2, E] int64 tensor, got %s" % (who, got))
    E = edge_index.shape[1]
    if edge_weights is not None and (edge_weights.dim() != 1 or edge_weights.shape[0] != E):
        raise L.RaindropB200Error("%s: edge_weights must have shape [E] = [%d] like edge_index, got %s"
                                  % (who, E, tuple(edge_weights.shape)))
    return E


def _check_geom(who, geom, rows):
    """geom = (n_nodes, n_graphs, node_stride, graph_stride) must map (node, graph) one-to-one onto the `rows` rows of x:
    node-major (n_graphs, 1) or graph-major (1, n_nodes).  Anything else would index past the projections."""
    n_nodes, n_graphs, node_stride, graph_stride = (int(v) for v in geom)
    if n_nodes < 1 or n_graphs < 1:
        raise L.RaindropB200Error("%s: geom needs n_nodes >= 1 and n_graphs >= 1, got %s" % (who, tuple(geom)))
    dense = node_stride == 1 if n_graphs == 1 else (node_stride, graph_stride) in ((n_graphs, 1), (1, n_nodes))
    if not dense:
        raise L.RaindropB200Error("%s: geom strides (node_stride, graph_stride) = (%d, %d) are not a dense layout of %d "
                                  "nodes x %d graphs: use (%d, 1) or (1, %d)"
                                  % (who, node_stride, graph_stride, n_nodes, n_graphs, n_graphs, n_nodes))
    if rows != n_nodes * n_graphs:
        raise L.RaindropB200Error("%s: x has %d rows but geom describes n_nodes * n_graphs = %d * %d"
                                  % (who, rows, n_nodes, n_graphs))
    return n_nodes, n_graphs, node_stride, graph_stride


class ObPropBetaFunction(torch.autograd.Function):
    """Observation_progation.forward(use_beta=True) for one sample (code/Ob_propagation.py:161-211) with gradients:
    rd_obprop_beta_fwd / rd_obprop_beta_bwd.  Returns (out [N, C], alpha [K], pruned edge list [2, K] (data))."""

    @staticmethod
    def forward(ctx, x, p_t, edge_weights, src_i, tgt_i, d_ob, inc_w, inc_b, map_w, val_w, val_b):
        lib = L.load()
        x, p_t, w = _as_f32(x), _as_f32(p_t), _as_f32(edge_weights)
        N, Cc = x.shape
        T = Cc // d_ob
        E = src_i.numel()
        K = E // 2
        out = torch.empty(N, Cc, dtype=torch.float32, device=x.device)
        ei = torch.empty(2, K, dtype=torch.int64, device=x.device)
        alpha = torch.empty(K, dtype=torch.float32, device=x.device)
        sc = torch.empty(lib.rd_obprop_beta_scratch_bytes(N, T, d_ob, E) // 4, dtype=torch.float32, device=x.device)
        ps = [_as_f32(t) for t in (inc_w, inc_b, map_w, val_w, val_b)]
        rc = lib.rd_obprop_beta_fwd(x.data_ptr(), p_t.data_ptr(), src_i.data_ptr(), tgt_i.data_ptr(), w.data_ptr(), E, N, T,
                                    d_ob, *[p.data_ptr() for p in ps], out.data_ptr(), ei[0].data_ptr(), ei[1].data_ptr(),
                                    alpha.data_ptr(), sc.data_ptr(), L.stream_ptr(x.device))
        L.check(rc, "rd_obprop_beta_fwd")
        ctx.save_for_backward(x, p_t, w, src_i, tgt_i, *ps)
        ctx.d_ob = d_ob
        ctx.mark_non_differentiable(ei)
        return out, alpha, ei

    @staticmethod
    def backward(ctx, d_out, d_alpha, _d_ei):
        lib = L.load()
        x, p_t, w, src_i, tgt_i, inc_w, inc_b, map_w, val_w, val_b = ctx.saved_tensors
        N, Cc = x.shape
        d_ob = ctx.d_ob
        T, E = Cc // d_ob, src_i.numel()
        dev = x.device
        d_out = _as_f32(d_out) if d_out is not None else torch.zeros(N, Cc, dtype=torch.float32, device=dev)
        d_alpha = None if d_alpha is None else _as_f32(d_alpha)
        f32 = dict(dtype=torch.float32, device=dev)
        d_x = torch.empty(N, Cc, **f32) if ctx.needs_input_grad[0] else None
        d_pt = torch.empty(T, 16, **f32) if ctx.needs_input_grad[1] else None
        d_w = torch.empty(E, **f32)
        g_iw = torch.empty_like(inc_w); g_ib = torch.empty_like(inc_b); g_mw = torch.empty_like(map_w)
        g_vw = torch.empty_like(val_w); g_vb = torch.empty_like(val_b)
        sc = torch.empty(lib.rd_obprop_beta_bwd_scratch_bytes(N, T, d_ob, E) // 4, **f32)
        rc = lib.rd_obprop_beta_bwd(x.data_ptr(), p_t.data_ptr(), src_i.data_ptr(), tgt_i.data_ptr(), w.data_ptr(), E, N, T, d_ob,
                                    inc_w.data_ptr(), inc_b.data_ptr(), map_w.data_ptr(), val_w.data_ptr(), val_b.data_ptr(),
                                    d_out.data_ptr(), L.ptr(d_alpha), L.ptr(d_x), d_w.data_ptr(), L.ptr(d_pt),
                                    g_iw.data_ptr(), g_ib.data_ptr(), g_mw.data_ptr(), g_vw.data_ptr(), g_vb.data_ptr(),
                                    sc.data_ptr(), L.stream_ptr(dev))
        L.check(rc, "rd_obprop_beta_bwd")
        return d_x, d_pt, d_w, None, None, None, g_iw, g_ib, g_mw, g_vw, g_vb


def obprop_beta(x, p_t, edge_index, edge_weights, d_ob, inc_w, inc_b, map_w, val_w, val_b):
    """Observation_progation.forward(use_beta=True) for one sample.  Returns (out [N, C], edge_index_pruned [2, K],
    alpha [K]); differentiable w.r.t. x, p_t, edge_weights and the five parameters."""
    if _check_edges("obprop_beta", edge_index, edge_weights) < 2:
        raise L.RaindropB200Error("obprop_beta: edge_index has E = %d edges, but use_beta keeps the top E // 2 of them "
                                  "and needs E >= 2" % edge_index.shape[1])
    src_i, tgt_i = edge_index[0].contiguous(), edge_index[1].contiguous()
    out, alpha, ei = ObPropBetaFunction.apply(x, p_t, edge_weights, src_i, tgt_i, d_ob, inc_w, inc_b, map_w, val_w, val_b)
    return out, ei, alpha


def node_scale(edge_index, edge_weights, n_nodes):
    """s[n] = sum over incoming edges of the segment softmax (rd_node_scale)."""
    _check_edges("node_scale", edge_index, edge_weights)
    lib = L.load()
    tgt = edge_index[1].contiguous()
    w = _as_f32(edge_weights)
    s = torch.empty(n_nodes, dtype=torch.float32, device=w.device)
    L.check(lib.rd_node_scale(tgt.data_ptr(), w.data_ptr(), tgt.numel(), n_nodes, s.data_ptr(), L.stream_ptr()),
            "rd_node_scale")
    return s


class PositionalEncodingFunction(torch.autograd.Function):
    """pe = [sin(times / ts), cos(times / ts)] (rd_positional_encoding), differentiable in times
    (rd_positional_encoding_bwd)."""

    @staticmethod
    def forward(ctx, t, max_len, d_pe):
        lib = L.load()
        out = torch.empty(t.shape + (d_pe,), dtype=torch.float32, device=t.device)
        ts = (C.c_float * (d_pe // 2))(*[float(v) for v in pe_timescales(max_len, d_pe)])
        L.check(lib.rd_positional_encoding(t.data_ptr(), t.numel(), ts, d_pe, out.data_ptr(), d_pe, 0, L.stream_ptr(t.device)),
                "rd_positional_encoding")
        ctx.save_for_backward(t)
        ctx.ts, ctx.d_pe = ts, d_pe
        return out

    @staticmethod
    def backward(ctx, d_pe):
        lib = L.load()
        (t,) = ctx.saved_tensors
        d_pe = _as_f32(d_pe)
        d_t = torch.empty_like(t)
        L.check(lib.rd_positional_encoding_bwd(t.data_ptr(), d_pe.data_ptr(), t.numel(), ctx.ts, ctx.d_pe, ctx.d_pe, 0,
                                               d_t.data_ptr(), L.stream_ptr(t.device)), "rd_positional_encoding_bwd")
        return d_t, None, None


def positional_encoding(times, max_len, d_pe=16):
    """[T, B] -> [T, B, d_pe] on the device (rd_positional_encoding); d_pe even, <= 64.  Differentiable in times."""
    return PositionalEncodingFunction.apply(_as_f32(times), max_len, d_pe)


def linear(x, weight, bias=None, relu=False):
    """x [rows, in] -> [rows, out] through the encoder's projection GEMM (rd_linear_fwd); inference only."""
    lib = L.load()
    x, weight = _as_f32(x), _as_f32(weight)
    rows, in_f = x.shape
    out_f = weight.shape[0]
    out = torch.empty(rows, out_f, dtype=torch.float32, device=x.device)
    sc = torch.empty(lib.rd_linear_scratch_bytes(in_f, out_f) // 4, dtype=torch.float32, device=x.device)
    b = None if bias is None else _as_f32(bias)
    L.check(lib.rd_linear_fwd(x.data_ptr(), weight.data_ptr(), L.ptr(b), rows, in_f, out_f, int(relu), out.data_ptr(),
                              sc.data_ptr(), L.stream_ptr()), "rd_linear_fwd")
    return out


class TransformerConvFunction(torch.autograd.Function):
    """TransformerConv.forward (code/transformer_conv.py:139-207) with gradients: rd_transformer_conv_fwd / _bwd.
    x [rows, in] holds `n_graphs` graphs of `n_nodes` nodes sharing one edge list; row(node i, graph g) =
    i * node_stride + g * graph_stride.  Returns (out [rows, H*F], alpha [n_graphs, E, H])."""

    @staticmethod
    def forward(ctx, x, edge_index, edge_weights, geom, heads, out_channels, wq, bq, wk, bk, wv, bv, ws, bs):
        E = _check_edges("transformer_conv", edge_index, edge_weights)
        n_nodes, n_graphs, node_stride, graph_stride = geom = _check_geom("transformer_conv", geom, x.shape[0])
        lib = L.load()
        x = _as_f32(x)
        rows, in_ch = x.shape
        src_i = edge_index[0].contiguous()
        tgt_i = edge_index[1].contiguous()
        ew = None if edge_weights is None else _as_f32(edge_weights)
        out = torch.empty(rows, heads * out_channels, dtype=torch.float32, device=x.device)
        alpha = torch.empty(n_graphs, E, heads, dtype=torch.float32, device=x.device)
        sc = torch.empty(max(1, lib.rd_transformer_conv_scratch_bytes(n_nodes, n_graphs, in_ch, heads, out_channels, E, 0) // 4),
                         dtype=torch.float32, device=x.device)
        ps = [_as_f32(t) for t in (wq, bq, wk, bk, wv, bv, ws, bs)]
        rc = lib.rd_transformer_conv_fwd(x.data_ptr(), n_nodes, n_graphs, node_stride, graph_stride, in_ch, heads, out_channels,
                                         src_i.data_ptr(), tgt_i.data_ptr(), L.ptr(ew), E, *[p.data_ptr() for p in ps],
                                         out.data_ptr(), alpha.data_ptr(), sc.data_ptr(), L.stream_ptr(x.device))
        L.check(rc, "rd_transformer_conv_fwd")
        ctx.save_for_backward(x, src_i, tgt_i, alpha, *ps)
        ctx.ew = ew
        ctx.geom, ctx.heads, ctx.out_channels = geom, heads, out_channels
        ctx.mark_non_differentiable(alpha)       # the reference only ever uses the returned alpha as data (detached by cdist/mean)
        return out, alpha

    @staticmethod
    def backward(ctx, d_out, _d_alpha):
        lib = L.load()
        x, src_i, tgt_i, alpha, wq, bq, wk, bk, wv, bv, ws, bs = ctx.saved_tensors
        n_nodes, n_graphs, node_stride, graph_stride = ctx.geom
        heads, F_ = ctx.heads, ctx.out_channels
        rows, in_ch = x.shape
        E = src_i.numel()
        d_out = _as_f32(d_out)
        dev = x.device
        d_x = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        gw = [torch.empty(heads * F_, in_ch, dtype=torch.float32, device=dev) for _ in range(4)]
        gb = [torch.empty(heads * F_, dtype=torch.float32, device=dev) for _ in range(4)]
        d_ew = torch.zeros(E, dtype=torch.float32, device=dev) if (ctx.ew is not None and ctx.needs_input_grad[2]) else None
        sc = torch.empty(max(1, lib.rd_transformer_conv_scratch_bytes(n_nodes, n_graphs, in_ch, heads, F_, E, 1) // 4),
                         dtype=torch.float32, device=dev)
        rc = lib.rd_transformer_conv_bwd(x.data_ptr(), n_nodes, n_graphs, node_stride, graph_stride, in_ch, heads, F_,
                                         src_i.data_ptr(), tgt_i.data_ptr(), L.ptr(ctx.ew), E, wq.data_ptr(), bq.data_ptr(),
                                         wk.data_ptr(), bk.data_ptr(), wv.data_ptr(), bv.data_ptr(), ws.data_ptr(),
                                         alpha.data_ptr(), d_out.data_ptr(), L.ptr(d_x), gw[0].data_ptr(), gb[0].data_ptr(),
                                         gw[1].data_ptr(), gb[1].data_ptr(), gw[2].data_ptr(), gb[2].data_ptr(), gw[3].data_ptr(),
                                         gb[3].data_ptr(), L.ptr(d_ew), sc.data_ptr(), L.stream_ptr(dev))
        L.check(rc, "rd_transformer_conv_bwd")
        return (d_x, None, d_ew, None, None, None, gw[0], gb[0], gw[1], gb[1], gw[2], gb[2], gw[3], gb[3])


def transformer_conv(x, edge_index, edge_weights, heads, out_channels, wq, bq, wk, bk, wv, bv, ws, bs, geom=None):
    """TransformerConv forward with autograd (code/transformer_conv.py:139-207).  Returns (out, alpha); alpha is
    [E, heads] for a single graph, [n_graphs, E, heads] when `geom` = (n_nodes, n_graphs, node_stride, graph_stride)."""
    single = geom is None
    if single:
        geom = (x.shape[0], 1, 1, 0)
    out, alpha = TransformerConvFunction.apply(x, edge_index, edge_weights, geom, heads, out_channels, wq, bq, wk, bk, wv, bv, ws, bs)
    return out, (alpha[0] if single else alpha)


class LinearFunction(torch.autograd.Function):
    """y = x W^T + b on the error-compensated tensor-core GEMM (rd_linear_fwd); backward: dX through the same kernel
    against W^T, dW / db through the grouped weight-gradient kernel (rd_linear_wgrad_group)."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        return linear(x, weight, bias)

    @staticmethod
    def backward(ctx, dy):
        lib = L.load()
        x, weight = ctx.saved_tensors
        dy = _as_f32(dy)
        dx = linear(dy, weight.t().contiguous()) if ctx.needs_input_grad[0] else None
        rows, out_f = dy.shape
        in_f = x.shape[1]
        dW = torch.empty_like(weight)
        db = torch.empty(out_f, dtype=torch.float32, device=dy.device)
        part = torch.empty(max(1, lib.rd_linear_wgrad_partial_bytes(rows, out_f, in_f) // 4), dtype=torch.float32, device=dy.device)
        it = (L.RdWgradItem * 1)()
        it[0].d_out, it[0].x, it[0].rows, it[0].out_features, it[0].in_features = dy.data_ptr(), _as_f32(x).data_ptr(), rows, out_f, in_f
        it[0].d_weight, it[0].d_bias, it[0].partial = dW.data_ptr(), db.data_ptr(), part.data_ptr()
        L.check(lib.rd_linear_wgrad_group(it, 1, L.stream_ptr(dy.device)), "rd_linear_wgrad_group")
        return dx, dW, (db if ctx.has_bias else None)


class DropoutFunction(torch.autograd.Function):
    """nn.Dropout on the library's counter-based stream (rd_dropout); the backward re-applies the same mask."""

    @staticmethod
    def forward(ctx, x, p, rng, site):
        lib = L.load()
        x = _as_f32(x)
        y = torch.empty_like(x)
        L.check(lib.rd_dropout(x.data_ptr(), x.numel(), p, rng.data_ptr(), site, y.data_ptr(), L.stream_ptr(x.device)), "rd_dropout")
        ctx.p, ctx.site = p, site
        ctx.save_for_backward(rng)
        return y

    @staticmethod
    def backward(ctx, dy):
        lib = L.load()
        (rng,) = ctx.saved_tensors
        dy = _as_f32(dy)
        dx = torch.empty_like(dy)
        L.check(lib.rd_dropout(dy.data_ptr(), dy.numel(), ctx.p, rng.data_ptr(), ctx.site, dx.data_ptr(), L.stream_ptr(dy.device)),
                "rd_dropout")
        return dx, None, None, None


class EncoderHeadFunction(torch.autograd.Function):
    """Temporal encoder + masked-mean pooling + mlp_static on a given encoder input z0 [T, B, D] (rd_encoder_head_fwd /
    _bwd): the part of the model that legacy Raindrop v1 shares with Raindrop_v2 (code/models_rd.py:168-191)."""

    @staticmethod
    def forward(ctx, plan, training, z0, static, lengths, *params):
        lib = L.load()
        z0 = _as_f32(z0)
        T, B, D = z0.shape
        dims = plan.dims(B, training)
        keep = [_as_f32(t) for t in params]
        P = L.RdParams()
        for (key, path), t in zip(plan.fields, keep):
            _set_field(P, path, t.data_ptr())
        ws = torch.empty(lib.rd_workspace_bytes(C.byref(dims)) // 4, dtype=torch.float32, device=z0.device)
        n = C.c_int64(0)
        off = lib.rd_workspace_offset(C.byref(dims), L.WS_ENC_IN, C.byref(n))
        if off < 0 or n.value != z0.numel():
            raise L.RaindropB200Error("encoder input must be [T=%d, B, D=%d], got %s" % (plan.T, n.value // max(1, T * B), tuple(z0.shape)))
        ws[off // 4: off // 4 + n.value].copy_(z0.reshape(-1))
        logits = torch.empty(B, plan.n_classes, dtype=torch.float32, device=z0.device)
        rc = lib.rd_encoder_head_fwd(C.byref(dims), C.byref(P), L.ptr(static), lengths.data_ptr(), L.ptr(plan.rng_state),
                                     ws.data_ptr(), logits.data_ptr(), None, None, None, L.stream_ptr(z0.device))
        L.check(rc, "rd_encoder_head_fwd")
        ctx.plan, ctx.dims, ctx.P, ctx.ws, ctx.keep = plan, dims, P, ws, (keep, static, lengths)
        ctx.shape = (T, B, D)
        return logits

    @staticmethod
    def backward(ctx, d_logits):
        lib = L.load()
        plan, dims = ctx.plan, ctx.dims
        keep, static, lengths = ctx.keep
        d_logits = _as_f32(d_logits)
        dev = d_logits.device
        offs, total = [], 0
        for t in keep:
            offs.append(total)
            total += t.numel()
        need_params = any(ctx.needs_input_grad[5:])
        flat = torch.empty(total, dtype=torch.float32, device=dev)
        G = L.RdGrads()
        for (key, path), off in zip(plan.fields, offs):
            _set_field(G, path, flat.data_ptr() + 4 * off)
        sc = torch.empty(lib.rd_backward_scratch_bytes(C.byref(dims)) // 4, dtype=torch.float32, device=dev)
        dz = torch.empty(ctx.shape, dtype=torch.float32, device=dev)
        rc = lib.rd_encoder_head_bwd(C.byref(dims), C.byref(ctx.P), L.ptr(static), lengths.data_ptr(), ctx.ws.data_ptr(),
                                     d_logits.data_ptr(), C.byref(G) if need_params else None, sc.data_ptr(), dz.data_ptr(),
                                     L.stream_ptr(dev))
        L.check(rc, "rd_encoder_head_bwd")
        d_static = None
        if ctx.needs_input_grad[3] and static is not None:
            d_static = torch.empty_like(static)
            L.check(lib.rd_raindrop_v2_input_grad(C.byref(dims), C.byref(ctx.P), None, None, None, ctx.ws.data_ptr(),
                                                  sc.data_ptr(), None, None, None, d_static.data_ptr(), L.stream_ptr(dev)),
                    "rd_raindrop_v2_input_grad")
        grads = torch._utils._unflatten_dense_tensors(flat, keep) if need_params else (None,) * len(keep)
        ctx.ws = None
        return (None, None, dz, d_static, None) + tuple(grads)


def workspace_view(plan, which):
    """Named activation buffer of the most recent forward (parity tests)."""
    lib = L.load()
    n = C.c_int64(0)
    off = lib.rd_workspace_offset(C.byref(plan.last_dims), which, C.byref(n))
    if off < 0:
        L.check(-2, "rd_workspace_offset")
    return plan.last_workspace[off // 4: off // 4 + n.value]
