"""Training-data influence of Raindrop_v2: TracIn (Pruthi et al. 2020; Captum's TracInCP) with the per-sample gradients
and their inner products computed on the device.

    influence(z_q, z_t) = sum_c lr_c < grad_theta l(z_q; theta_c), grad_theta l(z_t; theta_c) >

l = CrossEntropy of one sample, theta_c = the trained tensors at checkpoint c.  A large positive score marks a training
sample that pushed the query's prediction ("proponent"), a large negative one an "opponent"; a large self-influence
sum_c lr_c ||g_t||^2 marks training samples the model found hard, often mislabelled ones.

    scores = tracin(model, {"src": X, "static": S, "times": t, "lengths": n, "y": None},     # y None: predicted class
                    DeviceDataset(P, Pstatic, Ptime, y), checkpoints=[(sd1, 1e-4), (sd2, 1e-4)])

The gradient rows come from rd_raindrop_v2_per_sample_grads (a data-gradient backward that writes each sample's gradient
in the layout of TrainStep's flat bucket) and are contracted by rd_per_sample_grad_dot (wgmma 3xTF32, fp32 within
segments of at most RD_GRAD_DOT_SEGMENT columns, fp64 across them), so a score is bitwise the same for any chunking.
The model runs in eval arithmetic; the ob-prop layers run in their error-compensated mode unless the model pins the
single-pass mode (obprop_mode 1).  One GPU per call.

TracIn-RP (same paper): project() computes a GradientSketch of a data set once, its rows projected onto `dim` random +-1
directions on the tensor cores (rd_grad_projection, Omega drawn from Philox and never stored); tracin_sketch() scores two
sketches, an unbiased estimate of tracin's scores whose variance falls as 1 / dim.

EK-FAC influence functions (George et al. 2018; Grosse et al. 2023): ekfac_factors() computes the Kronecker-factored
Fisher of every encoder and ob-prop linear layer and its eigenbases once; ekfac_influence() scores
g_q^T (F + lambda I)^-1 g_t with the rows rotated into those bases on the device (rd_raindrop_v2_ekfac_rows).

TRAK (Park et al. 2023): trak_features() projects the margin gradient rows of a training set (per_sample_margin_grads)
as TracIn-RP does, per ensemble member, and computes their fp64 Gram (rd_trak_gram), its eigenbasis and the features
rotated into it (rd_trak_rotate); trak() scores queries against them with the inverse Gram and the training samples'
1 - p weights.
"""
import ctypes as C
import hashlib
import math
from dataclasses import dataclass

import numpy as np
import torch

from . import lib as L
from .attribution import DEFAULT_SCRATCH_BYTES, _Call, _check_call, _largest_chunk

SEGMENT = L.GRAD_DOT_SEGMENT


def grad_layout(model):
    """[(state-dict key, offset, shape)] of the trained tensors in a gradient row (TrainStep's flat bucket: each tensor
    at an offset rounded up to 4 floats)."""
    out, off = [], 0
    for (key, _), p in zip(model._plan.fields, model.used_parameters()):
        out.append((key, off, tuple(p.shape)))
        off += (p.numel() + 3) // 4 * 4
    return out


def _bucket_length(layout):
    key, off, shape = layout[-1]
    return off + (math.prod(shape) + 3) // 4 * 4


def _selected(layout, fields):
    keys = [k for k, _, _ in layout]
    if fields is None:
        return set(keys)
    if isinstance(fields, str):
        raise ValueError("fields must be a list of state-dict keys, not a string")
    sel = list(fields)
    unknown = [k for k in sel if k not in keys]
    if unknown:
        raise ValueError("unknown fields %s: pick from privacy.sqnorm_fields(model)" % unknown)
    if not sel or len(set(sel)) != len(sel):
        raise ValueError("fields must be a non-empty list without repeats")
    return set(sel)


def plan_segments(layout, fields=None):
    """(seg_off, seg_len) int64 arrays: the columns of the selected fields, each field cut into pieces of at most SEGMENT
    columns (every piece starts 4-aligned, since fields and SEGMENT are; no piece crosses a field)."""
    sel = _selected(layout, fields)
    offs, lens = [], []
    for key, off, shape in layout:
        if key not in sel:
            continue
        n = math.prod(shape)
        for s in range(0, n, SEGMENT):
            offs.append(off + s)
            lens.append(min(SEGMENT, n - s))
    return np.asarray(offs, dtype=np.int64), np.asarray(lens, dtype=np.int64)


def _dims(plan, B):
    """Eval dims of B rows with the ob-prop arithmetic pinned (auto -> error-compensated), so it cannot follow B."""
    cache = plan.__dict__.setdefault("_influence_dims", {})
    key = (B, plan.obprop_mode)
    d = cache.get(key)
    if d is None:
        src = plan.dims(B, False)
        d = L.RdDims()
        C.memmove(C.byref(d), C.byref(src), C.sizeof(src))
        if d.obprop_mode == 0:
            d.obprop_mode = 2
        d = cache[key] = d
    return d


def _rows_bytes(lib, plan, B, ldg):
    d = _dims(plan, B)
    return lib.rd_workspace_bytes(C.byref(d)) + lib.rd_per_sample_grads_scratch_bytes(C.byref(d)) + 4 * B * ldg


def _row_batch(lib, plan, ldg, cap=DEFAULT_SCRATCH_BYTES):
    """Samples per forward / backward of the row computation: a power of two <= 128 whose buffers fit in half the cap.
    It depends on the model alone, and rows are computed in batches aligned to its multiples, so every sample's row comes
    from the same batch whatever the chunking (the forward's arithmetic depends on the batch it runs in)."""
    r = 128
    while r > 1 and _rows_bytes(lib, plan, r, ldg) > cap // 2:
        r //= 2
    return r


def _rows_aligned(model, fetch, i0, i1, R, ldg, margin=False):
    """Rows of samples [i0, i1) (i0 a multiple of R), computed in batches [k R, (k + 1) R).  margin: (rows, Q) as _rows
    returns them."""
    G = Q = None
    for s0 in range(i0, i1, R):
        s1 = min(i1, s0 + R)
        g = _rows(model, *fetch(s0, s1), ldg, margin)
        g, q = g if margin else (g, None)
        if G is None:
            if s1 == i1:
                return (g, q) if margin else g
            G = torch.empty(i1 - i0, ldg, dtype=torch.float32, device=g.device)
            Q = torch.empty(i1 - i0, dtype=torch.float64, device=g.device) if margin else None
        G[s0 - i0:s1 - i0] = g
        if margin:
            Q[s0 - i0:s1 - i0] = q
        del g
    return (G, Q) if margin else G


def _rows(model, src, static, times, lengths, y, ldg, margin=False):
    """[B, ldg] float32 gradient rows of CrossEntropy(logits_b, y_b); y None: the predicted class (argmax of the logits).
    margin: the rows of the margin m_b = z_y - log sum_{c != y} exp(z_c) instead, seeded by rd_trak_margin_seed on the
    eval forward without labels, returned with Q [B] = sigmoid(-m_b) float64."""
    cl = _Call(model, src, static, times, lengths, None, False)
    lib, plan, dev = cl.lib, cl.plan, cl.device
    B = cl.x.shape[1]
    dims = _dims(plan, B)
    key = (B, dims.obprop_mode, dev.index)
    ws = cl.scratch("_psg_workspace", key, lib.rd_workspace_bytes(C.byref(dims)))
    f32 = dict(device=dev, dtype=torch.float32)
    logits, dlog, loss = torch.empty(B, plan.n_classes, **f32), torch.empty(B, plan.n_classes, **f32), torch.empty(1, **f32)
    st = L.stream_ptr(dev)

    def fwd(yv):
        L.check(lib.rd_raindrop_v2_fwd(C.byref(dims), C.byref(cl.params), cl.x.data_ptr(), L.ptr(cl.st), cl.tm.data_ptr(),
                                       cl.ln.data_ptr(), plan.node_scale.data_ptr(), L.ptr(plan.rng_state), ws.data_ptr(),
                                       logits.data_ptr(), L.ptr(yv), L.ptr(None if yv is None else loss),
                                       L.ptr(None if yv is None else dlog), st), "rd_raindrop_v2_fwd")

    Q = None
    if margin:
        fwd(None)
        yv = (logits.argmax(dim=1) if y is None else y).to(device=dev, dtype=torch.int64).contiguous()
        Q = torch.empty(B, dtype=torch.float64, device=dev)
        L.check(lib.rd_trak_margin_seed(logits.data_ptr(), B, plan.n_classes, yv.data_ptr(), dlog.data_ptr(),
                                        Q.data_ptr(), st), "rd_trak_margin_seed")
    else:
        if y is None:
            fwd(None)
            y = logits.argmax(dim=1)
        fwd(y.to(device=dev, dtype=torch.int64).contiguous())
    G = torch.empty(B, ldg, **f32)
    scratch = cl.scratch("_psg_scratch", key, lib.rd_per_sample_grads_scratch_bytes(C.byref(dims)))
    L.check(lib.rd_raindrop_v2_per_sample_grads(C.byref(dims), C.byref(cl.params), L.ptr(cl.st), cl.ln.data_ptr(),
                                                plan.node_scale.data_ptr(), ws.data_ptr(), dlog.data_ptr(), scratch.data_ptr(),
                                                G.data_ptr(), ldg, st), "rd_raindrop_v2_per_sample_grads")
    return (G, Q) if margin else G


def _check_labels(y, B, n_classes, allow_none=False):
    if y is None:
        if allow_none:
            return None
        raise ValueError("y (labels [B]) is required")
    t = torch.as_tensor(y)
    if t.is_floating_point() or t.is_complex() or t.dtype == torch.bool:
        raise ValueError("y must hold integer class indices")
    if tuple(t.shape) != (B,):
        raise ValueError("y must be [B=%d], got %s" % (B, tuple(t.shape)))
    if B:
        lo, hi = torch.stack(torch.aminmax(t)).tolist()
        if lo < 0 or hi >= n_classes:
            raise ValueError("y values must lie in [0, %d), got [%d, %d]" % (n_classes, lo, hi))
    return t


def per_sample_grads(model, src, static, times, lengths, y):
    """[B, bucket] float32 on the device: row b = the gradient of CrossEntropy(logits_b, y_b) (not divided by B) with
    respect to every trained tensor, laid out as grad_layout(model) (padding columns 0).  Eval mode only; parameters and
    their .grad are left unchanged.  Raises RaindropB200Error without CUDA or without the built library."""
    _check_call("per_sample_grads", model, src, static, None, None)
    y = _check_labels(y, src.shape[1], model._plan.n_classes)
    with torch.no_grad():
        return _rows(model, src, static, times, lengths, y, _bucket_length(grad_layout(model)))


def per_sample_margin_grads(model, src, static, times, lengths, y=None):
    """(G [B, bucket] float32, Q [B] float64) on the device: row b = the gradient of the margin
    m_b = z_y - log sum_{c != y} exp(z_c) of the eval logits z (y None: the predicted class) with respect to every trained
    tensor, laid out as per_sample_grads; Q_b = 1 - p_y = sigmoid(-m_b).  The loss rows are -Q times these, since
    d CE / d logits = -Q d m / d logits.  The model needs 2 classes or more.  Eval mode only; parameters and their .grad
    are left unchanged.  Raises RaindropB200Error without CUDA or without the built library."""
    _check_call("per_sample_margin_grads", model, src, static, None, None)
    y = _check_labels(y, src.shape[1], model._plan.n_classes, allow_none=True)
    _check_margin_classes(model)
    with torch.no_grad():
        return _rows(model, src, static, times, lengths, y, _bucket_length(grad_layout(model)), margin=True)


def _check_margin_classes(model):
    if model._plan.n_classes < 2:
        raise ValueError("the margin needs a model of 2 classes or more")


# ---- data sources: a dict of tensors, or a DeviceDataset (optionally with an index subset) ----------------------------
def _source(data, what, unlabelled=False):
    """-> (n, fetch(i0, i1) -> (src, static, times, lengths, y)).  data: dict(src, static, times, lengths, y),
    a data.DeviceDataset, or a pair (DeviceDataset, indices).  unlabelled: a DeviceDataset without labels is served
    with y = None."""
    from .data import BatchBuffers, DeviceDataset
    idx = None
    if isinstance(data, tuple) and len(data) == 2 and isinstance(data[0], DeviceDataset):
        data, idx = data
    if isinstance(data, DeviceDataset):
        ds = data
        idx = torch.arange(ds.n, dtype=torch.int64) if idx is None else torch.as_tensor(idx, dtype=torch.int64).reshape(-1)
        if idx.numel() and (int(idx.min()) < 0 or int(idx.max()) >= ds.n):
            raise ValueError("%s indices must lie in [0, %d)" % (what, ds.n))
        if ds.y is None and not unlabelled:
            raise ValueError("%s DeviceDataset has no labels" % what)
        idx = idx.to(ds.P.device)

        def fetch(i0, i1):
            buf = BatchBuffers(ds.T, i1 - i0, ds.width, 0 if ds.Pstatic is None else ds.Pstatic.shape[1], device=ds.P.device)
            ds.fill(buf, idx[i0:i1])
            return buf.src, buf.static, buf.times, buf.lengths, None if ds.y is None else buf.y
        return idx.numel(), fetch
    if not isinstance(data, dict):
        raise TypeError("%s must be a dict (src, static, times, lengths, y) or a DeviceDataset" % what)
    missing = [k for k in ("src", "times", "lengths") if data.get(k) is None]
    if missing:
        raise ValueError("%s is missing %s" % (what, missing))
    src, static, times, lengths, y = (data["src"], data.get("static"), data["times"], data["lengths"], data.get("y"))

    def fetch(i0, i1):
        return (src[:, i0:i1], None if static is None else static[i0:i1], times[:, i0:i1], lengths[i0:i1],
                None if y is None else y[i0:i1])
    return src.shape[1], fetch


def _check_data(model, data, what, allow_none_y, unlabelled=False):
    """Host-side checks of a data argument against the model, before anything touches the device: a dict's tensor
    shapes and labels, or a DeviceDataset's T, width, static width, indices and the labels it will serve.  unlabelled:
    a DeviceDataset may have no labels (as _source(..., unlabelled=True) serves it)."""
    from .data import DeviceDataset
    from .models_rd import Raindrop_v2
    plan = model._plan
    if isinstance(data, tuple) and len(data) == 2 and isinstance(data[0], DeviceDataset):
        ds, idx = data
    else:
        ds, idx = data, None
    if isinstance(ds, DeviceDataset):
        if not isinstance(model, Raindrop_v2):
            raise TypeError("%s takes a raindrop_b200 Raindrop_v2 model, got %s" % (what, type(model).__name__))
        if model.training:
            raise ValueError("%s runs the model in eval arithmetic: call model.eval() first" % what)
        ds_static = 0 if ds.Pstatic is None else ds.Pstatic.shape[1]
        if ds.T != plan.T or ds.width != 2 * plan.N or (model.static and ds_static != plan.d_static):
            raise ValueError("%s DeviceDataset holds [T=%d, n, %d] with %d static columns; the model needs [T=%d, n, %d] "
                             "with %d" % (what, ds.T, ds.width, ds_static, plan.T, 2 * plan.N,
                                          plan.d_static if model.static else 0))
        if tuple(ds.Ptime.shape) != (ds.T, ds.n):
            raise ValueError("%s DeviceDataset times must be [T, n]" % what)
        if ds.y is None and not unlabelled:
            raise ValueError("%s DeviceDataset has no labels" % what)
        if ds.y is not None and tuple(ds.y.shape) != (ds.n,):
            raise ValueError("%s DeviceDataset labels must be [n]" % what)
        sel = torch.arange(ds.n, dtype=torch.int64) if idx is None else torch.as_tensor(idx).reshape(-1)
        if sel.is_floating_point() or sel.dtype == torch.bool:
            raise ValueError("%s indices must be integers" % what)
        if sel.numel():
            lo, hi = torch.stack(torch.aminmax(sel.to(torch.int64))).tolist()
            if lo < 0 or hi >= ds.n:
                raise ValueError("%s indices must lie in [0, %d)" % (what, ds.n))
            if ds.y is None:
                return
            ys = ds.y[sel.to(ds.y.device)] if idx is not None else ds.y
            lo, hi = torch.stack(torch.aminmax(ys)).tolist()         # one host sync
            if lo < 0 or hi >= plan.n_classes:
                raise ValueError("%s labels must lie in [0, %d), got [%d, %d]" % (what, plan.n_classes, lo, hi))
        return
    if not isinstance(data, dict):
        raise TypeError("%s must be a dict (src, static, times, lengths, y), a DeviceDataset or (DeviceDataset, indices)"
                        % what)
    src = data.get("src")
    if src is None:
        raise ValueError("%s is missing ['src']" % what)
    _check_call(what, model, src, data.get("static"), None, None)
    B = src.shape[1]
    shapes = [("times", (plan.T, B)), ("lengths", (B,))]
    if model.static:
        shapes.append(("static", (B, plan.d_static)))
    for k, shape in shapes:
        v = data.get(k)
        if v is None or tuple(v.shape) != shape:
            raise ValueError("%s[%r] must be %s" % (what, k, shape))
    _check_labels(data.get("y"), B, plan.n_classes, allow_none=allow_none_y)


def _checkpoints(model, checkpoints):
    """[(state_dict or None, lr)]; None = the current weights with lr 1."""
    if checkpoints is None:
        return [(None, 1.0)]
    out = []
    keys = [k for k, _ in model._plan.fields]
    shapes = {k: tuple(p.shape) for k, p in zip(keys, model.used_parameters())}
    for c in checkpoints:
        if not isinstance(c, (tuple, list)) or len(c) != 2:
            raise ValueError("each checkpoint must be a pair (state_dict, lr)")
        sd, lr = c
        lr = float(lr)
        if not math.isfinite(lr):
            raise ValueError("checkpoint lr must be finite")
        missing = [k for k in keys if k not in sd]
        if missing:
            raise ValueError("checkpoint state_dict is missing %s" % missing[:4])
        bad = [k for k in keys if tuple(sd[k].shape) != shapes[k]]
        if bad:
            raise ValueError("checkpoint tensors of the wrong shape: %s" % bad[:4])
        out.append((sd, lr))
    if not out:
        raise ValueError("checkpoints must not be empty")
    return out


class _Weights:
    """Loads checkpoints into the trained tensors in place; restores the original values, the mode and the dropout
    counter on exit."""

    def __init__(self, model):
        self.model = model

    def __enter__(self):
        m = self.model
        self.params = m.used_parameters()
        self.saved = [p.detach().clone() for p in self.params]
        self.training = m.training
        rs = m._plan.rng_state
        self.rng = None if rs is None else rs.clone()
        return self

    def load(self, sd):
        with torch.no_grad():
            for (key, _), p in zip(self.model._plan.fields, self.params):
                p.copy_(sd[key])

    def __exit__(self, *exc):
        with torch.no_grad():
            for p, s in zip(self.params, self.saved):
                p.copy_(s)
            if self.rng is not None:
                self.model._plan.rng_state.copy_(self.rng)
        self.model.train(self.training)
        return False


def _check_batch_size(internal_batch_size):
    if internal_batch_size is not None and int(internal_batch_size) < 1:
        raise ValueError("internal_batch_size must be >= 1")


def _blocks(lib, plan, ldg, n_seg, nq, nt, internal_batch_size, cap=DEFAULT_SCRATCH_BYTES):
    """(query block, train chunk, row batch R): blocks are multiples of R (internal_batch_size is rounded up to one).
    By default the query block is the largest whose rows, their remainder image (the dot's scratch) and one row batch's
    buffers fit in `cap`, and the train chunk the largest whose rows, one row batch's buffers and the dot's partial sums
    do; both are resident during a dot, so a call holds at most about 2 `cap` (2 GiB) besides the scores."""
    R = _row_batch(lib, plan, ldg, cap)
    up = lambda b: max(R, (b + R - 1) // R * R)
    down = lambda b: max(R, b // R * R)
    qb = down(_largest_chunk(lambda b: 8 * b * ldg + _rows_bytes(lib, plan, min(b, R), ldg), nq, cap))
    tc = down(_largest_chunk(lambda b: 4 * b * ldg + _rows_bytes(lib, plan, min(b, R), ldg) + 4 * n_seg * qb * b, nt, cap))
    if internal_batch_size is not None:
        qb = tc = up(int(internal_batch_size))
    return qb, tc, R


def tracin(model, query, train, checkpoints=None, fields=None, internal_batch_size=None):
    """TracIn scores [n_query, n_train] float64 on the device: sum_c lr_c <g_q(theta_c), g_t(theta_c)> over the selected
    fields (default: all trained tensors; a subset of privacy.sqnorm_fields(model), Captum's `layers`).

    query: dict(src, static, times, lengths, y); y None = each query's predicted class.  train: such a dict with y, a
    data.DeviceDataset, or a pair (DeviceDataset, indices).  checkpoints: [(state_dict, lr)] holding the trained tensors
    (default: the current weights, lr 1); the weights, the mode and the dropout counter are restored afterwards.
    internal_batch_size: rows per train chunk and per query block, rounded up to a multiple of the row batch (at most
    128 samples per forward; default: the largest whose buffers fit in 1 GiB each, so a call holds about 2 GiB).
    The query rows are computed once per checkpoint and query block, the train rows once per checkpoint, query
    block and chunk.  Eval mode only."""
    from .models_rd import _device_of
    if not isinstance(query, dict):
        raise TypeError("query must be a dict (src, static, times, lengths, y)")
    _check_data(model, query, "query", allow_none_y=True)
    _check_data(model, train, "train", allow_none_y=False)
    _check_batch_size(internal_batch_size)
    layout = grad_layout(model)
    ldg = _bucket_length(layout)
    seg_off, seg_len = plan_segments(layout, fields)
    ckpts = _checkpoints(model, checkpoints)
    dev = _device_of(query["src"])
    lib = L.load()
    plan = model._prepare(dev)
    nq, q_fetch = _source(query, "query")
    nt, t_fetch = _source(train, "train")
    n_seg = len(seg_off)
    scores = torch.zeros(nq, nt, dtype=torch.float64, device=dev)
    if nq == 0 or nt == 0:
        return scores
    qb, tc, R = _blocks(lib, plan, ldg, n_seg, nq, nt, internal_batch_size)
    offs = (C.c_int64 * n_seg)(*seg_off.tolist())
    lens = (C.c_int64 * n_seg)(*seg_len.tolist())
    st = L.stream_ptr(dev)
    with torch.no_grad(), _Weights(model) as w:
        for sd, lr in ckpts:
            if sd is not None:
                w.load(sd)
            for q0 in range(0, nq, qb):
                q1 = min(nq, q0 + qb)
                Gq = _rows_aligned(model, q_fetch, q0, q1, R, ldg)
                for t0 in range(0, nt, tc):
                    t1 = min(nt, t0 + tc)
                    Gt = _rows_aligned(model, t_fetch, t0, t1, R, ldg)
                    nb = lib.rd_per_sample_grad_dot_scratch_bytes(q1 - q0, t1 - t0, ldg, n_seg)
                    sc = torch.empty((nb + 3) // 4, dtype=torch.float32, device=dev)
                    L.check(lib.rd_per_sample_grad_dot(Gq.data_ptr(), q1 - q0, Gt.data_ptr(), t1 - t0, ldg, offs, lens, n_seg,
                                                       lr, scores.data_ptr() + 8 * (q0 * nt + t0), nt, sc.data_ptr(), st),
                            "rd_per_sample_grad_dot")
                    del Gt, sc
                del Gq
    return scores


def self_influence(model, data, checkpoints=None, fields=None, internal_batch_size=None):
    """[n] float64 on the device: sum_c lr_c ||g(theta_c)||^2 over the selected fields, from per_sample_grad_sqnorms
    (raindrop_b200.privacy; no gradient rows are materialised).  data: as tracin's train argument.  Chunks of tracin's
    row batch (internal_batch_size rounds up to a multiple of it), in tracin's ob-prop arithmetic."""
    from .models_rd import _device_of
    from .privacy import per_sample_grad_sqnorms, sqnorm_fields
    _check_data(model, data, "data", allow_none_y=False)
    _check_batch_size(internal_batch_size)
    if model.training:
        raise ValueError("self_influence runs the model in eval arithmetic: call model.eval() first")
    keys = sqnorm_fields(model)
    sel = _selected(grad_layout(model), fields)
    cols = torch.tensor([i for i, k in enumerate(keys) if k in sel], dtype=torch.int64)
    ckpts = _checkpoints(model, checkpoints)
    n, fetch = _source(data, "data")
    dev = _device_of(data["src"]) if isinstance(data, dict) else (data[0] if isinstance(data, tuple) else data).P.device
    out = torch.zeros(n, dtype=torch.float64, device=dev)
    lib = L.load()
    plan = model._prepare(dev)
    # chunks of tracin's row batch (so each chunk's buffers fit the cap), in tracin's ob-prop arithmetic: auto is pinned
    # to the error-compensated mode for the call, so the diagonal of tracin(X, X) and this agree
    R = _row_batch(lib, plan, _bucket_length(grad_layout(model)))
    chunk = R if internal_batch_size is None else max(R, (int(internal_batch_size) + R - 1) // R * R)
    mode = plan.obprop_mode
    try:
        if mode == 0:
            plan.obprop_mode = 2
        with torch.no_grad(), _Weights(model) as w:
            for sd, lr in ckpts:
                if sd is not None:
                    w.load(sd)
                for i0 in range(0, n, chunk):
                    i1 = min(n, i0 + chunk)
                    sq = per_sample_grad_sqnorms(model, *fetch(i0, i1))
                    out[i0:i1] += lr * sq[:, cols.to(dev)].sum(dim=1)
    finally:
        plan.obprop_mode = mode
    return out


def tracin_from_grads(Gq, Gt, lrs):
    """Host restatement of tracin in float64: Gq [n_ckpt, n_query, K] and Gt [n_ckpt, n_train, K] gradient rows (any
    array-likes; a 2-D pair is one checkpoint), lrs [n_ckpt] -> sum_c lrs[c] Gq[c] Gt[c]^T [n_query, n_train]."""
    Gq = np.asarray(Gq, dtype=np.float64)
    Gt = np.asarray(Gt, dtype=np.float64)
    if Gq.ndim == 2:
        Gq, Gt = Gq[None], Gt[None]
    lrs = np.atleast_1d(np.asarray(lrs, dtype=np.float64))
    if Gq.ndim != 3 or Gt.ndim != 3 or Gq.shape[0] != Gt.shape[0] or Gq.shape[2] != Gt.shape[2] or lrs.shape != (Gq.shape[0],):
        raise ValueError("Gq [c, q, K], Gt [c, t, K] and lrs [c] do not match: %s, %s, %s" % (Gq.shape, Gt.shape, lrs.shape))
    return np.einsum("c,cqk,ctk->qt", lrs, Gq, Gt)


# ---- TracIn-RP: random projections of the gradient rows (Pruthi et al. 2020, section 3.2) ------------------------------
PROJECTION_DIM_MULTIPLE, PROJECTION_DIM_MAX = 128, 32768


@dataclass
class GradientSketch:
    """Random projections phi = g Omega / sqrt(dim) of a data set's gradient rows, one block per checkpoint (project).
    features [n_ckpt, n, dim] float32; E[phi_q . phi_t] = g_q . g_t, with a variance that falls as 1 / dim.  Omega is
    the +-1 matrix of rd_grad_projection, fixed by `seed`; two sketches score against each other (tracin_sketch) only when
    dim, seed, fields, layout, lrs and the checkpoints' fingerprints (sha256 of their trained tensors) all agree."""
    features: torch.Tensor
    lrs: tuple
    dim: int
    seed: int
    fields: tuple            # None: every trained tensor
    layout: tuple            # ((state-dict key, shape), ...) of the gradient rows
    fingerprints: tuple      # sha256 hex digest per checkpoint

    def save(self, path):
        torch.save(dict(features=self.features.detach().cpu(), lrs=list(self.lrs), dim=self.dim, seed=self.seed,
                        fields=None if self.fields is None else list(self.fields),
                        layout=[[k, list(s)] for k, s in self.layout], fingerprints=list(self.fingerprints)), path)

    @classmethod
    def load(cls, path, map_location=None):
        d = torch.load(path, map_location=map_location, weights_only=True)
        return cls(features=d["features"], lrs=tuple(float(x) for x in d["lrs"]), dim=int(d["dim"]), seed=int(d["seed"]),
                   fields=None if d["fields"] is None else tuple(d["fields"]),
                   layout=tuple((k, tuple(int(x) for x in s)) for k, s in d["layout"]),
                   fingerprints=tuple(d["fingerprints"]))


def _check_projection(dim, seed):
    if isinstance(dim, bool) or not isinstance(dim, (int, np.integer)):
        raise ValueError("dim must be an integer")
    if dim % PROJECTION_DIM_MULTIPLE or not PROJECTION_DIM_MULTIPLE <= dim <= PROJECTION_DIM_MAX:
        raise ValueError("dim must be a multiple of %d in [%d, %d], got %d"
                         % (PROJECTION_DIM_MULTIPLE, PROJECTION_DIM_MULTIPLE, PROJECTION_DIM_MAX, dim))
    if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)) or not 0 <= seed < 1 << 64:
        raise ValueError("seed must be an integer in [0, 2**64)")


def _fingerprint(params):
    h = hashlib.sha256()
    for p in params:
        h.update(p.detach().to(torch.float32).contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def project(model, data, checkpoints=None, dim=4096, seed=0, fields=None, internal_batch_size=None):
    """GradientSketch of `data` (tracin's train argument, or a query dict whose y is None: the predicted class): the
    gradient rows of every sample at every checkpoint, projected onto `dim` random +-1 directions by rd_grad_projection
    (wgmma TF32 with Omega drawn in registers; fp32 within segments, fp64 across them).  The rows are computed as for
    tracin (eval arithmetic, ob-prop auto pinned to the error-compensated mode) chunk by chunk, and the full rows of the
    set are never held.  checkpoints, fields: as for tracin.  internal_batch_size: rows per chunk, rounded up to a
    multiple of the row batch (default: the largest whose rows and projection scratch fit in 1 GiB).  Features are
    bitwise the same for any internal_batch_size, data source or run.  The weights, the mode and the dropout counter are
    restored afterwards."""
    from .models_rd import _device_of
    _check_projection(dim, seed)
    _check_data(model, data, "data", allow_none_y=True)
    _check_batch_size(internal_batch_size)
    if model.training:
        raise ValueError("project runs the model in eval arithmetic: call model.eval() first")
    dim, seed = int(dim), int(seed)
    layout = grad_layout(model)
    ldg = _bucket_length(layout)
    seg_off, seg_len = plan_segments(layout, fields)
    sel_fields = None if fields is None else tuple(fields)
    ckpts = _checkpoints(model, checkpoints)
    dev = _device_of(data["src"]) if isinstance(data, dict) else (data[0] if isinstance(data, tuple) else data).P.device
    lib = L.load()
    plan = model._prepare(dev)
    n, fetch = _source(data, "data")
    n_seg = len(seg_off)
    features = torch.zeros(len(ckpts), n, dim, dtype=torch.float32, device=dev)
    R = _row_batch(lib, plan, ldg)
    if internal_batch_size is not None:
        chunk = max(R, (int(internal_batch_size) + R - 1) // R * R)
    else:
        chunk = max(R, _largest_chunk(lambda b: 4 * b * ldg + _rows_bytes(lib, plan, min(b, R), ldg) +
                                      lib.rd_grad_projection_scratch_bytes(b, ldg, dim, n_seg), max(n, 1)) // R * R)
    offs = (C.c_int64 * n_seg)(*seg_off.tolist())
    lens = (C.c_int64 * n_seg)(*seg_len.tolist())
    st = L.stream_ptr(dev)
    prints = []
    with torch.no_grad(), _Weights(model) as w:
        for c, (sd, lr) in enumerate(ckpts):
            if sd is not None:
                w.load(sd)
            prints.append(_fingerprint(w.params))
            for i0 in range(0, n, chunk):
                i1 = min(n, i0 + chunk)
                G = _rows_aligned(model, fetch, i0, i1, R, ldg)
                _project_rows(lib, G, ldg, offs, lens, n_seg, dim, seed, features[c, i0:i1], st)
                del G
    return GradientSketch(features=features, lrs=tuple(lr for _, lr in ckpts), dim=dim, seed=seed, fields=sel_fields,
                          layout=tuple((k, tuple(s)) for k, _, s in layout), fingerprints=tuple(prints))


def _project_rows(lib, G, ldg, offs, lens, n_seg, dim, seed, out, st):
    """out [rows, dim] (a contiguous float32 view) = rd_grad_projection of the rows G [rows, ldg]."""
    rows = G.shape[0]
    nb = lib.rd_grad_projection_scratch_bytes(rows, ldg, dim, n_seg)
    sc = torch.empty((nb + 3) // 4, dtype=torch.float32, device=G.device)
    L.check(lib.rd_grad_projection(G.data_ptr(), rows, ldg, offs, lens, n_seg, dim, seed, out.data_ptr(), dim,
                                   sc.data_ptr(), st), "rd_grad_projection")


def _check_sketches(q, t):
    for name in ("dim", "seed", "fields", "layout", "lrs", "fingerprints"):
        a, b = getattr(q, name), getattr(t, name)
        if a != b:
            raise ValueError("the sketches differ in %s: %s against %s" % (name, str(a)[:120], str(b)[:120]))
    if q.features.dim() != 3 or t.features.dim() != 3 or q.features.shape[0] != len(q.lrs) or \
            t.features.shape[0] != len(t.lrs) or q.features.shape[2] != q.dim or t.features.shape[2] != t.dim:
        raise ValueError("sketch features must be [n_ckpt, n, dim]: %s, %s"
                         % (tuple(q.features.shape), tuple(t.features.shape)))
    if q.features.device != t.features.device:
        raise ValueError("the sketches are on different devices: %s, %s" % (q.features.device, t.features.device))


def tracin_sketch(query_sketch, train_sketch, cap=DEFAULT_SCRATCH_BYTES):
    """TracIn-RP scores [n_query, n_train] float64 on the device: sum_c lr_c phi_q,c . phi_t,c, through
    rd_per_sample_grad_dot (ldg = dim, segments of RD_GRAD_DOT_SEGMENT columns), an unbiased estimate of tracin's
    scores.  Raises ValueError on the host when the sketches do not match (dim, seed, fields, layout, lrs, checkpoint
    fingerprints)."""
    _check_sketches(query_sketch, train_sketch)
    Fq, Ft = query_sketch.features, train_sketch.features
    nq, nt, dim = Fq.shape[1], Ft.shape[1], query_sketch.dim
    if Fq.device.type != "cuda":
        raise L.RaindropB200Error("tracin_sketch runs on a CUDA device; the sketches are on %s" % Fq.device)
    dev = Fq.device
    lib = L.load()
    scores = torch.zeros(nq, nt, dtype=torch.float64, device=dev)
    if nq == 0 or nt == 0:
        return scores
    Fq, Ft = Fq.to(torch.float32).contiguous(), Ft.to(torch.float32).contiguous()
    seg_off = np.arange(0, dim, SEGMENT, dtype=np.int64)
    seg_len = np.minimum(SEGMENT, dim - seg_off)
    n_seg = len(seg_off)
    offs = (C.c_int64 * n_seg)(*seg_off.tolist())
    lens = (C.c_int64 * n_seg)(*seg_len.tolist())
    qb = min(nq, 4096)
    tc = _largest_chunk(lambda b: lib.rd_per_sample_grad_dot_scratch_bytes(qb, b, dim, n_seg), nt, cap)
    st = L.stream_ptr(dev)
    for c, lr in enumerate(query_sketch.lrs):
        for q0 in range(0, nq, qb):
            q1 = min(nq, q0 + qb)
            for t0 in range(0, nt, tc):
                t1 = min(nt, t0 + tc)
                nb = lib.rd_per_sample_grad_dot_scratch_bytes(q1 - q0, t1 - t0, dim, n_seg)
                sc = torch.empty((nb + 3) // 4, dtype=torch.float32, device=dev)
                L.check(lib.rd_per_sample_grad_dot(Fq[c, q0].data_ptr(), q1 - q0, Ft[c, t0].data_ptr(), t1 - t0, dim, offs,
                                                   lens, n_seg, lr, scores.data_ptr() + 8 * (q0 * nt + t0), nt,
                                                   sc.data_ptr(), st), "rd_per_sample_grad_dot")
                del sc
    return scores


# ---- EK-FAC influence functions (George et al. 2018; Grosse et al. 2023) -----------------------------------------------
FISHER_MODES = ("true", "empirical")
EKFAC_DAMPING_FACTOR = 0.1       # damping=None: lambda_f = 0.1 * mean(Lambda) over each block or diagonal field


def kfac_blocks(model):
    """[(weight key, bias key, Nout, Kin)] of the Kronecker-factored blocks, in bucket order: per encoder layer in_proj,
    out_proj, linear1, linear2, then the lin_value of ob-prop layers 1 and 2 (the linear layers whose per-sample tiles the
    backward writes).  Every other trained tensor (LayerNorm gamma / beta, the head) is a diagonal field."""
    return _blocks_of_layout(tuple((k, tuple(s)) for k, _, s in grad_layout(model)))


def _check_block_fields(model, fields):
    """Selected keys; a linear weight without its bias (or the reverse) is refused: a block covers both."""
    sel = _selected(grad_layout(model), fields)
    for w, b, _, _ in kfac_blocks(model):
        if (w in sel) != (b in sel):
            raise ValueError("EK-FAC blocks cover a linear layer's weight and bias together: select both %s and %s, or "
                             "neither" % (w, b))
    return sel


def _check_fisher(fisher, seed):
    if fisher not in FISHER_MODES:
        raise ValueError("fisher must be one of %s, got %r" % (FISHER_MODES, fisher))
    if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)) or not 0 <= seed < 1 << 64:
        raise ValueError("seed must be an integer in [0, 2**64)")


def _check_damping(damping):
    if damping is None:
        return None
    if isinstance(damping, bool) or not isinstance(damping, (int, float, np.floating, np.integer)):
        raise ValueError("damping must be None or a positive float")
    d = float(damping)
    if not (math.isfinite(d) and d > 0):
        raise ValueError("damping must be None or a finite float > 0, got %r" % damping)
    return d


def _backward(model, src, static, times, lengths, y, kind, ldg=None, out=None, bases=None, fisher_seed=None, index0=0):
    """One eval forward and data-gradient backward of a row batch.  y None: labels drawn from the softmax
    (rd_fisher_labels, global indices index0..) when fisher_seed is set, else the predicted class.  kind "factors": adds
    the K-FAC sums into `out` (fp64); "rows": returns [B, ldg] EK-FAC rows rotated by `bases` (fp32 on the device)."""
    cl = _Call(model, src, static, times, lengths, None, False)
    lib, plan, dev = cl.lib, cl.plan, cl.device
    B = cl.x.shape[1]
    dims = _dims(plan, B)
    key = (B, dims.obprop_mode, dev.index)
    ws = cl.scratch("_psg_workspace", key, lib.rd_workspace_bytes(C.byref(dims)))
    f32 = dict(device=dev, dtype=torch.float32)
    logits, dlog, loss = torch.empty(B, plan.n_classes, **f32), torch.empty(B, plan.n_classes, **f32), torch.empty(1, **f32)
    st = L.stream_ptr(dev)

    def fwd(yv):
        L.check(lib.rd_raindrop_v2_fwd(C.byref(dims), C.byref(cl.params), cl.x.data_ptr(), L.ptr(cl.st), cl.tm.data_ptr(),
                                       cl.ln.data_ptr(), plan.node_scale.data_ptr(), L.ptr(plan.rng_state), ws.data_ptr(),
                                       logits.data_ptr(), L.ptr(yv), L.ptr(None if yv is None else loss),
                                       L.ptr(None if yv is None else dlog), st), "rd_raindrop_v2_fwd")

    if y is None:
        fwd(None)
        if fisher_seed is None:
            y = logits.argmax(dim=1)
        else:
            y = torch.empty(B, dtype=torch.int64, device=dev)
            L.check(lib.rd_fisher_labels(logits.data_ptr(), B, plan.n_classes, fisher_seed, index0, y.data_ptr(), st),
                    "rd_fisher_labels")
    fwd(y.to(device=dev, dtype=torch.int64).contiguous())
    if kind == "factors":
        scratch = cl.scratch("_kfac_scratch", key, lib.rd_kfac_factors_scratch_bytes(C.byref(dims)))
        L.check(lib.rd_raindrop_v2_kfac_factors(C.byref(dims), C.byref(cl.params), L.ptr(cl.st), cl.ln.data_ptr(),
                                                plan.node_scale.data_ptr(), ws.data_ptr(), dlog.data_ptr(),
                                                scratch.data_ptr(), out.data_ptr(), st), "rd_raindrop_v2_kfac_factors")
        return None
    G = torch.empty(B, ldg, **f32)
    scratch = cl.scratch("_ekfac_scratch", key, lib.rd_ekfac_rows_scratch_bytes(C.byref(dims)))
    L.check(lib.rd_raindrop_v2_ekfac_rows(C.byref(dims), C.byref(cl.params), L.ptr(cl.st), cl.ln.data_ptr(),
                                          plan.node_scale.data_ptr(), ws.data_ptr(), dlog.data_ptr(), bases.data_ptr(),
                                          scratch.data_ptr(), G.data_ptr(), ldg, st), "rd_raindrop_v2_ekfac_rows")
    return G


def _ekfac_rows_aligned(model, fetch, i0, i1, R, ldg, bases, fisher_seed=None):
    """EK-FAC rows of samples [i0, i1) (i0 a multiple of R), computed in batches [k R, (k + 1) R) as tracin's rows."""
    G = None
    for s0 in range(i0, i1, R):
        s1 = min(i1, s0 + R)
        src, static, times, lengths, y = fetch(s0, s1)
        g = _backward(model, src, static, times, lengths, None if fisher_seed is not None else y, "rows", ldg=ldg,
                      bases=bases, fisher_seed=fisher_seed, index0=s0)
        if G is None:
            if s1 == i1:
                return g
            G = torch.empty(i1 - i0, ldg, dtype=torch.float32, device=g.device)
        G[s0 - i0:s1 - i0] = g
        del g
    return G


def _factor_offsets(blocks):
    """[(a, s)] offsets (doubles) of each block's A and S in the packed factors (include/raindrop_b200.h)."""
    out, off = [], 0
    for _, _, nout, kin in blocks:
        out.append((off, off + (kin + 1) ** 2))
        off += (kin + 1) ** 2 + nout * nout
    return out, off


def _flat_bases(blocks, bases):
    """fp32 [rd_ekfac_bases_floats] on the host: per block Q_S^T [Nout, Nout] (padded to 4 floats), Q_A[:Kin]^T [Np, Kin]
    and Q_A[Kin] [Np], Np = Kin + 1 rounded up to 4 (zero past Kin + 1)."""
    parts = []
    for (_, _, nout, kin), (QA, QS) in zip(blocks, bases):
        npad = (kin + 4) // 4 * 4
        qs = torch.zeros((nout * nout + 3) // 4 * 4, dtype=torch.float64)
        qs[:nout * nout] = torch.as_tensor(QS).T.reshape(-1)
        qa = torch.zeros(npad, kin, dtype=torch.float64)
        qa[:kin + 1] = torch.as_tensor(QA)[:kin].T
        qb = torch.zeros(npad, dtype=torch.float64)
        qb[:kin + 1] = torch.as_tensor(QA)[kin]
        parts += [qs, qa.reshape(-1), qb]
    return torch.cat(parts).to(torch.float32)


def _eigh(M):
    """float64 eigendecomposition (ascending) with each eigenvector's largest-magnitude component made positive (the
    first such component on ties), so the basis is reproducible."""
    M = np.asarray(M, dtype=np.float64)
    w, Q = np.linalg.eigh(0.5 * (M + M.T))
    i = np.argmax(np.abs(Q), axis=0)
    sign = np.where(Q[i, np.arange(Q.shape[1])] < 0, -1.0, 1.0)
    return w, Q * sign


@dataclass
class EKFACFactors:
    """EK-FAC factors of one model's current weights (ekfac_factors): per Kronecker block (kfac_blocks) the float64 bases
    (Q_A [Kin + 1, Kin + 1], Q_S [Nout, Nout]), the corrected eigenvalues Lambda [bucket] float64 in the bucket layout
    (Lambda_j = (1/n) sum_b G~_bj^2; 0 outside the selected fields), n, fisher, seed, fields, layout and the sha256
    fingerprint of the trained tensors.  bases_flat: the fp32 bases as rd_raindrop_v2_ekfac_rows takes them."""
    bases: tuple             # ((Q_A, Q_S) float64 numpy per block)
    bases_flat: torch.Tensor
    eigenvalues: torch.Tensor
    n: int
    fisher: str
    seed: int
    fields: tuple            # None: every trained tensor
    layout: tuple            # ((state-dict key, shape), ...) of the gradient rows
    fingerprint: str

    def save(self, path):
        torch.save(self._state(), path)

    @classmethod
    def load(cls, path, map_location=None):
        return cls._from_state(torch.load(path, map_location=map_location, weights_only=True))

    def _state(self):
        """The dict save() writes: tensors, numbers, strings and lists only (torch.load's weights_only)."""
        return dict(bases=[[torch.from_numpy(np.ascontiguousarray(a)), torch.from_numpy(np.ascontiguousarray(s))]
                           for a, s in self.bases],
                    bases_flat=self.bases_flat.detach().cpu(), eigenvalues=self.eigenvalues.detach().cpu(), n=self.n,
                    fisher=self.fisher, seed=self.seed, fields=None if self.fields is None else list(self.fields),
                    layout=[[k, list(s)] for k, s in self.layout], fingerprint=self.fingerprint)

    @classmethod
    def _from_state(cls, d):
        return cls(bases=tuple((a.cpu().numpy(), s.cpu().numpy()) for a, s in d["bases"]), bases_flat=d["bases_flat"],
                   eigenvalues=d["eigenvalues"], n=int(d["n"]), fisher=str(d["fisher"]), seed=int(d["seed"]),
                   fields=None if d["fields"] is None else tuple(d["fields"]),
                   layout=tuple((k, tuple(int(x) for x in s)) for k, s in d["layout"]), fingerprint=str(d["fingerprint"]))


def _data_device(data):
    from .models_rd import _device_of
    return _device_of(data["src"]) if isinstance(data, dict) else (data[0] if isinstance(data, tuple) else data).P.device


def kfac_covariances(model, data, fisher="true", seed=0, internal_batch_size=None):
    """[(A, S)] float64 on the device, per Kronecker block (kfac_blocks): A = (1/n) sum_b sum_r x~_r x~_r^T over the
    layer's input rows x~ = [x | 1], S = (1/n) sum_b sum_r dy_r dy_r^T over its output gradients (of l_b, not l_b / B),
    encoder rows t*B + b for all T, ob-prop rows b*N + n.  fisher "true": labels drawn from the model's softmax
    (rd_fisher_labels, keyed by (seed, sample index)); "empirical": data's labels.  Computed in tracin's row batches, so
    the result is bitwise the same for any internal_batch_size (accepted for symmetry; it rounds up to the row batch)."""
    _check_fisher(fisher, seed)
    _check_data(model, data, "data", allow_none_y=fisher == "true")
    _check_batch_size(internal_batch_size)
    if model.training:
        raise ValueError("kfac_covariances runs the model in eval arithmetic: call model.eval() first")
    if fisher == "empirical" and isinstance(data, dict) and data.get("y") is None:
        raise ValueError("fisher='empirical' needs the data's labels y")
    dev = _data_device(data)
    lib = L.load()
    plan = model._prepare(dev)
    blocks = kfac_blocks(model)
    offs, total = _factor_offsets(blocks)
    n, fetch = _source(data, "data")
    R = _row_batch(lib, plan, _bucket_length(grad_layout(model)))
    d = _dims(plan, R)
    if lib.rd_kfac_factors_doubles(C.byref(d)) != total:
        raise L.RaindropB200Error("the K-FAC factor layout of the library and of influence.py disagree")
    acc = torch.zeros(total, dtype=torch.float64, device=dev)
    with torch.no_grad(), _Weights(model):
        for s0 in range(0, n, R):
            src, static, times, lengths, y = fetch(s0, min(n, s0 + R))
            _backward(model, src, static, times, lengths, None if fisher == "true" else y, "factors", out=acc,
                      fisher_seed=int(seed) if fisher == "true" else None, index0=s0)
    acc /= max(n, 1)
    return [(acc[a:a + (kin + 1) ** 2].view(kin + 1, kin + 1), acc[s:s + nout * nout].view(nout, nout))
            for (a, s), (_, _, nout, kin) in zip(offs, blocks)]


def _segments(seg_off, seg_len):
    n_seg = len(seg_off)
    return (C.c_int64 * n_seg)(*seg_off.tolist()), (C.c_int64 * n_seg)(*seg_len.tolist()), n_seg


def ekfac_factors(model, train, fisher="true", seed=0, fields=None, internal_batch_size=None):
    """EKFACFactors of `train` (tracin's train argument) at the model's current weights.  Two passes: the K-FAC factors
    (kfac_covariances) and their float64 eigenbases (numpy eigh on the host, signs fixed), then the rotated rows
    (rd_raindrop_v2_ekfac_rows, in tracin's row batches) whose squares rd_ekfac_accumulate_sq adds into Lambda; no rows
    are kept.  The same labels serve both passes.  fields: a subset of the trained tensors, chosen at block granularity
    (a linear layer's weight and bias together).  The weights, the mode and the dropout counter are restored."""
    _check_fisher(fisher, seed)
    sel = _check_block_fields(model, fields)
    _check_data(model, train, "train", allow_none_y=fisher == "true")
    _check_batch_size(internal_batch_size)
    if model.training:
        raise ValueError("ekfac_factors runs the model in eval arithmetic: call model.eval() first")
    layout = grad_layout(model)
    ldg = _bucket_length(layout)
    blocks = kfac_blocks(model)
    cov = kfac_covariances(model, train, fisher, seed, internal_batch_size)
    bases = []
    for A, S in cov:
        bases.append((_eigh(A.cpu().numpy())[1], _eigh(S.cpu().numpy())[1]))
    dev = _data_device(train)
    lib = L.load()
    plan = model._prepare(dev)
    flat = _flat_bases(blocks, bases)
    R = _row_batch(lib, plan, ldg)
    if lib.rd_ekfac_bases_floats(C.byref(_dims(plan, R))) != flat.numel():
        raise L.RaindropB200Error("the EK-FAC basis layout of the library and of influence.py disagree")
    flat_dev = flat.to(dev)
    seg_off, seg_len = plan_segments(layout, None if fields is None else list(fields))
    offs, lens, n_seg = _segments(seg_off, seg_len)
    n, fetch = _source(train, "train")
    lam = torch.zeros(ldg, dtype=torch.float64, device=dev)
    st = L.stream_ptr(dev)
    fs = int(seed) if fisher == "true" else None
    with torch.no_grad(), _Weights(model) as w:
        for s0 in range(0, n, R):
            s1 = min(n, s0 + R)
            G = _ekfac_rows_aligned(model, fetch, s0, s1, R, ldg, flat_dev, fs)
            L.check(lib.rd_ekfac_accumulate_sq(G.data_ptr(), s1 - s0, ldg, offs, lens, n_seg, lam.data_ptr(), st),
                    "rd_ekfac_accumulate_sq")
            del G
        fp = _fingerprint(w.params)
    lam /= max(n, 1)
    return EKFACFactors(bases=tuple(bases), bases_flat=flat, eigenvalues=lam, n=n, fisher=fisher, seed=int(seed),
                        fields=None if fields is None else tuple(fields),
                        layout=tuple((k, tuple(s)) for k, _, s in layout), fingerprint=fp)


def _damping_groups(layout, blocks, fields):
    """[(column ranges)] of the selected blocks (weight and bias together) and diagonal fields, in bucket order."""
    sel = _selected(layout, None if fields is None else list(fields))
    where = {k: (off, math.prod(shape)) for k, off, shape in layout}
    in_block = {}
    for w, b, _, _ in blocks:
        in_block[w] = in_block[b] = (w, b)
    groups, seen = [], set()
    for k, _, _ in layout:
        if k not in sel or k in seen:
            continue
        keys = in_block.get(k, (k,))
        seen.update(keys)
        groups.append([where[x] for x in keys])
    return groups


def ekfac_weights(factors, damping=None):
    """float64 numpy [bucket]: w_j = 1 / (Lambda_j + lambda_f(j)) on the selected columns, 0 elsewhere.  damping None:
    lambda_f = 0.1 * mean(Lambda) over each block (weight and bias) or diagonal field; a float: that value everywhere."""
    damping = _check_damping(damping)
    lam = factors.eigenvalues.detach().cpu().numpy().astype(np.float64)
    layout = [(k, off, s) for (k, s), off in zip(factors.layout, _offsets(factors.layout))]
    blocks = _blocks_of_layout(factors.layout)
    w = np.zeros_like(lam)
    for ranges in _damping_groups(layout, blocks, factors.fields):
        cols = np.concatenate([np.arange(o, o + n) for o, n in ranges])
        lf = EKFAC_DAMPING_FACTOR * lam[cols].mean() if damping is None else damping
        if not lf > 0:
            lf = np.finfo(np.float64).tiny
        w[cols] = 1.0 / (lam[cols] + lf)
    return w


def _offsets(layout_shapes):
    out, off = [], 0
    for _, s in layout_shapes:
        out.append(off)
        off += (math.prod(s) + 3) // 4 * 4
    return out


def _blocks_of_layout(layout_shapes):
    """kfac_blocks from a ((key, shape), ...) layout: the head has 6 fields with a static embedding, else 4."""
    keys = [k for k, _ in layout_shapes]
    head = 6 if keys[0].startswith("emb") else 4
    nl = (len(keys) - head - 4) // 12
    idx = [head + 12 * l + k for l in range(nl) for k in (0, 2, 4, 6)] + [head + 12 * nl, head + 12 * nl + 2]
    return [(keys[i], keys[i + 1], layout_shapes[i][1][0], layout_shapes[i][1][1]) for i in idx]


def _check_factors(model, factors):
    if not isinstance(factors, EKFACFactors):
        raise TypeError("factors must be an EKFACFactors (ekfac_factors)")
    layout = tuple((k, tuple(s)) for k, _, s in grad_layout(model))
    if factors.layout != layout:
        raise ValueError("the factors were computed for a model of another layout")
    if factors.fields is not None:
        _check_block_fields(model, list(factors.fields))
    if factors.eigenvalues.numel() != _bucket_length(grad_layout(model)):
        raise ValueError("the factors' eigenvalues do not span the model's gradient rows")
    if len(factors.bases) != len(kfac_blocks(model)):
        raise ValueError("the factors hold %d bases; the model has %d blocks" % (len(factors.bases), len(kfac_blocks(model))))
    fp = _fingerprint(model.used_parameters())
    if fp != factors.fingerprint:
        raise ValueError("the factors were computed for other weights (fingerprint %s..., the model's %s...)"
                         % (factors.fingerprint[:12], fp[:12]))


def ekfac_influence(model, query, train, factors, damping=None, internal_batch_size=None):
    """EK-FAC influence scores [n_query, n_train] float64 on the device: sum_j G~_qj G~_tj / (Lambda_j + lambda_f(j))
    over the factors' fields, G~ the gradient rows rotated into the Kronecker eigenbases (rd_raindrop_v2_ekfac_rows;
    LayerNorm and head fields unrotated).  Positive = proponent, as for tracin.  query: dict (y None = the predicted
    class); train: as tracin's (its true labels).  The query rows are scaled by w = 1 / (Lambda + lambda)
    (rd_ekfac_scale_rows, fp32) and contracted with the train rows by rd_per_sample_grad_dot, in tracin's blocks, so
    scores are bitwise the same for any internal_batch_size, data source or run.  Factors that do not match the model
    (layout, fields, weight fingerprint) are refused on the host.  The weights, mode and dropout counter are restored."""
    if not isinstance(query, dict):
        raise TypeError("query must be a dict (src, static, times, lengths, y)")
    _check_data(model, query, "query", allow_none_y=True)
    _check_data(model, train, "train", allow_none_y=False)
    _check_batch_size(internal_batch_size)
    damping = _check_damping(damping)
    _check_factors(model, factors)
    layout = grad_layout(model)
    ldg = _bucket_length(layout)
    seg_off, seg_len = plan_segments(layout, None if factors.fields is None else list(factors.fields))
    dev = _data_device(query)
    lib = L.load()
    plan = model._prepare(dev)
    nq, q_fetch = _source(query, "query")
    nt, t_fetch = _source(train, "train")
    offs, lens, n_seg = _segments(seg_off, seg_len)
    scores = torch.zeros(nq, nt, dtype=torch.float64, device=dev)
    if nq == 0 or nt == 0:
        return scores
    w = torch.from_numpy(ekfac_weights(factors, damping)).to(device=dev, dtype=torch.float32)
    bases = factors.bases_flat.to(device=dev, dtype=torch.float32).contiguous()
    qb, tc, R = _blocks(lib, plan, ldg, n_seg, nq, nt, internal_batch_size)
    st = L.stream_ptr(dev)
    with torch.no_grad(), _Weights(model):
        for q0 in range(0, nq, qb):
            q1 = min(nq, q0 + qb)
            Gq = _ekfac_rows_aligned(model, q_fetch, q0, q1, R, ldg, bases)
            L.check(lib.rd_ekfac_scale_rows(Gq.data_ptr(), q1 - q0, ldg, offs, lens, n_seg, w.data_ptr(), st),
                    "rd_ekfac_scale_rows")
            for t0 in range(0, nt, tc):
                t1 = min(nt, t0 + tc)
                Gt = _ekfac_rows_aligned(model, t_fetch, t0, t1, R, ldg, bases)
                nb = lib.rd_per_sample_grad_dot_scratch_bytes(q1 - q0, t1 - t0, ldg, n_seg)
                sc = torch.empty((nb + 3) // 4, dtype=torch.float32, device=dev)
                L.check(lib.rd_per_sample_grad_dot(Gq.data_ptr(), q1 - q0, Gt.data_ptr(), t1 - t0, ldg, offs, lens, n_seg,
                                                   1.0, scores.data_ptr() + 8 * (q0 * nt + t0), nt, sc.data_ptr(), st),
                        "rd_per_sample_grad_dot")
                del Gt, sc
            del Gq
    return scores


def ekfac_self_influence(model, data, factors, damping=None, internal_batch_size=None):
    """[n] float64 on the device: sum_j G~_j^2 / (Lambda_j + lambda_f(j)) of each sample with its own label, for ranking
    candidate mislabels.  Each row batch's scaled rows are contracted with its rows by rd_per_sample_grad_dot and the
    diagonal kept, so the result equals the diagonal of ekfac_influence(data, data) (data's labels on both sides)
    bitwise.  internal_batch_size: accepted for symmetry (the work runs in tracin's row batches)."""
    _check_data(model, data, "data", allow_none_y=False)
    _check_batch_size(internal_batch_size)
    damping = _check_damping(damping)
    if model.training:
        raise ValueError("ekfac_self_influence runs the model in eval arithmetic: call model.eval() first")
    _check_factors(model, factors)
    layout = grad_layout(model)
    ldg = _bucket_length(layout)
    seg_off, seg_len = plan_segments(layout, None if factors.fields is None else list(factors.fields))
    offs, lens, n_seg = _segments(seg_off, seg_len)
    dev = _data_device(data)
    lib = L.load()
    plan = model._prepare(dev)
    n, fetch = _source(data, "data")
    out = torch.zeros(n, dtype=torch.float64, device=dev)
    if n == 0:
        return out
    w = torch.from_numpy(ekfac_weights(factors, damping)).to(device=dev, dtype=torch.float32)
    bases = factors.bases_flat.to(device=dev, dtype=torch.float32).contiguous()
    R = _row_batch(lib, plan, ldg)
    st = L.stream_ptr(dev)
    with torch.no_grad(), _Weights(model):
        for s0 in range(0, n, R):
            s1 = min(n, s0 + R)
            b = s1 - s0
            G = _ekfac_rows_aligned(model, fetch, s0, s1, R, ldg, bases)
            Gs = G.clone()
            L.check(lib.rd_ekfac_scale_rows(Gs.data_ptr(), b, ldg, offs, lens, n_seg, w.data_ptr(), st),
                    "rd_ekfac_scale_rows")
            sq = torch.zeros(b, b, dtype=torch.float64, device=dev)
            nb = lib.rd_per_sample_grad_dot_scratch_bytes(b, b, ldg, n_seg)
            sc = torch.empty((nb + 3) // 4, dtype=torch.float32, device=dev)
            L.check(lib.rd_per_sample_grad_dot(Gs.data_ptr(), b, G.data_ptr(), b, ldg, offs, lens, n_seg, 1.0,
                                               sq.data_ptr(), b, sc.data_ptr(), st), "rd_per_sample_grad_dot")
            out[s0:s1] = sq.diagonal()
            del G, Gs, sc, sq
    return out


def ekfac_rotate(G, factors):
    """float64 numpy restatement of the rotation: G [n, bucket] gradient rows -> G~ with each block's [Nout, Kin + 1]
    tile [W | b] replaced by Q_S^T [W | b] Q_A (LayerNorm and head fields, and padding, unchanged)."""
    G = np.array(G, dtype=np.float64, copy=True)
    offs = dict(zip([k for k, _ in factors.layout], _offsets(factors.layout)))
    for (wk, bk, nout, kin), (QA, QS) in zip(_blocks_of_layout(factors.layout), factors.bases):
        ow, ob = offs[wk], offs[bk]
        M = np.concatenate([G[:, ow:ow + nout * kin].reshape(-1, nout, kin), G[:, ob:ob + nout, None]], axis=2)
        Mt = np.asarray(QS, np.float64).T @ M @ np.asarray(QA, np.float64)
        G[:, ow:ow + nout * kin] = Mt[:, :, :kin].reshape(len(G), -1)
        G[:, ob:ob + nout] = Mt[:, :, kin]
    return G


def ekfac_from_grads(Gq, Gt, factors, damping=None):
    """Host restatement of ekfac_influence in float64: Gq [n_query, bucket] and Gt [n_train, bucket] plain gradient rows
    (per_sample_grads), rotated with the factors' float64 bases (ekfac_rotate) and contracted with the weights
    ekfac_weights(factors, damping) -> [n_query, n_train]."""
    w = ekfac_weights(factors, damping)
    Gq, Gt = np.asarray(Gq, dtype=np.float64), np.asarray(Gt, dtype=np.float64)
    if Gq.ndim != 2 or Gt.ndim != 2 or Gq.shape[1] != w.shape[0] or Gt.shape[1] != w.shape[0]:
        raise ValueError("Gq [q, %d] and Gt [t, %d] do not match: %s, %s" % (w.shape[0], w.shape[0], Gq.shape, Gt.shape))
    return (ekfac_rotate(Gq, factors) * w) @ ekfac_rotate(Gt, factors).T


# ---- TRAK (Park et al. 2023) -------------------------------------------------------------------------------------------
TRAK_DIM_MAX = L.TRAK_DIM_MAX


@dataclass
class TRAKFeatures:
    """TRAK features of a training set (trak_features), one block per model k (an ensemble member's weights):
    features [M, n, dim] float32, the projected margin rows rotated into the eigenbasis of their Gram, Phi_k V_k;
    eigenvalues [M, dim] float64 (ascending) and eigenvectors V [M, dim, dim] float64 of K_k = Phi_k^T Phi_k; Q [M, n]
    float64 = sigmoid(-margin) of each training sample under each model.  Omega is rd_grad_projection's +-1 matrix for
    `seed`; scoring (trak) refuses features whose dim, fields, layout or weight fingerprints (sha256 of each model's
    trained tensors) do not match the model and checkpoints it is given."""
    features: torch.Tensor
    eigenvalues: torch.Tensor
    eigenvectors: torch.Tensor
    Q: torch.Tensor
    dim: int
    seed: int
    fields: tuple            # None: every trained tensor
    layout: tuple            # ((state-dict key, shape), ...) of the gradient rows
    fingerprints: tuple      # sha256 hex digest per model

    def save(self, path):
        torch.save(dict(features=self.features.detach().cpu(), eigenvalues=self.eigenvalues.detach().cpu(),
                        eigenvectors=self.eigenvectors.detach().cpu(), Q=self.Q.detach().cpu(), dim=self.dim,
                        seed=self.seed, fields=None if self.fields is None else list(self.fields),
                        layout=[[k, list(s)] for k, s in self.layout], fingerprints=list(self.fingerprints)), path)

    @classmethod
    def load(cls, path, map_location=None):
        d = torch.load(path, map_location=map_location, weights_only=True)
        return cls(features=d["features"], eigenvalues=d["eigenvalues"], eigenvectors=d["eigenvectors"], Q=d["Q"],
                   dim=int(d["dim"]), seed=int(d["seed"]), fields=None if d["fields"] is None else tuple(d["fields"]),
                   layout=tuple((k, tuple(int(x) for x in s)) for k, s in d["layout"]),
                   fingerprints=tuple(d["fingerprints"]))


def _check_trak_dim(dim, seed):
    if isinstance(dim, bool) or not isinstance(dim, (int, np.integer)):
        raise ValueError("dim must be an integer")
    if dim % PROJECTION_DIM_MULTIPLE or not PROJECTION_DIM_MULTIPLE <= dim <= TRAK_DIM_MAX:
        raise ValueError("dim must be a multiple of %d in [%d, %d] (the Gram and its eigenvectors are dim^2 float64 per "
                         "model), got %d" % (PROJECTION_DIM_MULTIPLE, PROJECTION_DIM_MULTIPLE, TRAK_DIM_MAX, dim))
    _check_projection(int(dim), seed)


def _check_trak_regularisation(damping, rcond):
    """(damping, rcond) as floats: damping finite >= 0; rcond None (dim * 2^-52 at use) or finite >= 0."""
    out = []
    for name, v in (("damping", damping), ("rcond", rcond)):
        if v is None and name == "rcond":
            out.append(None)
            continue
        if isinstance(v, bool) or not isinstance(v, (int, float, np.floating, np.integer)):
            raise ValueError("%s must be a float >= 0" % name)
        f = float(v)
        if not (math.isfinite(f) and f >= 0):
            raise ValueError("%s must be a finite float >= 0, got %r" % (name, v))
        out.append(f)
    return tuple(out)


def trak_weights(eigenvalues, damping=0.0, rcond=None):
    """float64 numpy [M, dim]: w_kj = 1 / (lambda_kj + damping), and 0 where lambda_kj <= rcond * max_j lambda_kj
    (rcond None: dim * 2^-52, the usual pseudo-inverse rule, so rank-deficient sketches work)."""
    damping, rcond = _check_trak_regularisation(damping, rcond)
    lam = np.atleast_2d(np.asarray(eigenvalues.detach().cpu() if torch.is_tensor(eigenvalues) else eigenvalues,
                                   dtype=np.float64))
    rc = lam.shape[1] * 2.0 ** -52 if rcond is None else rcond
    keep = lam > rc * lam.max(axis=1, keepdims=True)
    return np.where(keep, 1.0 / np.where(keep, lam + damping, 1.0), 0.0)


def _trak_models(model, checkpoints):
    """[(state_dict or None, 1.0)] of the ensemble: checkpoints is None (the current weights) or a list of state dicts."""
    from collections.abc import Mapping
    if checkpoints is None:
        return _checkpoints(model, None)
    if isinstance(checkpoints, Mapping) or not all(isinstance(sd, Mapping) for sd in checkpoints):
        raise ValueError("checkpoints must be a list of state dicts (one per model)")
    return _checkpoints(model, [(sd, 1.0) for sd in checkpoints])


def _model_fingerprints(model, ckpts):
    keys = [k for k, _ in model._plan.fields]
    return tuple(_fingerprint(model.used_parameters() if sd is None else [sd[k] for k in keys]) for sd, _ in ckpts)


def _trak_chunk(lib, plan, ldg, dim, n_seg, n, R, internal_batch_size, cap=DEFAULT_SCRATCH_BYTES):
    """Rows per chunk of the margin rows: a multiple of R (internal_batch_size rounded up to one; default the largest
    whose rows, row buffers, projection scratch and projected / rotated rows fit in `cap`)."""
    if internal_batch_size is not None:
        return max(R, (int(internal_batch_size) + R - 1) // R * R)
    return max(R, _largest_chunk(lambda b: 4 * b * ldg + _rows_bytes(lib, plan, min(b, R), ldg) + 8 * b * dim +
                                 lib.rd_grad_projection_scratch_bytes(b, ldg, dim, n_seg), max(n, 1), cap) // R * R)


def _trak_sketch(model, fetch, n, dim, seed, seg, chunk, R, ldg):
    """(Phi [n, dim] float32, Q [n] float64) of the current weights: the margin rows of samples [0, n), projected by
    rd_grad_projection chunk by chunk (the full rows of the set are never held)."""
    lib, dev = L.load(), model._plan.node_scale.device
    offs, lens, n_seg = seg
    Phi = torch.empty(n, dim, dtype=torch.float32, device=dev)
    Q = torch.empty(n, dtype=torch.float64, device=dev)
    st = L.stream_ptr(dev)
    for i0 in range(0, n, chunk):
        i1 = min(n, i0 + chunk)
        G, Q[i0:i1] = _rows_aligned(model, fetch, i0, i1, R, ldg, margin=True)
        _project_rows(lib, G, ldg, offs, lens, n_seg, dim, seed, Phi[i0:i1], st)
        del G
    return Phi, Q


def _trak_gram(Phi):
    """K = Phi^T Phi [dim, dim] float64 on the device (rd_trak_gram: one pass, rows in order, exactly symmetric)."""
    n, dim = Phi.shape
    K = torch.zeros(dim, dim, dtype=torch.float64, device=Phi.device)
    L.check(L.load().rd_trak_gram(Phi.data_ptr(), n, dim, K.data_ptr(), L.stream_ptr(Phi.device)), "rd_trak_gram")
    return K


def _trak_eigh(K):
    """(lambda ascending, V) of K by torch.linalg.eigh in float64 on K's device, each eigenvector's largest-magnitude
    component made positive (the first such component on ties), so the basis is reproducible."""
    lam, V = torch.linalg.eigh(K)
    i = V.abs().argmax(dim=0)
    sign = torch.where(V.gather(0, i[None]).squeeze(0) < 0, -1.0, 1.0).to(V.dtype)
    return lam, (V * sign).contiguous()


def _trak_rotate(Phi, V, out=None):
    """Phi V [n, dim] float32 on the device (rd_trak_rotate: fp64 products and sums, one rounding per element)."""
    n, dim = Phi.shape
    out = torch.empty(n, dim, dtype=torch.float32, device=Phi.device) if out is None else out
    L.check(L.load().rd_trak_rotate(Phi.data_ptr(), n, dim, V.data_ptr(), out.data_ptr(), L.stream_ptr(Phi.device)),
            "rd_trak_rotate")
    return out


def trak_features(model, train, checkpoints=None, dim=4096, seed=0, fields=None, internal_batch_size=None):
    """TRAKFeatures of `train` (tracin's train argument: a dict with y, a DeviceDataset or (DeviceDataset, indices)).
    Per model k (checkpoints: a list of state dicts holding the trained tensors, e.g. independently seeded runs; default
    the current weights): the margin gradient rows of every training sample with its label (per_sample_margin_grads, in
    tracin's row batches), projected onto `dim` +-1 directions (rd_grad_projection; phi = g Omega / sqrt(dim)), their fp64
    Gram K (rd_trak_gram), its eigendecomposition (torch.linalg.eigh in float64 on the device) and the features rotated
    into that basis (rd_trak_rotate).  fields: as for tracin.  dim: a multiple of 128 in [128, 8192] (K and V are dim^2
    float64 per model).  internal_batch_size: rows per chunk, rounded up to a multiple of the row batch.  The result is
    bitwise the same for any internal_batch_size, data source or run.  The weights, mode and dropout counter are
    restored.  Eval mode only."""
    _check_trak_dim(dim, seed)
    _check_data(model, train, "train", allow_none_y=False)
    _check_batch_size(internal_batch_size)
    if model.training:
        raise ValueError("trak_features runs the model in eval arithmetic: call model.eval() first")
    _check_margin_classes(model)
    dim, seed = int(dim), int(seed)
    layout = grad_layout(model)
    ldg = _bucket_length(layout)
    seg = _segments(*plan_segments(layout, fields))
    ckpts = _trak_models(model, checkpoints)
    dev = _data_device(train)
    lib = L.load()
    plan = model._prepare(dev)
    n, fetch = _source(train, "train")
    M = len(ckpts)
    R = _row_batch(lib, plan, ldg)
    chunk = _trak_chunk(lib, plan, ldg, dim, seg[2], n, R, internal_batch_size)
    features = torch.empty(M, n, dim, dtype=torch.float32, device=dev)
    lam = torch.empty(M, dim, dtype=torch.float64, device=dev)
    V = torch.empty(M, dim, dim, dtype=torch.float64, device=dev)
    Q = torch.empty(M, n, dtype=torch.float64, device=dev)
    prints = []
    with torch.no_grad(), _Weights(model) as w:
        for k, (sd, _) in enumerate(ckpts):
            if sd is not None:
                w.load(sd)
            prints.append(_fingerprint(w.params))
            Phi, Q[k] = _trak_sketch(model, fetch, n, dim, seed, seg, chunk, R, ldg)
            lam[k], V[k] = _trak_eigh(_trak_gram(Phi))
            _trak_rotate(Phi, V[k], out=features[k])
            del Phi
    return TRAKFeatures(features=features, eigenvalues=lam, eigenvectors=V, Q=Q, dim=dim, seed=seed,
                        fields=None if fields is None else tuple(fields),
                        layout=tuple((k, tuple(s)) for k, _, s in layout), fingerprints=tuple(prints))


def _check_trak_features(model, features, ckpts):
    if not isinstance(features, TRAKFeatures):
        raise TypeError("features must be a TRAKFeatures (trak_features)")
    layout = tuple((k, tuple(s)) for k, _, s in grad_layout(model))
    if features.layout != layout:
        raise ValueError("the features were computed for a model of another layout")
    if features.fields is not None:
        _selected(grad_layout(model), list(features.fields))
    _check_trak_dim(features.dim, features.seed)
    M, dim = len(features.fingerprints), features.dim
    F, lam, V, Q = features.features, features.eigenvalues, features.eigenvectors, features.Q
    if F.dim() != 3 or tuple(F.shape[::2]) != (M, dim) or tuple(lam.shape) != (M, dim) or \
            tuple(V.shape) != (M, dim, dim) or tuple(Q.shape) != (M, F.shape[1]):
        raise ValueError("features [M, n, dim], eigenvalues [M, dim], eigenvectors [M, dim, dim] and Q [M, n] do not "
                         "match M = %d, dim = %d" % (M, dim))
    if len(ckpts) != M:
        raise ValueError("the features hold %d models; %d were given" % (M, len(ckpts)))
    prints = _model_fingerprints(model, ckpts)
    for k, (a, b) in enumerate(zip(prints, features.fingerprints)):
        if a != b:
            raise ValueError("the features of model %d were computed for other weights (fingerprint %s..., the "
                             "weights' %s...)" % (k, b[:12], a[:12]))


def trak(model, query, features, damping=0.0, rcond=None, internal_batch_size=None, checkpoints=None):
    """TRAK scores [n_query, n_train] float64 on the device:
        tau(q, i) = [(1/M) sum_k sum_j w_kj phi~_k(q)_j phi~_k(z_i)_j] [(1/M) sum_k Q_k(i)],
    w_kj = 1 / (lambda_kj + damping) (0 where lambda_kj <= rcond max lambda_k; trak_weights), phi~ = the projected margin
    rows rotated into each model's eigenbasis.  Positive = proponent, as for tracin.  query: dict (y None = each model's
    predicted class).  checkpoints: the state dicts the features were computed with (default: the current weights, one
    model); features of other weights, layout, fields or dim are refused on the host.  Per model and query block: the
    margin rows (tracin's row batches), rd_grad_projection, rd_trak_rotate, rd_ekfac_scale_rows by w (fp32), and
    rd_per_sample_grad_dot with alpha = 1/M into the fp64 scores, whose columns are then scaled by the mean Q.  Bitwise
    the same for any internal_batch_size, data source or run.  The weights, mode and dropout counter are restored."""
    if not isinstance(query, dict):
        raise TypeError("query must be a dict (src, static, times, lengths, y)")
    _check_data(model, query, "query", allow_none_y=True)
    _check_batch_size(internal_batch_size)
    damping, rcond = _check_trak_regularisation(damping, rcond)
    if model.training:
        raise ValueError("trak runs the model in eval arithmetic: call model.eval() first")
    _check_margin_classes(model)
    ckpts = _trak_models(model, checkpoints)
    _check_trak_features(model, features, ckpts)
    dim, seed, M = features.dim, features.seed, len(ckpts)
    layout = grad_layout(model)
    ldg = _bucket_length(layout)
    seg = _segments(*plan_segments(layout, None if features.fields is None else list(features.fields)))
    dev = _data_device(query)
    lib = L.load()
    plan = model._prepare(dev)
    nq, q_fetch = _source(query, "query")
    nt = features.features.shape[1]
    scores = torch.zeros(nq, nt, dtype=torch.float64, device=dev)
    if nq == 0 or nt == 0:
        return scores
    W = torch.from_numpy(trak_weights(features.eigenvalues, damping, rcond)).to(device=dev, dtype=torch.float32)
    Ft = features.features.to(device=dev, dtype=torch.float32).contiguous()
    R = _row_batch(lib, plan, ldg)
    qb = _trak_chunk(lib, plan, ldg, dim, seg[2], nq, R, internal_batch_size)
    dot_off, dot_len, dot_n = _segments(np.arange(0, dim, SEGMENT, dtype=np.int64),
                                        np.minimum(SEGMENT, dim - np.arange(0, dim, SEGMENT, dtype=np.int64)))
    tc = _largest_chunk(lambda b: lib.rd_per_sample_grad_dot_scratch_bytes(min(qb, nq), b, dim, dot_n), nt)
    whole = _segments(np.zeros(1, np.int64), np.full(1, dim, np.int64))
    st = L.stream_ptr(dev)
    with torch.no_grad(), _Weights(model) as w:
        for k, (sd, _) in enumerate(ckpts):
            if sd is not None:
                w.load(sd)
            V = features.eigenvectors[k].to(device=dev, dtype=torch.float64).contiguous()
            for q0 in range(0, nq, qb):
                q1 = min(nq, q0 + qb)
                Phi, _ = _trak_sketch(model, lambda a, b: q_fetch(q0 + a, q0 + b), q1 - q0, dim, seed, seg, qb, R, ldg)
                Pr = _trak_rotate(Phi, V)
                del Phi
                L.check(lib.rd_ekfac_scale_rows(Pr.data_ptr(), q1 - q0, dim, *whole, W[k].data_ptr(), st),
                        "rd_ekfac_scale_rows")
                for t0 in range(0, nt, tc):
                    t1 = min(nt, t0 + tc)
                    nb = lib.rd_per_sample_grad_dot_scratch_bytes(q1 - q0, t1 - t0, dim, dot_n)
                    sc = torch.empty((nb + 3) // 4, dtype=torch.float32, device=dev)
                    L.check(lib.rd_per_sample_grad_dot(Pr.data_ptr(), q1 - q0, Ft[k, t0].data_ptr(), t1 - t0, dim,
                                                       dot_off, dot_len, dot_n, 1.0 / M,
                                                       scores.data_ptr() + 8 * (q0 * nt + t0), nt, sc.data_ptr(), st),
                            "rd_per_sample_grad_dot")
                    del sc
                del Pr
    scores *= features.Q.to(device=dev, dtype=torch.float64).mean(dim=0)[None, :]
    return scores


def trak_self_influence(features, damping=0.0, rcond=None):
    """[n] float64 on the device: the leverages (1/M) sum_k sum_j w_kj phi~_k(z_i)_j^2 times the mean Q of each training
    sample, the diagonal of trak(train, train) with each model's labels on both sides (to rounding: this sums the
    float32 features' squares in float64).  With one model and damping 0 the leverage (before Q) lies in [0, 1] and the
    leverages sum to the rank of the sketch; large values flag candidate mislabels or outliers, as self_influence."""
    if not isinstance(features, TRAKFeatures):
        raise TypeError("features must be a TRAKFeatures (trak_features)")
    _check_trak_regularisation(damping, rcond)
    F = features.features
    if F.device.type != "cuda":
        raise L.RaindropB200Error("trak_self_influence runs on a CUDA device; the features are on %s" % F.device)
    W = torch.from_numpy(trak_weights(features.eigenvalues, damping, rcond)).to(F.device)
    M, n = F.shape[0], F.shape[1]
    out = torch.zeros(n, dtype=torch.float64, device=F.device)
    step = max(1, (1 << 27) // max(1, features.dim))
    for k in range(M):
        for i0 in range(0, n, step):
            out[i0:i0 + step] += F[k, i0:i0 + step].double().square() @ W[k]
    return out / M * features.Q.to(F.device).double().mean(dim=0)


def trak_from_features(Fq, Ft, Q, damping=0.0, rcond=None):
    """Host restatement of trak in float64: Fq [M, n_query, dim] and Ft [M, n_train, dim] projected (unrotated) margin
    features, Q [M, n_train] (2-D / 1-D arrays: one model) -> [n_query, n_train]: per model the eigendecomposition of
    Ft^T Ft (numpy eigh), the weights trak_weights(lambda, damping, rcond), the weighted products of the rotated
    features averaged over models, times the mean Q of each training sample."""
    Fq, Ft, Q = (np.asarray(a, dtype=np.float64) for a in (Fq, Ft, Q))
    if Fq.ndim == 2:
        Fq, Ft, Q = Fq[None], Ft[None], Q[None]
    if Fq.ndim != 3 or Ft.ndim != 3 or Q.ndim != 2 or Fq.shape[0] != Ft.shape[0] or Fq.shape[2] != Ft.shape[2] or \
            Q.shape != Ft.shape[:2]:
        raise ValueError("Fq [M, q, dim], Ft [M, t, dim] and Q [M, t] do not match: %s, %s, %s"
                         % (Fq.shape, Ft.shape, Q.shape))
    M = Fq.shape[0]
    S = np.zeros((Fq.shape[1], Ft.shape[1]))
    for k in range(M):
        lam, V = np.linalg.eigh(Ft[k].T @ Ft[k])
        w = trak_weights(lam[None], damping, rcond)[0]
        S += ((Fq[k] @ V) * w) @ (Ft[k] @ V).T
    return S / M * Q.mean(axis=0)[None, :]
