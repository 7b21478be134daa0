"""Integrated-gradients (IG) attribution of Raindrop_v2, computed on the device in one call
(rd_raindrop_v2_integrated_gradients), and the per-sensor ranking that the reference's leave-sensors-out experiment
with feature_removal_level='set' reads (code/Raindrop.py:227-231, IG_density_scores_<dataset>.npy).

    attr_src, attr_static = integrated_gradients(model.eval(), src, static, times, lengths, target=y)
    ranking = sensor_ranking(sensor_importance(attr_src, model.d_inp), names)
    idx = data.removal_indices(B, model.d_inp, 0.5, level="set", density_scores=ranking[:, 0])

Argument names follow Captum's IntegratedGradients.attribute.
"""
import ctypes as C

import numpy as np
import torch

from . import functional as RF
from . import lib as L

METHODS = ("gausslegendre", "riemann_trapezoid")
DEFAULT_SCRATCH_BYTES = 1 << 30      # default chunking: the largest one whose scratch fits in 1 GiB


def quadrature(n_steps, method="gausslegendre"):
    """(alphas, weights) of an n_steps-point rule on [0, 1], float64 numpy arrays; the weights sum to 1.
    gausslegendre: numpy.polynomial.legendre.leggauss mapped from [-1, 1]; riemann_trapezoid: linspace(0, 1, n) with
    weights 1/(n-1), halved at both ends (Captum's rule of that name)."""
    n = int(n_steps)
    if method == "gausslegendre":
        if n < 1:
            raise ValueError("n_steps must be >= 1, got %d" % n)
        x, w = np.polynomial.legendre.leggauss(n)
        return (x + 1.0) / 2.0, w / 2.0
    if method == "riemann_trapezoid":
        if n < 2:
            raise ValueError("riemann_trapezoid needs n_steps >= 2, got %d" % n)
        w = np.full(n, 1.0 / (n - 1))
        w[0] = w[-1] = 0.5 / (n - 1)
        return np.linspace(0.0, 1.0, n), w
    raise ValueError("method must be one of %s, got %r" % (", ".join(METHODS), method))


def _nodes(plan, n_steps, method, device):
    """Device fp32 copies of the quadrature rule, cached per plan (a CUDA-graph capture of a call copies nothing)."""
    cache = plan.__dict__.setdefault("_ig_nodes", {})
    key = (n_steps, method, device.index)
    got = cache.get(key)
    if got is None:
        a, w = quadrature(n_steps, method)
        got = cache[key] = (torch.tensor(a, dtype=torch.float32, device=device),
                            torch.tensor(w, dtype=torch.float32, device=device))
    return got


def _default_steps_per_chunk(lib, dims, n_steps, cap=DEFAULT_SCRATCH_BYTES):
    """Largest steps_per_chunk <= n_steps whose scratch fits in `cap` bytes (host-only size queries); at least 1."""
    lo, hi = 1, n_steps
    while lo < hi:
        mid = (lo + hi + 1) // 2
        nb = lib.rd_integrated_gradients_scratch_bytes(C.byref(dims), mid)
        if 0 < nb <= cap:
            lo = mid
        else:
            hi = mid - 1
    return lo


def _check_target(target, B, n_classes):
    """None, an int, or an integer tensor [B]; the range is checked on the host (one sync for a device tensor)."""
    if target is None:
        return None
    if isinstance(target, (int, np.integer)):
        if not 0 <= int(target) < n_classes:
            raise ValueError("target %d out of range for %d classes" % (int(target), n_classes))
        return int(target)
    t = torch.as_tensor(target)
    if t.is_floating_point() or t.is_complex() or t.dtype == torch.bool:
        raise ValueError("target must hold integer class indices")
    if t.dim() == 0:
        t = t.expand(B)
    if tuple(t.shape) != (B,):
        raise ValueError("target must be an int or have shape [B=%d], got %s" % (B, tuple(t.shape)))
    lo, hi = torch.stack(torch.aminmax(t)).tolist()
    if lo < 0 or hi >= n_classes:
        raise ValueError("target values must lie in [0, %d), got [%d, %d]" % (n_classes, lo, hi))
    return t


def _target_tensor(target, B, device):
    if target is None:
        return None
    if isinstance(target, int):
        return torch.full((B,), target, dtype=torch.int64, device=device)
    return target.to(device=device, dtype=torch.int64).contiguous()


def _baseline(b, like):
    if b is None:
        return torch.zeros_like(like)
    b = torch.as_tensor(b).to(device=like.device, dtype=torch.float32)
    try:
        return torch.broadcast_to(b, like.shape).contiguous()
    except RuntimeError as exc:
        raise ValueError("baseline of shape %s does not broadcast to %s" % (tuple(b.shape), tuple(like.shape))) from exc


def integrated_gradients(model, src, static, times, lengths, target=None, baselines=None, n_steps=50,
                         method="gausslegendre", internal_batch_size=None, return_convergence_delta=False):
    """Integrated gradients of F = logits[b, target[b]] of an eval-mode Raindrop_v2 with respect to the value half of
    `src` and to `static`, along the straight path from the baseline to the input:

        attr_src[t, b, n]  = (x - x')[t, b, n] * sum_k w_k dF/dsrc[t, b, n] (x' + alpha_k (x - x'))
        attr_static[b, j]  = (s - s')[b, j]   * sum_k w_k dF/dstatic[b, j] (same points)

    Returns (attr_src [T, B, 2N], attr_static [B, d_static] or None), fp32 on the model's device, plus
    delta [B] = sum of the sample's attributions - (F(x) - F(x')) when return_convergence_delta (completeness error of
    the quadrature).  The mask half of attr_src is 0: the mask is not interpolated, nor are `times` and `lengths`.

    target:     None (the argmax class of the logits at x, chosen on the device), an int, or [B] class indices.
    baselines:  None = zeros for both -- in the normalised space that is each feature's mean, since mask_normalize
                centres the observed values -- or a pair (src_baseline, static_baseline), each None, a number or a
                tensor broadcastable to src / static (only the value half of src_baseline is read).
    method:     "gausslegendre" (default) or "riemann_trapezoid"; nodes and weights are computed in fp64 on the host.
    internal_batch_size: (sample, step) rows per chunk, i.e. max(1, internal_batch_size // B) steps per chunk.  Default:
                the largest chunk whose scratch fits in 1 GiB.  With obprop_mode 0 (auto) the ob-prop arithmetic follows
                the chunk's row count, so pin model._plan.obprop_mode for results independent of the chunking.

    The call is stream-ordered and sync-free (a device-tensor target costs one sync for its range check): it neither
    changes the parameters, their .grad, the model's dropout rng state nor a bound FlatAdam.  Raises ValueError for a
    model in training mode and RaindropB200Error without CUDA."""
    from .models_rd import Raindrop_v2, _device_of
    if not isinstance(model, Raindrop_v2):
        raise TypeError("integrated_gradients takes a raindrop_b200 Raindrop_v2 model, got %s" % type(model).__name__)
    if model.training:
        raise ValueError("integrated_gradients runs the model in eval arithmetic: call model.eval() first")
    n_steps = int(n_steps)
    quadrature(n_steps, method)                       # validates method and n_steps
    if internal_batch_size is not None and int(internal_batch_size) < 1:
        raise ValueError("internal_batch_size must be >= 1")
    plan = model._plan
    T, B = src.shape[0], src.shape[1]
    if src.dim() != 3 or T != plan.T or src.shape[2] != 2 * plan.N:
        raise ValueError("src must be [max_len=%d, B, 2*d_inp=%d], got %s" % (plan.T, 2 * plan.N, tuple(src.shape)))
    if model.static and static is None:
        raise ValueError("this model was built with static=True: `static` must be a tensor")
    if baselines is not None and (not isinstance(baselines, (tuple, list)) or len(baselines) != 2):
        raise ValueError("baselines must be None or a pair (src_baseline, static_baseline)")
    target = _check_target(target, B, plan.n_classes)
    device = _device_of(src)                          # RaindropB200Error without CUDA
    lib = L.load()
    tgt = _target_tensor(target, B, device)
    plan = model._prepare(device)
    f32 = dict(device=device, dtype=torch.float32)
    x = src.detach().to(**f32).contiguous()
    tm = times.detach().to(**f32).contiguous()
    ln = lengths.detach().to(device=device, dtype=torch.int64).contiguous()
    st = static.detach().to(**f32).contiguous() if model.static else None
    b_src, b_st = baselines if baselines is not None else (None, None)
    x0 = _baseline(b_src, x)
    st0 = _baseline(b_st, st) if st is not None else None

    params = [p.detach() for p in model.used_parameters()]
    if params[0].device != device:
        raise ValueError("the model's parameters are on %s, the inputs on %s" % (params[0].device, device))
    keep = [t if (t.dtype == torch.float32 and t.is_contiguous()) else t.float().contiguous() for t in params]
    P = L.RdParams()
    P.R_u = plan.R_u.data_ptr()
    for (_, path), t in zip(plan.fields, keep):
        RF._set_field(P, path, t.data_ptr())

    dims = plan.dims(B, False)
    if internal_batch_size is None:
        mc = _default_steps_per_chunk(lib, dims, n_steps)
    else:
        mc = max(1, int(internal_batch_size) // B)
    mc = min(mc, n_steps)
    nbytes = lib.rd_integrated_gradients_scratch_bytes(C.byref(dims), mc)
    if nbytes == 0:
        L.check(-2, "rd_integrated_gradients_scratch_bytes")
    key = (B, mc, dims.obprop_mode, device.index)
    cached = plan.__dict__.get("_ig_attr_scratch")
    if cached is None or cached[0] != key:             # one buffer per plan: a new shape replaces the old one
        plan.__dict__["_ig_attr_scratch"] = None
        cached = plan.__dict__["_ig_attr_scratch"] = (key, torch.empty(nbytes // 4, **f32))
    scratch = cached[1]
    alphas, weights = _nodes(plan, n_steps, method, device)

    attr_src = torch.empty_like(x)
    attr_st = torch.empty_like(st) if st is not None else None
    ends = torch.empty(2, B, plan.n_classes, **f32)
    L.check(lib.rd_raindrop_v2_integrated_gradients(C.byref(dims), C.byref(P), x.data_ptr(), L.ptr(st), tm.data_ptr(),
                                                    ln.data_ptr(), plan.node_scale.data_ptr(), x0.data_ptr(), L.ptr(st0),
                                                    L.ptr(tgt), alphas.data_ptr(), weights.data_ptr(), n_steps, mc,
                                                    scratch.data_ptr(), attr_src.data_ptr(), L.ptr(attr_st), ends.data_ptr(),
                                                    L.stream_ptr(device)), "rd_raindrop_v2_integrated_gradients")
    if not return_convergence_delta:
        return attr_src, attr_st
    idx = tgt if tgt is not None else ends[1].argmax(dim=1)
    f = ends.gather(2, idx.view(1, B, 1).expand(2, B, 1))[:, :, 0]          # [2, B]: F(x'), F(x)
    total = attr_src.sum(dim=(0, 2))
    if attr_st is not None:
        total = total + attr_st.sum(dim=1)
    return attr_src, attr_st, total - (f[1] - f[0])


def sensor_importance(attr_src, n_sensors):
    """Mean over samples of sum_t |attr_src[t, b, n]|, n < n_sensors: one importance score per sensor ([n_sensors])."""
    a = torch.as_tensor(attr_src)
    if a.dim() != 3 or a.shape[2] < n_sensors:
        raise ValueError("attr_src must be [T, B, >= n_sensors], got %s" % (tuple(a.shape),))
    return a[:, :, :n_sensors].abs().sum(dim=0).mean(dim=0)


def sensor_ranking(importance, names=None):
    """[N, 2] unicode array of (sensor index, sensor name) in descending importance, ties broken by the lower index:
    the layout of the reference's IG_density_scores_<dataset>.npy, whose column 0 removal_indices(level="set") reads.
    names: N sensor names (default: the indices).

    The reference ships those files but not the code that made them, so the exact recipe behind them (baseline, target,
    data split, aggregation) is not known; this ranking is the IG recipe of this module and is not claimed to reproduce
    the shipped files."""
    imp = torch.as_tensor(importance).detach().double().cpu().numpy().reshape(-1)
    n = imp.shape[0]
    if names is None:
        names = [str(i) for i in range(n)]
    names = [str(s) for s in names]
    if len(names) != n:
        raise ValueError("%d sensor names for %d sensors" % (len(names), n))
    order = np.lexsort((np.arange(n), -imp))
    return np.array([[str(i), names[i]] for i in order])
