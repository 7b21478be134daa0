"""Counterfactual explanations of Raindrop_v2, searched on the device in one call per batch
(rd_raindrop_v2_counterfactual): for each sample, the smallest sparse, bounded change of its recorded values that makes
the model predict a target class (Wachter et al. 2017; the elastic-net form of CEM, Dhurandhar et al. 2018).

    res = counterfactual(model.eval(), src, static, times, lengths)            # target: the runner-up class
    print(res.valid.float().mean(), res.sensors_changed[res.valid].sum(0))      # validity rate, sensors moved
    res = counterfactual(model.eval(), src, static, times, lengths, target=1, weights=1 / mad, lower=p1, upper=p99)

The search (also documented at rd_raindrop_v2_counterfactual in include/raindrop_b200.h):

* Target t_b: `target`, or by default the clean prediction's runner-up (the argmax over c != predicted, first index on
  ties; for a binary model the other class).
* Mutable set S_b, the threat model of adversarial.pgd: the value cells with mask > 0 of the sensors in `sensors`, plus
  the statics when perturb_static.  The mask half, times and lengths never change; an element with delta = 0 is
  returned as x bit for bit.
* Per element (given per sensor, then per static column): a weight w > 0 and a box [lower, upper] in normalised units;
  the effective box is [min(lower, x), max(upper, x)], so delta = 0 is always feasible.
* Objective over delta on S_b:  c_b max(0, kappa - m(x + delta)) + beta ||w delta||_1 + ||w delta||_2^2, with the logit
  margin m = z_t - max_{c != t} z_c (first index on ties).
* n_search rounds per replica; each restarts FISTA at the replica's start point (x_0 = y_0) and runs n_steps steps
      g = c grad(hinge)(y_k) + 2 w^2 y_k
      x_{k+1} = clip_box(S(y_k - alpha g, alpha beta w))            S the soft-threshold
      y_{k+1} = clip_box(x_{k+1} + k/(k+3) (x_{k+1} - x_k))
  with a forward at every y_k, k = 0 .. n_steps.  Element arithmetic is fp32; sums, distances and c are fp64.
* A point is valid when m > 0 and m >= kappa; its distance is d = beta ||w delta||_1 + ||w delta||_2^2.  The result is
  the valid evaluated point of smallest d over all rounds, steps and replicas (ties: the earliest (round, step), then
  the lowest replica).  Without one: x, the clean logits and d = +inf.
* Bisection on c per (sample, replica), lo = 0, hi = +inf, c = c_init; after each round: a valid point found:
  hi = min(hi, c), c = (lo + hi) / 2; else lo = max(lo, c), c = (lo + hi) / 2 if hi < inf, else 10 c.
* Restarts: n_restarts independent replicas per sample.  Replica 0 starts at delta = 0, replica r >= 1 at
  clip_box(init_scale (2u - 1)) on S_b with u uniform from the Philox stream at site 103, key (seed, step), index
  (b R + r)(T N + d_static) + e.  They matter for the reason PGD's random start does: at d_ob = 1 the lift relu(v R_u)
  has zero gradient at every value of the wrong sign, so such a cell never leaves delta = 0 from a zero start.
"""
import ctypes as C
import math
from dataclasses import dataclass

import numpy as np
import torch

from . import lib as L
from .adversarial import _check_key, _sensor_mask
from .attribution import _Call, _check_call, _largest_chunk
from .uncertainty import _device_key


@dataclass
class CounterfactualResult:
    """From the device: src [T, B, 2N] and static [B, d_static] (None without a static branch) the returned inputs;
    logits [B, C] at them and clean_logits [B, C] at x; target [B] int64; valid [B] bool; distance [B] float64
    (beta ||w delta||_1 + ||w delta||_2^2, +inf when invalid); c [B, R] float64 (each replica's loss weight after its
    last bisection update); round_valid [B, R, n_search] bool (whether the round found a valid point).
    From those with torch ops: l1 [B] = ||w delta||_1 and l2 [B] = ||w delta||_2 (float64, delta = returned - x over the
    mutable elements), l0 [B] int64 the number of elements changed, sensors_changed [B, d_inp] bool (some value cell of
    the sensor changed)."""
    src: object
    static: object
    logits: object
    clean_logits: object
    target: object
    valid: object
    distance: object
    c: object
    round_valid: object
    l1: object
    l2: object
    l0: object
    sensors_changed: object


def _per_element(v, name, N, ds, default, positive=False):
    """None, a number, or a 1-D [d_inp] / [d_inp + d_static] array -> float32 numpy [N + ds] (the statics part from
    `default` when only d_inp values are given).  NaN is refused; weights must be finite and > 0."""
    out = np.full(N + ds, default, dtype=np.float64)
    if v is not None:
        a = torch.as_tensor(v).detach().cpu().double().numpy() if torch.is_tensor(v) else np.asarray(v, dtype=np.float64)
        if a.ndim == 0:
            out[:] = float(a)
        elif a.shape == (N,):
            out[:N] = a
        elif a.shape == (N + ds,) and ds > 0:
            out[:] = a
        else:
            raise ValueError("%s must be a number or have shape [d_inp=%d]%s, got %s" %
                             (name, N, " or [d_inp + d_static=%d]" % (N + ds) if ds else "", tuple(a.shape)))
    if np.isnan(out).any():
        raise ValueError("%s must not hold NaN" % name)
    if positive and not (np.all(np.isfinite(out)) and np.all(out > 0)):
        raise ValueError("%s must be finite and > 0" % name)
    return out.astype(np.float32)


def _check_settings(kappa, beta, c_init, step_size, n_search, n_steps, n_restarts, init_scale):
    """Host checks of the search's settings -> an RdCfOptions without perturb_static."""
    o = L.RdCfOptions()
    for name, v, pos in (("kappa", kappa, False), ("beta", beta, False), ("c_init", c_init, True),
                         ("step_size", step_size, True), ("init_scale", init_scale, False)):
        v = float(v)
        if not math.isfinite(v) or v < 0 or (pos and v == 0):
            raise ValueError("%s must be finite and %s 0, got %r" % (name, ">" if pos else ">=", v))
        setattr(o, name, v)
    for name, v, lo in (("n_search", n_search, 1), ("n_steps", n_steps, 0), ("n_restarts", n_restarts, 1)):
        v = int(v)
        if not lo <= v < 1 << 31:
            raise ValueError("%s must be in [%d, 2^31), got %d" % (name, lo, v))
        setattr(o, name, v)
    return o


def _chunk_scratch(cl, dims, B, R, internal_batch_size):
    """(samples per chunk, scratch) as _Call.chunk_scratch picks them, for a query that takes the chunk before R."""
    def nbytes(c):
        return cl.lib.rd_counterfactual_scratch_bytes(C.byref(dims), c, R)
    chunk = _largest_chunk(nbytes, B) if internal_batch_size is None else min(B, int(internal_batch_size))
    nb = nbytes(chunk)
    if nb == 0:
        L.check(-2, "rd_counterfactual_scratch_bytes")
    return chunk, cl.scratch("_cf_scratch", (B, chunk, R, dims.obprop_mode, cl.device.index), nb)


def _device_array(plan, name, arr, device):
    """fp32 device copy of a host array, cached per plan by value (a CUDA-graph capture after an eager call with the same
    values copies nothing); a copy read under capture is held for the plan's lifetime."""
    cache = plan.__dict__.setdefault("_cf_arrays", {})
    k = (arr.tobytes(), device.index)
    got = cache.get(name)
    if got is None or got[0] != k:
        got = cache[name] = (k, torch.from_numpy(arr).to(device))
    if device.type == "cuda" and torch.cuda.is_current_stream_capturing():
        held = plan.__dict__.setdefault("_cf_arrays_captured", [])
        if not any(t is got[1] for t in held):
            held.append(got[1])
    return got[1]


def counterfactual(model, src, static, times, lengths, target=None, *, sensors=None, perturb_static=False, lower=None,
                   upper=None, weights=None, kappa=0.0, beta=0.1, c_init=1.0, step_size=0.01, n_search=5, n_steps=100,
                   n_restarts=1, init_scale=0.5, seed=0, step=0, internal_batch_size=None):
    """Counterfactuals of an eval-mode Raindrop_v2 (see the module docstring for the algorithm).  Returns a
    CounterfactualResult of tensors on the model's device.

    target:     None (the clean prediction's runner-up), an int, or [B] class indices.
    sensors:    None (every sensor) or a bool [d_inp]: only those sensors' observed cells may change.
    perturb_static: the static vector may change too (needs a model with a static branch).
    lower, upper: the box, in normalised units: None (unbounded), a number, or per sensor [d_inp] (then per static
                column: [d_inp + d_static]).  lower <= upper.
    weights:    w > 0 of the distance, same shapes (default 1; Wachter et al. use the inverse median absolute deviation).
    kappa:      the margin the target must win by (>= 0); beta: the L1 weight (>= 0); c_init: the hinge's first weight.
    step_size:  FISTA's alpha; n_search bisection rounds of n_steps steps; n_restarts replicas per sample.
    init_scale: half-width of the restarts' uniform start; seed, step: their Philox key.
    internal_batch_size: samples per chunk (each on n_restarts rows).  Default: the largest chunk whose scratch fits in
                1 GiB.  Results are bitwise independent of it once model._plan.obprop_mode is pinned.

    Stream-ordered and sync-free apart from the host checks (a device-tensor target costs one sync for its range check);
    it changes neither the parameters, their .grad, the model's rng state nor a bound FlatAdam.  Raises ValueError for a
    model in training mode or invalid arguments, and RaindropB200Error without CUDA."""
    _check_call("counterfactual", model, src, static, None, internal_batch_size)
    opt = _check_settings(kappa, beta, c_init, step_size, n_search, n_steps, n_restarts, init_scale)
    seed, step = _check_key(seed, step)
    if perturb_static and not model.static:
        raise ValueError("perturb_static needs a model with a static branch")
    opt.perturb_static = int(bool(perturb_static))
    plan = model._plan
    N, ds = plan.N, plan.d_static
    if sensors is not None:
        _sensor_mask(sensors, N, "cpu")               # shape and dtype checked before anything touches the device
    w = _per_element(weights, "weights", N, ds, 1.0, positive=True)
    lo = _per_element(lower, "lower", N, ds, -np.inf)
    hi = _per_element(upper, "upper", N, ds, np.inf)
    if np.any(lo > hi):
        raise ValueError("lower must be <= upper everywhere")
    with torch.no_grad():
        cl = _Call(model, src, static, times, lengths, target, False)
        lib, B, dev, R = cl.lib, src.shape[1], cl.device, opt.n_restarts
        sens = _sensor_mask(sensors, N, dev)
        dims = plan.dims(B, False)
        spc, scratch = _chunk_scratch(cl, dims, B, R, internal_batch_size)
        key = _device_key(plan, seed, step, dev)
        wd, lod, hid = (_device_array(plan, n, a, dev) for n, a in (("w", w), ("lo", lo), ("hi", hi)))
        f32 = dict(device=dev, dtype=torch.float32)
        src_cf = torch.empty_like(cl.x)
        st_cf = torch.empty_like(cl.st) if cl.st is not None else None
        logits = torch.empty(B, plan.n_classes, **f32)
        clean = torch.empty(B, plan.n_classes, **f32)
        tgt = torch.empty(B, dtype=torch.int64, device=dev)
        valid = torch.empty(B, dtype=torch.bool, device=dev)
        distance = torch.empty(B, dtype=torch.float64, device=dev)
        c = torch.empty(B, R, dtype=torch.float64, device=dev)
        round_valid = torch.empty(B, R, opt.n_search, dtype=torch.bool, device=dev)
        L.check(lib.rd_raindrop_v2_counterfactual(
            C.byref(dims), C.byref(cl.params), cl.x.data_ptr(), L.ptr(cl.st), cl.tm.data_ptr(), cl.ln.data_ptr(),
            plan.node_scale.data_ptr(), L.ptr(cl.tgt), L.ptr(sens), wd.data_ptr(), lod.data_ptr(), hid.data_ptr(),
            C.byref(opt), key.data_ptr(), spc, scratch.data_ptr(), src_cf.data_ptr(), L.ptr(st_cf), logits.data_ptr(),
            clean.data_ptr(), tgt.data_ptr(), valid.data_ptr(), distance.data_ptr(), c.data_ptr(), round_valid.data_ptr(),
            L.stream_ptr(dev)), "rd_raindrop_v2_counterfactual")
        l1, l2, l0, changed = _distances(cl.x, cl.st, src_cf, st_cf, wd, N)
    return CounterfactualResult(src_cf, st_cf, logits, clean, tgt, valid, distance, c, round_valid, l1, l2, l0, changed)


def _distances(x, st, src_cf, st_cf, w, N):
    """(l1, l2, l0, sensors_changed) of the returned inputs against x, with torch ops (no sync)."""
    d = src_cf[:, :, :N].double() - x[:, :, :N].double()                       # [T, B, N]
    moved = src_cf[:, :, :N].view(torch.int32) != x[:, :, :N].view(torch.int32)
    wd = d * w[:N].double()
    l1 = wd.abs().sum(dim=(0, 2))
    l2 = (wd * wd).sum(dim=(0, 2))
    l0 = moved.sum(dim=(0, 2))
    if st is not None and st_cf is not None:
        ds_ = st_cf.double() - st.double()
        ws = ds_ * w[N:].double()
        l1 = l1 + ws.abs().sum(1)
        l2 = l2 + (ws * ws).sum(1)
        l0 = l0 + (st_cf.view(torch.int32) != st.view(torch.int32)).sum(1)
    return l1, l2.sqrt(), l0, moved.any(dim=0)
