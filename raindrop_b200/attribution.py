"""Attribution of Raindrop_v2, computed on the device in one call per batch, and the per-sensor ranking that the
reference's leave-sensors-out experiment with feature_removal_level='set' reads (code/Raindrop.py:227-231,
IG_density_scores_<dataset>.npy):

* integrated_gradients (rd_raindrop_v2_integrated_gradients): per input value, along the straight path from a baseline;
* shapley_value_sampling and feature_ablation (rd_raindrop_v2_coalition_attribution): per sensor (group), of REMOVING
  it -- replacing its value columns by the baseline, as the experiment does -- with the static vector one more player;
* the same two with feature_mask (rd_raindrop_v2_cell_coalition_attribution): per player of a map of the value cells
  (t, b, n), e.g. (sensor, time window) players from time_window_mask -- "what does removing heart rate in hours 12-18
  do to this prediction?".  Removing a player writes the baseline into its cells of the value half; cells with id -1
  belong to no player and keep x;
* kernel_shap (rd_raindrop_v2_kernel_shap): Shapley values over the same players by KernelSHAP, the efficiency-
  constrained weighted regression over sampled coalitions (any budget; all_coalitions gives the exact values).

    attr_src, attr_static = integrated_gradients(model.eval(), src, static, times, lengths, target=y)
    ranking = sensor_ranking(sensor_importance(attr_src, model.d_inp), names)
    phi, phi_static = shapley_value_sampling(model.eval(), src, static, times, lengths, target=y)
    ranking = sensor_ranking(phi.abs().mean(dim=0), names)
    idx = data.removal_indices(B, model.d_inp, 0.5, level="set", density_scores=ranking[:, 0])
    mask, n_win = time_window_mask(times, 6.0, sensor_groups=model.d_inp)       # 6 units of `times` per window
    phi, phi_static = shapley_value_sampling(model.eval(), src, static, times, lengths, target=y, feature_mask=mask)
    per_cell = phi.view(-1, n_win, model.d_inp)                                  # [B, window, sensor]

Argument names follow Captum's IntegratedGradients, ShapleyValueSampling and FeatureAblation.
"""
import ctypes as C
import math

import numpy as np
import torch

from . import functional as RF
from . import lib as L

METHODS = ("gausslegendre", "riemann_trapezoid")
DEFAULT_SCRATCH_BYTES = 1 << 30      # default chunking: the largest one whose scratch fits in 1 GiB
RD_ATTR_SHAPLEY, RD_ATTR_ABLATION = 0, 1


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


def _largest_chunk(scratch_bytes, n, cap=DEFAULT_SCRATCH_BYTES):
    """Largest chunk c <= n whose scratch_bytes(c) fits in `cap` bytes (host-only size queries); at least 1."""
    lo, hi = 1, max(1, n)
    while lo < hi:
        mid = (lo + hi + 1) // 2
        nb = scratch_bytes(mid)
        if 0 < nb <= cap:
            lo = mid
        else:
            hi = mid - 1
    return lo


def _default_steps_per_chunk(lib, dims, n_steps, cap=DEFAULT_SCRATCH_BYTES):
    """Largest steps_per_chunk <= n_steps whose integrated-gradients scratch fits in `cap` bytes; at least 1."""
    return _largest_chunk(lambda c: lib.rd_integrated_gradients_scratch_bytes(C.byref(dims), c), n_steps, cap)


def _default_coalitions_per_chunk(lib, dims, n_players, n_coalitions, cap=DEFAULT_SCRATCH_BYTES):
    """Largest coalitions_per_chunk <= n_coalitions whose coalition-attribution scratch fits in `cap` bytes; at least 1."""
    return _largest_chunk(lambda c: lib.rd_coalition_attribution_scratch_bytes(C.byref(dims), n_players, c), n_coalitions,
                          cap)


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


def _check_call(fn, model, src, static, baselines, internal_batch_size):
    """The argument checks every attribution call shares (host only, before anything touches the device)."""
    from .models_rd import Raindrop_v2
    if not isinstance(model, Raindrop_v2):
        raise TypeError("%s takes a raindrop_b200 Raindrop_v2 model, got %s" % (fn, type(model).__name__))
    if model.training:
        raise ValueError("%s runs the model in eval arithmetic: call model.eval() first" % fn)
    if internal_batch_size is not None and int(internal_batch_size) < 1:
        raise ValueError("internal_batch_size must be >= 1")
    plan = model._plan
    if src.dim() != 3 or src.shape[0] != plan.T or src.shape[2] != 2 * plan.N:
        raise ValueError("src must be [max_len=%d, B, 2*d_inp=%d], got %s" % (plan.T, 2 * plan.N, tuple(src.shape)))
    if model.static and static is None:
        raise ValueError("this model was built with static=True: `static` must be a tensor")
    if baselines is not None and (not isinstance(baselines, (tuple, list)) or len(baselines) != 2):
        raise ValueError("baselines must be None or a pair (src_baseline, static_baseline)")


class _Call:
    """The device-side operands of one attribution call: inputs and baselines as contiguous fp32 / int64 device tensors,
    the target, and the parameter pointers (rd_params; `keep` holds the tensors they point into).  baselines=False: a
    call without baselines (x0 and st0 are None)."""

    def __init__(self, model, src, static, times, lengths, target, baselines):
        from .models_rd import _device_of
        B = src.shape[1]
        target = _check_target(target, B, model._plan.n_classes)
        self.device = device = _device_of(src)          # RaindropB200Error without CUDA
        self.lib = L.load()
        self.tgt = _target_tensor(target, B, device)
        self.plan = plan = model._prepare(device)
        f32 = dict(device=device, dtype=torch.float32)
        self.x = src.detach().to(**f32).contiguous()
        self.tm = times.detach().to(**f32).contiguous()
        self.ln = lengths.detach().to(device=device, dtype=torch.int64).contiguous()
        self.st = static.detach().to(**f32).contiguous() if model.static else None
        if baselines is False:
            self.x0 = self.st0 = None
        else:
            b_src, b_st = baselines if baselines is not None else (None, None)
            self.x0 = _baseline(b_src, self.x)
            self.st0 = _baseline(b_st, self.st) if self.st is not None else None

        params = [p.detach() for p in model.used_parameters()]
        if params[0].device != device:
            raise ValueError("the model's parameters are on %s, the inputs on %s" % (params[0].device, device))
        self.keep = [t if (t.dtype == torch.float32 and t.is_contiguous()) else t.float().contiguous() for t in params]
        self.params = L.RdParams()
        self.params.R_u = plan.R_u.data_ptr()
        for (_, path), t in zip(plan.fields, self.keep):
            RF._set_field(self.params, path, t.data_ptr())

    def scratch(self, name, key, nbytes):
        """fp32 scratch of at least `nbytes`, one buffer per plan and entry point: a new key, or a call that needs more
        bytes than the buffer holds, replaces the old one.  A buffer used by a call under CUDA-graph capture is also held
        for the plan's lifetime (plan._scratch_captured), so the graph's replays stay valid after a later call has
        replaced it."""
        plan = self.plan
        cached = plan.__dict__.get(name)
        if cached is None or cached[0] != key or cached[1].numel() * 4 < nbytes:
            plan.__dict__[name] = None
            cached = plan.__dict__[name] = (key, torch.empty(nbytes // 4, device=self.device, dtype=torch.float32))
        if self.device.type == "cuda" and torch.cuda.is_current_stream_capturing():
            held = plan.__dict__.setdefault("_scratch_captured", [])
            if not any(t is cached[1] for t in held):
                held.append(cached[1])
        return cached[1]


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
    _check_call("integrated_gradients", model, src, static, baselines, internal_batch_size)
    n_steps = int(n_steps)
    quadrature(n_steps, method)                       # validates method and n_steps
    cl = _Call(model, src, static, times, lengths, target, baselines)
    lib, plan, B = cl.lib, cl.plan, src.shape[1]

    dims = plan.dims(B, False)
    if internal_batch_size is None:
        mc = _default_steps_per_chunk(lib, dims, n_steps)
    else:
        mc = max(1, int(internal_batch_size) // B)
    mc = min(mc, n_steps)
    nbytes = lib.rd_integrated_gradients_scratch_bytes(C.byref(dims), mc)
    if nbytes == 0:
        L.check(-2, "rd_integrated_gradients_scratch_bytes")
    scratch = cl.scratch("_ig_attr_scratch", (B, mc, dims.obprop_mode, cl.device.index), nbytes)
    alphas, weights = _nodes(plan, n_steps, method, cl.device)

    attr_src = torch.empty_like(cl.x)
    attr_st = torch.empty_like(cl.st) if cl.st is not None else None
    ends = torch.empty(2, B, plan.n_classes, device=cl.device, dtype=torch.float32)
    L.check(lib.rd_raindrop_v2_integrated_gradients(C.byref(dims), C.byref(cl.params), cl.x.data_ptr(), L.ptr(cl.st),
                                                    cl.tm.data_ptr(), cl.ln.data_ptr(), plan.node_scale.data_ptr(),
                                                    cl.x0.data_ptr(), L.ptr(cl.st0), L.ptr(cl.tgt), alphas.data_ptr(),
                                                    weights.data_ptr(), n_steps, mc, scratch.data_ptr(), attr_src.data_ptr(),
                                                    L.ptr(attr_st), ends.data_ptr(), L.stream_ptr(cl.device)),
            "rd_raindrop_v2_integrated_gradients")
    if not return_convergence_delta:
        return attr_src, attr_st
    f = _endpoint_values(ends, cl.tgt)
    total = attr_src.sum(dim=(0, 2))
    if attr_st is not None:
        total = total + attr_st.sum(dim=1)
    return attr_src, attr_st, total - (f[1] - f[0])


def _endpoint_values(ends, tgt):
    """[2, B]: F(x') and F(x) from the endpoint logits [2, B, n_classes] (tgt None: the argmax class at x)."""
    B = ends.shape[1]
    idx = tgt if tgt is not None else ends[1].argmax(dim=1)
    return ends.gather(2, idx.view(1, B, 1).expand(2, B, 1))[:, :, 0]


# ---- coalition attribution: Shapley-value sampling and leave-one-out ablation -----------------------------------------
def sample_permutations(n_players, n_samples, seed=0):
    """[n_samples, n_players] int64: n_samples permutations of range(n_players) drawn by numpy.random.default_rng(seed),
    one rng.permutation call each.  The same seed gives the same permutations."""
    n_players, n_samples = int(n_players), int(n_samples)
    if n_players < 1 or n_samples < 1:
        raise ValueError("n_players and n_samples must be >= 1, got %d and %d" % (n_players, n_samples))
    rng = np.random.default_rng(seed)
    return np.stack([rng.permutation(n_players) for _ in range(n_samples)]).astype(np.int64)


def _check_groups(sensor_groups, N):
    """int64 numpy [N] with values in [0, G), every group non-empty (default: one group per sensor), and G."""
    if sensor_groups is None:
        return np.arange(N, dtype=np.int64), N
    g = torch.as_tensor(sensor_groups)
    if g.is_floating_point() or g.is_complex() or g.dtype == torch.bool:
        raise ValueError("sensor_groups must hold integer group indices")
    g = g.cpu().numpy().astype(np.int64)
    if g.shape != (N,):
        raise ValueError("sensor_groups must have shape [d_inp=%d], got %s" % (N, g.shape))
    if g.min() < 0:
        raise ValueError("sensor_groups values must be >= 0, got %d" % g.min())
    G = int(g.max()) + 1
    empty = np.setdiff1d(np.arange(G), g)
    if empty.size:
        raise ValueError("sensor group(s) %s have no sensor: groups must be 0..G-1, each non-empty" % empty.tolist())
    return g, G


def _check_permutations(permutations, P):
    p = torch.as_tensor(permutations)
    if p.is_floating_point() or p.is_complex() or p.dtype == torch.bool:
        raise ValueError("permutations must hold integer player indices")
    p = p.cpu().numpy().astype(np.int64)
    if p.ndim != 2 or p.shape[1] != P or p.shape[0] < 1:
        raise ValueError("permutations must have shape [m >= 1, n_players=%d], got %s" % (P, p.shape))
    bad = np.nonzero(np.any(np.sort(p, axis=1) != np.arange(P), axis=1))[0]
    if bad.size:
        raise ValueError("permutations row %d is not a permutation of range(%d)" % (bad[0], P))
    return p


def _device_int32(plan, kind, arr, device):
    """Device int32 copy of a small host array, cached per plan (a CUDA-graph capture of a call copies nothing)."""
    cache = plan.__dict__.setdefault("_coal_" + kind, {})
    key = (arr.shape, arr.tobytes(), device.index)
    got = cache.get(key)
    if got is None:
        got = cache[key] = torch.tensor(arr, dtype=torch.int32, device=device)
    return got


def _device_cells(plan, arr, device):
    """Device int32 copy of a host feature mask, cached per plan in ONE entry that a mask of other content replaces:
    repeated calls with the same mask, and a CUDA-graph capture after an eager call with it, copy nothing, while a loop
    over batches with per-sample host masks keeps a single mask on the device.  A copy read by a call under CUDA-graph
    capture is also held for the plan's lifetime (plan._coal_cells_captured), so replays stay valid after later calls
    replace the entry."""
    key = (arr.shape, arr.tobytes(), device.index)
    cached = plan.__dict__.get("_coal_cells")
    if cached is None or cached[0] != key:
        plan.__dict__["_coal_cells"] = None
        cached = plan.__dict__["_coal_cells"] = (key, torch.tensor(arr, dtype=torch.int32, device=device))
    if device.type == "cuda" and torch.cuda.is_current_stream_capturing():
        held = plan.__dict__.setdefault("_coal_cells_captured", [])
        if not any(t is cached[1] for t in held):
            held.append(cached[1])
    return cached[1]


def _check_feature_mask(feature_mask, T, B, N):
    """The integer tensor feature_mask, [T, N] or [T, B, N] with ids >= -1, on the device it was given on, and
    G = max id + 1 >= 1 (one sync for a device tensor)."""
    m = torch.as_tensor(feature_mask)
    if m.is_floating_point() or m.is_complex() or m.dtype == torch.bool:
        raise ValueError("feature_mask must hold integer player ids")
    if tuple(m.shape) not in ((T, N), (T, B, N)):
        raise ValueError("feature_mask must have shape [max_len=%d, d_inp=%d] or [max_len=%d, B=%d, d_inp=%d], got %s"
                         % (T, N, T, B, N, tuple(m.shape)))
    lo, hi = torch.stack(torch.aminmax(m)).tolist()
    if lo < -1:
        raise ValueError("feature_mask ids must be >= -1 (-1: the cell belongs to no player), got %d" % lo)
    if hi < 0:
        raise ValueError("feature_mask names no player: every id is -1")
    if hi >= 1 << 30:
        raise ValueError("feature_mask ids must be < 2^30, got %d" % hi)
    return m, hi + 1


def _cell_players(plan, mask, device):
    """(device int32 map, stride_t, stride_b) for rd_raindrop_v2_cell_coalition_attribution.  A host mask goes through
    the plan's one-entry cache (_device_cells); a device mask is used in place when it is int32 with unit stride along
    the sensors, and its strides select the layout (an expanded [T, B, N] view works)."""
    if mask.device.type == "cpu":
        mask = _device_cells(plan, np.ascontiguousarray(mask.numpy().astype(np.int32)), device)
    else:
        mask = mask.to(device=device, dtype=torch.int32)
        if mask.stride(-1) != 1:
            mask = mask.contiguous()
    if mask.dim() == 2:
        return mask, mask.stride(0), 0
    return mask, mask.stride(0), mask.stride(1)


def time_window_mask(times, window, n_windows=None, sensor_groups=None):
    """(mask [T, B, N] int32 on the device of `times`, n_windows): a per-sample feature_mask of (sensor group, time
    window) players for shapley_value_sampling and feature_ablation.  The value cell (t, b, n) belongs to player
    w * G + g, g = sensor_groups[n], with the window of its row

        w = min(floor(times[t, b] / window), n_windows - 1)        (window in the units of `times`, > 0)

    so players 0..G-1 are the groups in window 0, G..2G-1 in window 1, and so on: phi.view(B, n_windows, G).
    Padding rows -- rows t > 0 with times[t, b] == 0, the data pipeline's padding -- get -1 (no player): the ob-prop
    GEMM mixes all T steps of a sensor, so a nonzero baseline written into padding rows would change F.  Row 0 is always
    a real row, also when the first timestamp is 0 (first_time_zero data).  A window with no row in a sample is a player
    with no cell there: it gets exactly 0.

    times:          [T, B] (src's timestamps).
    n_windows:      default max(1, ceil(max(times) / window)), one sync; give it to share one layout over batches.
    sensor_groups:  required: d_inp (an int, one group per sensor) or an integer array [d_inp] of groups 0..G-1, each
                    non-empty, as for sensor_groups of feature_ablation."""
    tm = torch.as_tensor(times)
    if tm.dim() != 2 or tm.is_complex():
        raise ValueError("times must be a real [max_len, B] tensor, got shape %s" % (tuple(tm.shape),))
    window = float(window)
    if not (window > 0 and math.isfinite(window)):
        raise ValueError("window must be a positive finite number, got %r" % window)
    if sensor_groups is None:
        raise ValueError("time_window_mask needs sensor_groups: d_inp (one group per sensor) or a group array [d_inp]")
    if isinstance(sensor_groups, (int, np.integer)):
        if int(sensor_groups) < 1:
            raise ValueError("sensor_groups as a sensor count must be >= 1, got %d" % int(sensor_groups))
        groups, G = np.arange(int(sensor_groups), dtype=np.int64), int(sensor_groups)
    else:
        g = torch.as_tensor(sensor_groups)
        if g.dim() != 1:
            raise ValueError("sensor_groups must be an int or a 1-D array [d_inp], got shape %s" % (tuple(g.shape),))
        groups, G = _check_groups(g, g.shape[0])
    t = tm.detach().double()
    if n_windows is None:
        n_windows = max(1, math.ceil(float(t.max()) / window)) if t.numel() else 1
    n_windows = int(n_windows)
    if n_windows < 1:
        raise ValueError("n_windows must be >= 1, got %d" % n_windows)
    w = torch.floor(t / window).clamp_(0, n_windows - 1).long()                              # [T, B]
    row = torch.arange(t.shape[0], device=t.device)[:, None]
    pad = (row > 0) & (t == 0)
    ids = w[:, :, None] * G + torch.as_tensor(groups, device=t.device)[None, None, :]       # [T, B, N]
    return torch.where(pad[:, :, None], -1, ids).to(torch.int32).contiguous(), n_windows


def _players(model, src, sensor_groups, feature_mask):
    """(groups [N] or None, feature mask or None, G, P = G + the static player) of an attribution call."""
    if feature_mask is None:
        groups, G = _check_groups(sensor_groups, model._plan.N)
        cells = None
    else:
        if sensor_groups is not None:
            raise ValueError("give sensor_groups or feature_mask, not both")
        cells, G = _check_feature_mask(feature_mask, model._plan.T, src.shape[1], model._plan.N)
        groups = None
    return groups, cells, G, G + (1 if model.static else 0)


def _coalition_attribution(fn, method, model, src, static, times, lengths, target, baselines, sensor_groups,
                           orders_host, internal_batch_size, feature_mask=None):
    """attr [B, P] of rd_raindrop_v2_coalition_attribution (sensor groups) or rd_raindrop_v2_cell_coalition_attribution
    (feature_mask), the endpoint logits [2, B, ncls], the target and G."""
    groups, cells, G, P = _players(model, src, sensor_groups, feature_mask)
    if feature_mask is not None:
        fn = "rd_raindrop_v2_cell_coalition_attribution"
    orders = orders_host(P) if method == RD_ATTR_SHAPLEY else None
    cl = _Call(model, src, static, times, lengths, target, baselines)
    lib, plan, device, B = cl.lib, cl.plan, cl.device, src.shape[1]
    if method == RD_ATTR_SHAPLEY:
        m = orders.shape[0]
        n_coal = m * (P - 1)
        orders_d = _device_int32(plan, "orders", orders, device)
    else:
        m, n_coal, orders_d = 0, P, None
    if feature_mask is None:
        player = _device_int32(plan, "players", groups, device)
    else:
        player, stride_t, stride_b = _cell_players(plan, cells, device)

    dims = plan.dims(B, False)
    if internal_batch_size is None:
        cc = _default_coalitions_per_chunk(lib, dims, P, n_coal)
    else:
        cc = max(1, int(internal_batch_size) // B)
    cc = max(1, min(cc, n_coal))
    nbytes = lib.rd_coalition_attribution_scratch_bytes(C.byref(dims), P, cc)
    if nbytes == 0:
        L.check(-2, "rd_coalition_attribution_scratch_bytes")
    # the scratch layout follows (B, P, cc) on every call, so a buffer that is large enough is reused: with feature_mask
    # P changes whenever a batch does not reach the last time window, and that must not reallocate the scratch
    scratch = cl.scratch("_coal_attr_scratch", device.index, nbytes)

    attr = torch.empty(B, P, device=device, dtype=torch.float32)
    ends = torch.empty(2, B, plan.n_classes, device=device, dtype=torch.float32)
    head = (C.byref(dims), C.byref(cl.params), cl.x.data_ptr(), L.ptr(cl.st), cl.tm.data_ptr(), cl.ln.data_ptr(),
            plan.node_scale.data_ptr(), cl.x0.data_ptr(), L.ptr(cl.st0), L.ptr(cl.tgt), player.data_ptr())
    tail = (P, L.ptr(orders_d), m, method, cc, scratch.data_ptr(), attr.data_ptr(), ends.data_ptr(), L.stream_ptr(device))
    if feature_mask is None:
        rc = lib.rd_raindrop_v2_coalition_attribution(*head, *tail)
    else:
        rc = lib.rd_raindrop_v2_cell_coalition_attribution(*head, stride_t, stride_b, *tail)
    L.check(rc, fn)
    return attr, ends, cl.tgt, G


def _split(attr, G):
    return attr[:, :G], (attr[:, G] if attr.shape[1] > G else None)


def feature_ablation(model, src, static, times, lengths, target=None, baselines=None, sensor_groups=None,
                     internal_batch_size=None, feature_mask=None):
    """Leave-one-out ablation of F = logits[b, target[b]] of an eval-mode Raindrop_v2 over sensor groups and the static
    vector:

        attr[b, g] = F(x) - F(x with player g removed)

    Players: the groups of `sensor_groups` (an int array [N] with values in [0, G), each group non-empty; default: one
    group per sensor) and, when the model has statics, the static vector.  Removing a group replaces the value columns
    src[:, b, n] of its sensors by the baseline (default 0: the reference's removal, data.remove_features_); removing
    the static player replaces static[b] by its baseline.  The mask half, `times` and `lengths` never change.
    Returns (attr_sensors [B, G], attr_static [B] or None), fp32 on the model's device.

    feature_mask: instead of sensor_groups (giving both is a ValueError), an integer map of the value cells (Captum's
                name): [T, N] shared by the batch or [T, B, N] per sample (time_window_mask builds (sensor, time window)
                players).  Ids 0..G-1, G = max id + 1, are players, removing one writes the baseline into its cells of
                the value half; -1 marks a cell of no player, which keeps x; the static vector is player G as before.
                An id may have no cell (a time window can be empty in a batch): that player gets exactly 0.  The
                result is (attr_players [B, G], attr_static [B] or None).  A host mask is kept on the device in a
                one-entry cache per model that a mask of other content replaces: repeated calls with the same mask and
                a CUDA-graph capture after an eager call with it copy nothing, and a loop over per-sample host masks
                holds one mask on the device.  A device mask costs one sync for its range check (so it cannot be captured)
                and is read in place.
    target, baselines: as for integrated_gradients.  A static baseline equal to `static` holds the statics fixed (their
                attribution is then exactly 0).
    internal_batch_size: (sample, coalition) rows per chunk.  Default: the largest chunk whose scratch fits in 1 GiB.

    The call runs one forward on 2B rows for F(x') and F(x) and one forward per coalition, all on the device, and is
    stream-ordered, sync-free (a device-tensor target or sensor_groups costs one sync) and CUDA-graph capturable; it
    changes neither the parameters, their .grad, the dropout rng state nor a bound FlatAdam.  Raises ValueError for a
    model in training mode or bad arguments, TypeError for another model class and RaindropB200Error without CUDA."""
    _check_call("feature_ablation", model, src, static, baselines, internal_batch_size)
    attr, _, _, G = _coalition_attribution("rd_raindrop_v2_coalition_attribution", RD_ATTR_ABLATION, model, src, static,
                                           times, lengths, target, baselines, sensor_groups, None, internal_batch_size,
                                           feature_mask)
    return _split(attr, G)


def shapley_value_sampling(model, src, static, times, lengths, target=None, baselines=None, sensor_groups=None,
                           n_samples=25, seed=0, permutations=None, internal_batch_size=None,
                           return_convergence_delta=False, feature_mask=None):
    """Shapley values, by permutation sampling, of the game v(S) = F(x with the players outside S removed),
    F = logits[b, target[b]] of an eval-mode Raindrop_v2; players and removal as for feature_ablation:

        phi[b, g] = (1/m) sum_p [F(S_pg + {g}) - F(S_pg)],  S_pg = the players ahead of g in permutation p

    Players are sensor groups or, with feature_mask, the players of a map of the value cells (see feature_ablation);
    the m permutations of the P players (the static player has index G) are shared by the batch, as in Captum: drawn
    by sample_permutations(P, n_samples, seed), or given as `permutations` [m, P] (all P! of them give the exact
    Shapley values).  Efficiency: sum_g phi[b, g] (+ the static player's) = F(x) - F(x') up to rounding.

    Returns (attr_sensors [B, G], attr_static [B] or None), plus delta [B] = sum of the sample's attributions -
    (F(x) - F(x')) when return_convergence_delta.  The call evaluates m*(P-1) coalitions on the device besides the
    endpoints; everything else is as for feature_ablation."""
    _check_call("shapley_value_sampling", model, src, static, baselines, internal_batch_size)
    if permutations is None:
        n_samples = int(n_samples)
        if n_samples < 1:
            raise ValueError("n_samples must be >= 1, got %d" % n_samples)

        def orders_host(P):
            return sample_permutations(P, n_samples, seed)
    else:
        def orders_host(P):
            return _check_permutations(permutations, P)
    attr, ends, tgt, G = _coalition_attribution("rd_raindrop_v2_coalition_attribution", RD_ATTR_SHAPLEY, model, src,
                                                static, times, lengths, target, baselines, sensor_groups, orders_host,
                                                internal_batch_size, feature_mask)
    out = _split(attr, G)
    if not return_convergence_delta:
        return out
    f = _endpoint_values(ends, tgt).double()
    return out + ((attr.double().sum(dim=1) - (f[1] - f[0])).float(),)


# ---- KernelSHAP: Shapley values by an efficiency-constrained weighted regression over sampled coalitions ---------------
KERNEL_SHAP_MAX_PLAYERS = 4096       # the solve operator is P^2 fp64 on the device and a pinv of O(P^3) on the host
ALL_COALITIONS_MAX_PLAYERS = 20


def _shapley_kernel(P, sizes):
    """Probability ~ (P-1) / (s (P-s)) of a coalition size s in [1, P-1] (the Shapley kernel summed over a size)."""
    return (P - 1) / (sizes * (P - sizes))


def sample_coalitions(n_players, n_samples, seed=0):
    """(Z uint8 [M, P], w float64 [M]): paired coalitions for kernel_shap, drawn by numpy.random.default_rng(seed).
    Each pair draws a size s in [1, P-1] with probability ~ (P-1) / (s (P-s)), then a uniform subset of that size (the
    s players of smallest rng.random key); the subset is row 2i and its complement row 2i+1.  M = n_samples rounded up
    to even, w = 1/M.  P = 1 has no proper non-empty coalition: M = 0.  The same seed gives the same set."""
    P, n = int(n_players), int(n_samples)
    if P < 1 or n < 1:
        raise ValueError("n_players and n_samples must be >= 1, got %d and %d" % (P, n))
    if P == 1:
        return np.zeros((0, 1), dtype=np.uint8), np.zeros(0)
    rng = np.random.default_rng(seed)
    pairs = (n + 1) // 2
    sizes = np.arange(1, P)
    p = _shapley_kernel(P, sizes.astype(np.float64))
    s = rng.choice(sizes, size=pairs, p=p / p.sum())
    rank = np.argsort(np.argsort(rng.random((pairs, P)), axis=1), axis=1)
    z = (rank < s[:, None]).astype(np.uint8)
    Z = np.empty((2 * pairs, P), dtype=np.uint8)
    Z[0::2], Z[1::2] = z, 1 - z
    return Z, np.full(2 * pairs, 1.0 / (2 * pairs))


def all_coalitions(n_players):
    """(Z uint8 [2^P - 2, P], w float64): every proper non-empty coalition (row i - 1 keeps the players of the set bits
    of i) with the Shapley-kernel weights w(s) = (P-1) / (C(P, s) s (P-s)); kernel_shap over these returns the exact
    Shapley values.  P <= 20."""
    P = int(n_players)
    if not 1 <= P <= ALL_COALITIONS_MAX_PLAYERS:
        raise ValueError("all_coalitions takes 1 <= n_players <= %d, got %d" % (ALL_COALITIONS_MAX_PLAYERS, P))
    idx = np.arange(1, (1 << P) - 1, dtype=np.int64)
    Z = ((idx[:, None] >> np.arange(P)) & 1).astype(np.uint8)
    s = Z.sum(axis=1, dtype=np.int64)
    comb = np.array([math.comb(P, k) for k in range(P + 1)], dtype=np.float64)
    return Z, _shapley_kernel(P, s.astype(np.float64)) / comb[s]


def kernel_shap_operator(Z, w):
    """[K | k] float64 [P, P+1]: the first P rows of pinv([[A, 1], [1^T, 0]]), A = sum_j w_j z_j z_j^T, the KKT system
    of the weighted least-squares fit of the coalition values under efficiency.  Any coalition set gives a well defined
    operator (the minimum-norm solution when A is singular), and sum_g phi[g] = v(all) - v(empty) holds."""
    Z = np.asarray(Z, dtype=np.float64)
    w = np.asarray(w, dtype=np.float64)
    P = Z.shape[1]
    kkt = np.zeros((P + 1, P + 1))
    kkt[:P, :P] = (Z.T * w) @ Z
    kkt[:P, P] = kkt[P, :P] = 1.0
    return np.linalg.pinv(kkt)[:P]


def kernel_shap_from_values(values, v_empty, v_all, Z, w, operator=None):
    """The KernelSHAP estimate on the host in fp64, [B, P]: phi_b = K r_b + k (v_b(all) - v_b(empty)),
    r_b = sum_j w_j z_j (values[j, b] - v_b(empty)).  values [M, B] are v_b(z_j); v_empty, v_all [B]."""
    Z = np.asarray(Z, dtype=np.float64)
    w = np.asarray(w, dtype=np.float64)
    v0, v1 = np.asarray(v_empty, dtype=np.float64), np.asarray(v_all, dtype=np.float64)
    v = np.asarray(values, dtype=np.float64).reshape(Z.shape[0], v0.shape[0])
    op = kernel_shap_operator(Z, w) if operator is None else operator
    r = (Z * w[:, None]).T @ (v - v0[None, :])                                  # [P, B]
    return (op[:, :-1] @ r + op[:, -1:] * (v1 - v0)[None, :]).T


def _check_coalitions(coalitions, P):
    """(Z uint8 [M, P] of 0/1, w float64 [M], finite and >= 0) from a pair (Z, w)."""
    if not isinstance(coalitions, (tuple, list)) or len(coalitions) != 2:
        raise ValueError("coalitions must be a pair (Z [M, n_players], w [M])")
    z = torch.as_tensor(coalitions[0])
    if z.is_floating_point() or z.is_complex():
        raise ValueError("coalitions Z must hold 0/1 integers or booleans")
    Z = z.cpu().numpy()
    if Z.ndim != 2 or Z.shape[1] != P:
        raise ValueError("coalitions Z must have shape [M, n_players=%d], got %s" % (P, Z.shape))
    if Z.size and (Z.min() < 0 or Z.max() > 1):
        raise ValueError("coalitions Z must hold 0/1 entries")
    w = torch.as_tensor(coalitions[1]).detach().cpu().double().numpy()
    if w.shape != (Z.shape[0],):
        raise ValueError("coalition weights must have shape [M=%d], got %s" % (Z.shape[0], w.shape))
    if not np.all(np.isfinite(w)) or np.any(w < 0):
        raise ValueError("coalition weights must be finite and >= 0")
    if Z.shape[0] >= 1 << 31:
        raise ValueError("at most 2^31 - 1 coalitions")
    return np.ascontiguousarray(Z.astype(np.uint8)), np.ascontiguousarray(w)


def _sampled_key(P, n, seed):
    """Cache key of sample_coalitions(P, n, seed): only an int seed names a fixed set; None, a Generator or a
    SeedSequence draws anew on every call, so it gets None (never cached)."""
    if isinstance(seed, (int, np.integer)) and not isinstance(seed, bool):
        return ("sampled", P, n, int(seed))
    return None


def _kernel_shap_operands(plan, key, make, device):
    """Device (Z uint8, w float64, [K | k] float64) of a coalition set, in ONE cache entry per plan that another set
    replaces: the pinv runs and the copies are made once per set, so repeated calls and a CUDA-graph capture after an
    eager call copy nothing, while the entry bounds the device memory to one set.  key None (a seed that is not an int,
    e.g. None or a numpy Generator, whose draws differ from call to call) never hits.  Operands read under CUDA-graph
    capture are held for the plan's lifetime (plan._kshap_captured), as are the scratch (_Call.scratch) and a host
    feature mask (_device_cells), so a captured call's replays stay valid after later calls replace any of them."""
    cached = plan.__dict__.get("_kshap")
    if key is None or cached is None or cached[0] != key + (device.index,):
        plan.__dict__["_kshap"] = None
        Z, w = make()
        op = kernel_shap_operator(Z, w)
        got = (torch.tensor(Z, dtype=torch.uint8, device=device), torch.tensor(w, dtype=torch.float64, device=device),
               torch.tensor(op, dtype=torch.float64, device=device))
        cached = plan.__dict__["_kshap"] = (None if key is None else key + (device.index,), got)
    if device.type == "cuda" and torch.cuda.is_current_stream_capturing():
        held = plan.__dict__.setdefault("_kshap_captured", [])
        if not any(t is cached[1] for t in held):
            held.append(cached[1])
    return cached[1]


def kernel_shap(model, src, static, times, lengths, target=None, baselines=None, sensor_groups=None, feature_mask=None,
                n_samples=None, seed=0, coalitions=None, internal_batch_size=None, return_convergence_delta=False):
    """Shapley values by KernelSHAP of the game v(S) = F(x with the players outside S removed), F = logits[b, target[b]]
    of an eval-mode Raindrop_v2; players (sensor_groups, or feature_mask, plus the static player G) and removal as for
    shapley_value_sampling.  With coalitions z_j and weights w_j shared by the batch,

        phi_b = K r_b + k (v_b(all) - v_b(empty)),   r_b = sum_j w_j z_j (v_b(z_j) - v_b(empty)),
        [K | k] = the first P rows of pinv([[A, 1], [1^T, 0]]),   A = sum_j w_j z_j z_j^T

    the weighted least-squares fit of the coalition values with efficiency as a constraint: sum_g phi[b, g] =
    F(x) - F(x') up to rounding, for any coalition set.  Unlike permutation sampling, whose cost is m*(P-1) forwards,
    any budget M works and every coalition informs every player.

    n_samples:  coalitions to sample (default 2P + 2048), drawn paired by sample_coalitions(P, n_samples, seed).  An
                int seed names a fixed set, which is cached; any other seed numpy.random.default_rng takes (None, a
                Generator) draws a new set on every call.
    coalitions: instead, a pair (Z [M, P] of 0/1, w [M] >= 0); all_coalitions(P) gives the exact Shapley values.
    A player with no cell is fitted like any other: exhaustive coalitions give it 0 up to the rounding of the solve.

    Returns (attr_players [B, G], attr_static [B] or None), plus delta [B] = sum of the sample's attributions -
    (F(x) - F(x')) when return_convergence_delta.  The operator is computed on the host in fp64 once per coalition set and
    kept on the device with the set in a one-entry cache per model.  The call evaluates M coalitions on the device besides
    the endpoints, accumulates r in fp64 in coalition order (bitwise independent of internal_batch_size with the ob-prop
    mode pinned) and applies the operator in fp64; everything else is as for shapley_value_sampling.  P is at most
    KERNEL_SHAP_MAX_PLAYERS."""
    _check_call("kernel_shap", model, src, static, baselines, internal_batch_size)
    groups, cells, G, P = _players(model, src, sensor_groups, feature_mask)
    if P > KERNEL_SHAP_MAX_PLAYERS:
        raise ValueError("kernel_shap takes at most %d players, got %d" % (KERNEL_SHAP_MAX_PLAYERS, P))
    if coalitions is None:
        n = 2 * P + 2048 if n_samples is None else int(n_samples)
        if n < 1:
            raise ValueError("n_samples must be >= 1, got %d" % n)
        key = _sampled_key(P, n, seed)

        def make():
            return sample_coalitions(P, n, seed)
    else:
        Z, w = _check_coalitions(coalitions, P)
        key = ("given", Z.shape, Z.tobytes(), w.tobytes())

        def make():
            return Z, w
    cl = _Call(model, src, static, times, lengths, target, baselines)
    lib, plan, device, B = cl.lib, cl.plan, cl.device, src.shape[1]
    z_d, w_d, op_d = _kernel_shap_operands(plan, key, make, device)
    M = z_d.shape[0]
    if groups is not None:
        player, stride_t, stride_b = _device_int32(plan, "players", groups, device), 0, 0
    else:
        player, stride_t, stride_b = _cell_players(plan, cells, device)

    dims = plan.dims(B, False)
    if internal_batch_size is None:
        cc = _default_coalitions_per_chunk(lib, dims, P, max(M, 1))
    else:
        cc = max(1, int(internal_batch_size) // B)
    cc = max(1, min(cc, M))
    nbytes = lib.rd_coalition_attribution_scratch_bytes(C.byref(dims), P, cc)
    if nbytes == 0:
        L.check(-2, "rd_coalition_attribution_scratch_bytes")
    scratch = cl.scratch("_coal_attr_scratch", device.index, nbytes)

    attr = torch.empty(B, P, device=device, dtype=torch.float32)
    ends = torch.empty(2, B, plan.n_classes, device=device, dtype=torch.float32)
    L.check(lib.rd_raindrop_v2_kernel_shap(C.byref(dims), C.byref(cl.params), cl.x.data_ptr(), L.ptr(cl.st),
                                           cl.tm.data_ptr(), cl.ln.data_ptr(), plan.node_scale.data_ptr(), cl.x0.data_ptr(),
                                           L.ptr(cl.st0), L.ptr(cl.tgt), player.data_ptr(), stride_t, stride_b, P,
                                           z_d.data_ptr() if M else 0, w_d.data_ptr() if M else 0, M, op_d.data_ptr(), cc,
                                           scratch.data_ptr(), attr.data_ptr(), ends.data_ptr(), L.stream_ptr(device)),
            "rd_raindrop_v2_kernel_shap")
    out = _split(attr, G)
    if not return_convergence_delta:
        return out
    f = _endpoint_values(ends, cl.tgt).double()
    return out + ((attr.double().sum(dim=1) - (f[1] - f[0])).float(),)


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
