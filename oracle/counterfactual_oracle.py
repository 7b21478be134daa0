"""TEST INFRASTRUCTURE ONLY -- a float64 replay of the counterfactual search (raindrop_b200.counterfactual,
rd_raindrop_v2_counterfactual): FISTA with the elastic-net proximal step, the per-element box, the bisection over the
loss weight c and independent restarts, on the oracle model's forward_dense with autograd for the input gradient.

The restarts' start points are restated in numpy (`start_deltas`): u = (word >> 8) 2^-24 of the Philox4x32-10 stream at
site 103, key (seed, step), index (b*R + r)*(T*N + d_static) + e, word i & 3 of the block at counter i >> 2 (the
dropout stream's word rule, oracle/dropout_masks.py), delta = clip_box(init_scale (2u - 1)) in fp32.
"""
import numpy as np
import torch

from .dropout_masks import dropout_words_at

SITE_CF_START = 103


def soft_threshold(v, lam):
    """S(v, lam) = sign(v) max(|v| - lam, 0), elementwise."""
    return torch.sign(v) * torch.clamp(v.abs() - lam, min=0.0)


def prox_step(y, g, alpha, beta, w, dlo, dhi):
    """One proximal-gradient step in delta units: clip(S(y - alpha g, alpha beta w), dlo, dhi).  Returns (x_new, v) with
    v = y - alpha g, the soft-threshold's input."""
    v = y - alpha * g
    return torch.minimum(torch.maximum(soft_threshold(v, alpha * beta * w), dlo), dhi), v


def boxes(x, lower, upper):
    """(dlo, dhi): the effective box [min(lower, x), max(upper, x)] in delta units."""
    return torch.minimum(lower, x) - x, torch.maximum(upper, x) - x


def start_deltas(src, static, R, init_scale, seed, step, sensors=None, perturb_static=False, lower=None, upper=None):
    """The replicas' start points as the kernels draw them: (d_src [R, T, B, N], d_static [R, B, ds] or None), float32,
    replica 0 all zero, zero outside S_b.  lower / upper: float32 [N + ds] or None (unbounded)."""
    src = np.asarray(src, dtype=np.float32)
    T, B, N2 = src.shape
    N = N2 // 2
    ds = 0 if static is None else np.asarray(static).shape[1]
    E = T * N + ds
    lo = np.full(N + ds, -np.inf, np.float32) if lower is None else np.asarray(lower, np.float32)
    hi = np.full(N + ds, np.inf, np.float32) if upper is None else np.asarray(upper, np.float32)
    pert = src[:, :, N:] > 0
    if sensors is not None:
        pert &= np.asarray(sensors, dtype=bool)[None, None, :]
    d_src = np.zeros((R, T, B, N), np.float32)
    d_st = None if static is None else np.zeros((R, B, ds), np.float32)
    e = np.arange(E, dtype=np.uint64)
    s = np.float32(init_scale)
    for b in range(B):
        xv = src[:, b, :N].reshape(-1)
        xs = np.zeros(0, np.float32) if static is None else np.asarray(static, np.float32)[b]
        xe = np.concatenate([xv, xs])
        col = np.concatenate([np.tile(np.arange(N), T), N + np.arange(ds)])
        dlo = np.minimum(lo[col], xe) - xe
        dhi = np.maximum(hi[col], xe) - xe
        for r in range(1, R):
            w = dropout_words_at(seed, step, SITE_CF_START, np.uint64((b * R + r) * E) + e)
            u = (w >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
            d = (s * (np.float32(2.0) * u - np.float32(1.0))).astype(np.float32)
            d = np.minimum(np.maximum(d, dlo), dhi).astype(np.float32)
            d_src[r, :, b, :] = np.where(pert[:, b, :], d[:T * N].reshape(T, N), 0)
            if ds and perturb_static:
                d_st[r, b] = d[T * N:]
    return d_src, d_st


def margins(logits, target):
    """(m, c*): m = z_t - max_{c != t} z_c, c* its first argmax."""
    z = logits.clone()
    z.scatter_(1, target[:, None], -float("inf"))
    cs = z.argmax(dim=1)                       # torch.argmax returns the first maximal index
    return logits.gather(1, target[:, None])[:, 0] - logits.gather(1, cs[:, None])[:, 0], cs


def search(o, src, static, times, lengths, target, *, n_restarts=1, starts=None, weights=None, lower=None, upper=None,
           sensors=None, perturb_static=False, kappa=0.0, beta=0.1, c_init=1.0, step_size=0.01, n_search=1, n_steps=5,
           dtype=torch.float64):
    """The search in `dtype` (float64; float32 with o.float() measures how much a trajectory moves under fp32 rounding)
    on the oracle model o of that dtype.  Inputs are CPU tensors; weights / lower / upper float
    [N + ds] or None; starts = start_deltas(...) or None (all zero).  Returns a list of records, one per evaluated point
    in (round, step, replica) order: dict(round, step, replica, m [B], valid [B], d [B], delta [T, B, N],
    delta_static [B, ds] or None, slack [T, B, N], gate [B], logits [B, C]), slack being, per value cell, the smallest
    | |v| - alpha beta w | of the (at most two) soft-threshold inputs that produced the point (inf for a start point), and
    gate the smallest |x + delta| over the sample's mutable value cells (how close the lift relu(v R_u) is to switching
    there); and the final c [B, R]."""
    src, times = src.to(dtype), times.to(dtype)
    st = None if static is None else static.to(dtype)
    T, B, N2 = src.shape
    N = N2 // 2
    ds = 0 if st is None else st.shape[1]
    one = torch.ones(N + ds, dtype=dtype)
    w = one if weights is None else torch.as_tensor(weights).to(dtype)
    lo = -np.inf * one if lower is None else torch.as_tensor(lower).to(dtype)
    hi = np.inf * one if upper is None else torch.as_tensor(upper).to(dtype)
    x = src[:, :, :N]
    pert = (src[:, :, N:] > 0).to(dtype)
    if sensors is not None:
        pert = pert * torch.as_tensor(np.asarray(sensors, bool)).to(dtype)[None, None, :]
    dlo, dhi = boxes(x, lo[:N], hi[:N])
    ps = bool(perturb_static) and st is not None
    sdlo, sdhi = (boxes(st, lo[N:], hi[N:]) if ps else (None, None))
    wv, ws = w[:N], w[N:]
    lam, lams = step_size * beta * wv, step_size * beta * ws
    records = []
    c = torch.full((B, n_restarts), float(c_init), dtype=torch.float64)
    clo = torch.zeros_like(c)
    chi = torch.full_like(c, float("inf"))

    def dist(yd, ysd):
        d = beta * (wv * yd).abs().sum(dim=(0, 2)) + ((wv * yd) ** 2).sum(dim=(0, 2))
        if ysd is not None:
            d = d + beta * (ws * ysd).abs().sum(1) + ((ws * ysd) ** 2).sum(1)
        return d

    states = []
    for r in range(n_restarts):
        s0 = torch.zeros_like(x) if starts is None else torch.as_tensor(starts[0][r]).to(dtype) * pert
        ss0 = None
        if ps:
            ss0 = torch.zeros_like(st) if starts is None or starts[1] is None else torch.as_tensor(starts[1][r]).to(dtype)
        states.append((s0, ss0))
    for s in range(n_search):
        found = torch.zeros(B, n_restarts, dtype=torch.bool)
        cur = []
        for r in range(n_restarts):
            s0, ss0 = states[r]
            cur.append(dict(xd=s0.clone(), yd=s0.clone(), xsd=None if ss0 is None else ss0.clone(),
                            ysd=None if ss0 is None else ss0.clone(), slack=torch.full_like(x, float("inf")),
                            prev=torch.full_like(x, float("inf"))))
        for k in range(n_steps + 1):
            for r in range(n_restarts):
                q = cur[r]
                xin = src.clone()
                xin[:, :, :N] = x + q["yd"]
                xin.requires_grad_(True)
                sin = None
                if st is not None:
                    sin = (st + q["ysd"]) if ps else st.clone()
                    sin.requires_grad_(True)
                logits = o.forward_dense(xin, sin, times, lengths)[0]
                m, cs = margins(logits.detach(), target)
                active = m <= kappa
                valid = (m > 0) & (m >= kappa)
                found[:, r] |= valid
                gate = torch.where(pert > 0, (x + q["yd"]).abs(), torch.full_like(x, float("inf"))).amin(dim=(0, 2))
                records.append(dict(round=s, step=k, replica=r, m=m, valid=valid, d=dist(q["yd"], q["ysd"]), gate=gate,
                                    delta=q["yd"].clone(), delta_static=None if q["ysd"] is None else q["ysd"].clone(),
                                    slack=q["slack"].clone(), logits=logits.detach()))
                if k == n_steps:
                    continue
                sel = c[:, r] * active.to(dtype)
                hinge = (sel * (logits.gather(1, cs[:, None])[:, 0] - logits.gather(1, target[:, None])[:, 0])).sum()
                grads = torch.autograd.grad(hinge, [xin] + ([sin] if ps else []))
                g = grads[0][:, :, :N] * pert + 2 * wv ** 2 * q["yd"]
                xn, v = prox_step(q["yd"], g, step_size, beta, wv, dlo, dhi)
                xn = xn * pert
                mom = k / (k + 3)
                yn = torch.minimum(torch.maximum(xn + mom * (xn - q["xd"]), dlo), dhi) * pert
                sl = (v.abs() - lam).abs()
                q["slack"] = torch.minimum(sl, q["prev"])
                q["prev"] = sl
                q["xd"], q["yd"] = xn, yn
                if ps:
                    gs = grads[1] + 2 * ws ** 2 * q["ysd"]
                    xsn, _ = prox_step(q["ysd"], gs, step_size, beta, ws, sdlo, sdhi)
                    ysn = torch.minimum(torch.maximum(xsn + mom * (xsn - q["xsd"]), sdlo), sdhi)
                    q["xsd"], q["ysd"] = xsn, ysn
        for r in range(n_restarts):
            for b in range(B):
                cb, lb, hb = float(c[b, r]), float(clo[b, r]), float(chi[b, r])
                cb, lb, hb = bisect(bool(found[b, r]), cb, lb, hb)
                c[b, r], clo[b, r], chi[b, r] = cb, lb, hb
    return records, c


def bisect(found, c, lo, hi):
    """One bisection update of (c, lo, hi) after a round, in Python floats (IEEE double, as the kernels)."""
    if found:
        hi = min(hi, c)
        c = (lo + hi) / 2.0
    else:
        lo = max(lo, c)
        c = (lo + hi) / 2.0 if hi < float("inf") else 10.0 * c
    return c, lo, hi


def best_points(records, B):
    """Per sample, the index into records of the selected point (smallest d among valid points, ties: the earliest
    record), or -1."""
    best, bd = [-1] * B, [float("inf")] * B
    for i, rec in enumerate(records):
        for b in range(B):
            if bool(rec["valid"][b]) and float(rec["d"][b]) < bd[b]:
                bd[b], best[b] = float(rec["d"][b]), i
    return best
