"""Differentially private training of Raindrop_v2 (DP-SGD, Abadi et al. 2016) with the per-sample gradient work on the
device, and the privacy accountant for it.

A DP step on a batch of B slots with weights w_b in {0, 1} (Poisson sampling with rate q, padded to a fixed capacity so
that the step stays one CUDA graph) hands Adam

    g = ( sum_b w_b c_b g_b + sigma C xi ) / L,    c_b = min(1, C / (||g_b|| + 1e-6)),    xi ~ N(0, I),

where g_b is sample b's gradient of its cross-entropy over all trained tensors, C the clipping norm, sigma the noise
multiplier and L = q n_train the expected batch size.  The per-sample norms come from one extra data-gradient backward
with per-sample norm kernels where the training path reduces weight gradients (include/raindrop_b200.h); the clipped sum
is the ordinary backward run on rescaled d(loss)/d(logits), since the gradient of sum_b c_b l_b with the c_b held fixed is
sum_b c_b g_b.

    sampler = PoissonSampler(n_train, q)
    step = DPTrainStep(model, sampler.capacity, max_grad_norm=1.0, noise_multiplier=1.1, expected_batch_size=q * n_train)
    ds = DeviceDataset(P, Pstatic, Ptime, y)                    # raindrop_b200.data
    for _ in range(n_steps):
        idx, weight = sampler.sample()
        ds.fill(step, torch.from_numpy(idx))
        step.weight.copy_(torch.from_numpy(weight))
        step.step()
    eps = epsilon(q, 1.1, n_steps, delta=1e-5)

tools/dp_train.py runs this loop over epochs and prints epsilon after each.

Caveats: the input normalisation statistics (feature_stats) are computed from the training set and are not private;
the reference's balanced upsampling sampler does not match the accountant, so DP training must draw its batches with
PoissonSampler; the noise comes from the Philox stream of the dropout masks, which is not a cryptographically secure
generator (as Opacus outside its secure_mode).
"""
import ctypes as C
import math
import os

import numpy as np
import torch
import torch.distributed as dist
from scipy import special

from . import lib as L
from .train import TrainStep

DEFAULT_ORDERS = tuple([1 + x / 10.0 for x in range(1, 100)] + list(range(12, 64)) + [128, 256, 512])


# ---- accountant: Renyi DP of the sampled Gaussian mechanism --------------------------------------------------------------
def _log_a_int(q, sigma, alpha):
    """log A_alpha for integer alpha: the binomial expansion of E_{z ~ N(0, sigma^2)}[((1-q) + q e^{(2z-1)/(2 sigma^2)})^alpha]
    (Mironov, Talwar & Zhang 2019, section 3.3)."""
    i = np.arange(int(alpha) + 1, dtype=np.float64)
    t = (special.gammaln(alpha + 1) - special.gammaln(i + 1) - special.gammaln(alpha - i + 1) + i * math.log(q) +
         (alpha - i) * math.log1p(-q) + (i * i - i) / (2.0 * sigma * sigma))
    return float(special.logsumexp(t))


def _log_a_frac(q, sigma, alpha):
    """log A_alpha for fractional alpha: the two convergent series of Mironov, Talwar & Zhang 2019 (section 3.3), split at
    z0 = sigma^2 log(1/q - 1) + 1/2, summed in blocks of terms until a whole block lies below e^-45 (A_alpha >= 1)."""
    z0 = sigma * sigma * math.log(1.0 / q - 1.0) + 0.5
    terms, signs = [], []
    start = 0
    while True:
        i = np.arange(start, start + 256, dtype=np.float64)
        j = alpha - i
        coef = special.binom(alpha, i)
        log_coef = np.log(np.abs(coef))
        log_s0 = (log_coef + i * math.log(q) + j * math.log1p(-q) + (i * i - i) / (2.0 * sigma * sigma) +
                  special.log_ndtr(-(i - z0) / sigma))
        log_s1 = (log_coef + j * math.log(q) + i * math.log1p(-q) + (j * j - j) / (2.0 * sigma * sigma) +
                  special.log_ndtr(-(z0 - j) / sigma))
        sg = np.sign(coef)
        terms += [log_s0, log_s1]
        signs += [sg, sg]
        start += 256
        if max(log_s0.max(), log_s1.max()) < -45:
            break
    out, sign = special.logsumexp(np.concatenate(terms), b=np.concatenate(signs), return_sign=True)
    if not sign > 0:      # A_alpha >= 1: a non-positive sum means the series was not summed accurately
        raise ArithmeticError("log A_alpha series gave a non-positive sum (q=%r, sigma=%r, alpha=%r)" % (q, sigma, alpha))
    return float(out)


def _check_q_sigma(q, sigma):
    q, sigma = float(q), float(sigma)
    if not 0.0 <= q <= 1.0:
        raise ValueError("sampling rate q must be in [0, 1], got %r" % q)
    if not sigma >= 0.0:
        raise ValueError("noise multiplier sigma must be >= 0, got %r" % sigma)
    return q, sigma


def rdp_sampled_gaussian(q, sigma, orders=DEFAULT_ORDERS):
    """Renyi-DP epsilon(alpha) of ONE step of the sampled Gaussian mechanism (Poisson rate q, noise multiplier sigma)
    at each order alpha > 1, float64 array: exact binomial sum at integer orders, the series at fractional ones."""
    q, sigma = _check_q_sigma(q, sigma)
    orders = np.atleast_1d(np.asarray(orders, dtype=np.float64))
    if np.any(orders <= 1):
        raise ValueError("RDP orders must be > 1")
    out = np.empty_like(orders)
    for k, a in enumerate(orders):
        if q == 0:
            out[k] = 0.0
        elif sigma == 0:
            out[k] = np.inf
        elif q == 1.0:
            out[k] = a / (2.0 * sigma * sigma)
        elif float(a).is_integer():
            out[k] = _log_a_int(q, sigma, int(a)) / (a - 1)
        else:
            out[k] = _log_a_frac(q, sigma, a) / (a - 1)
    return out


def epsilon(q, sigma, steps, delta, orders=DEFAULT_ORDERS):
    """(epsilon, delta)-DP of `steps` compositions of the sampled Gaussian mechanism, from RDP by the conversion of
    Balle et al. 2020 (Theorem 21), minimised over the orders."""
    q, sigma = _check_q_sigma(q, sigma)
    steps = int(steps)
    if steps < 0 or not 0.0 < float(delta) < 1.0:
        raise ValueError("steps must be >= 0 and delta in (0, 1)")
    if q == 0.0 or steps == 0:
        return 0.0
    orders = np.atleast_1d(np.asarray(orders, dtype=np.float64))
    rdp = steps * rdp_sampled_gaussian(q, sigma, orders)
    with np.errstate(invalid="ignore"):
        eps = rdp - (math.log(delta) + np.log(orders)) / (orders - 1) + np.log((orders - 1) / orders)
    eps = np.where(np.isnan(eps), np.inf, eps)
    return float(max(0.0, np.min(eps)))


def noise_multiplier_for(target_epsilon, delta, q, steps, orders=DEFAULT_ORDERS, tol=1e-10):
    """The smallest sigma (to `tol`) with epsilon(q, sigma, steps, delta) <= target_epsilon, by bisection."""
    target_epsilon = float(target_epsilon)
    if not target_epsilon > 0:
        raise ValueError("target_epsilon must be > 0")
    lo, hi = 0.0, 1.0
    while epsilon(q, hi, steps, delta, orders) > target_epsilon:
        lo, hi = hi, 2.0 * hi
        if hi > 1e6:
            raise ValueError("no noise multiplier below 1e6 reaches epsilon = %g" % target_epsilon)
    while hi - lo > tol * max(1.0, hi):
        mid = 0.5 * (lo + hi)
        if epsilon(q, mid, steps, delta, orders) > target_epsilon:
            lo = mid
        else:
            hi = mid
    return hi


# ---- Poisson sampling into a fixed capacity -------------------------------------------------------------------------------
class PoissonSampler:
    """Batches of Poisson sampling: every one of the n samples is in a batch independently with probability q.  Each
    draw is (idx int64 [capacity], weight float32 [capacity]): the drawn indices first (ascending) with weight 1, then
    empty slots holding index 0 with weight 0.  A draw larger than the capacity raises (truncating it would break the
    accounting); the default capacity q n + 8 sqrt(q n) makes that rare.  Iterating yields draws forever."""

    def __init__(self, n, q, capacity=None, seed=None):
        self.n, self.q = int(n), float(q)
        if self.n < 1 or not 0.0 < self.q <= 1.0:
            raise ValueError("PoissonSampler needs n >= 1 and q in (0, 1]")
        m = self.q * self.n
        self.capacity = int(capacity) if capacity is not None else max(1, int(math.ceil(m + 8.0 * math.sqrt(m))))
        if self.capacity < 1:
            raise ValueError("capacity must be >= 1")
        self.rng = np.random.default_rng(seed)

    def sample(self):
        drawn = np.flatnonzero(self.rng.random(self.n) < self.q)
        k = drawn.size
        if k > self.capacity:
            raise RuntimeError("Poisson draw of %d samples exceeds the batch capacity %d" % (k, self.capacity))
        idx = np.zeros(self.capacity, dtype=np.int64)
        weight = np.zeros(self.capacity, dtype=np.float32)
        idx[:k] = drawn
        weight[:k] = 1.0
        return idx, weight

    def __iter__(self):
        while True:
            yield self.sample()


# ---- device path ---------------------------------------------------------------------------------------------------------
def sqnorm_fields(model):
    """State-dict keys of the columns of per_sample_grad_sqnorms / DPTrainStep.sqnorms (the flat-bucket order)."""
    return [k for k, _ in model._plan.fields]


def per_sample_grad_sqnorms(model, src, static, times, lengths, y):
    """[B, n_fields] float64: ||grad of CrossEntropy(logits_b, y_b) w.r.t. each trained tensor||^2 for each sample b,
    columns in sqnorm_fields(model) order.  In train() mode the forward draws dropout masks from the model's stream and
    advances it by one step, as a module forward does.  Parameters and their .grad are left unchanged.  Raises
    RaindropB200Error without CUDA or without the built library."""
    from .attribution import _Call
    from .models_rd import Raindrop_v2
    if not isinstance(model, Raindrop_v2):
        raise TypeError("per_sample_grad_sqnorms takes a raindrop_b200 Raindrop_v2 model, got %s" % type(model).__name__)
    with torch.no_grad():
        cl = _Call(model, src, static, times, lengths, None, False)
        lib, plan, B, dev = cl.lib, cl.plan, src.shape[1], cl.device
        if src.dim() != 3 or src.shape[0] != plan.T or src.shape[2] != 2 * plan.N:
            raise ValueError("src must be [max_len=%d, B, 2*d_inp=%d], got %s" % (plan.T, 2 * plan.N, tuple(src.shape)))
        yv = torch.as_tensor(y).to(device=dev, dtype=torch.int64).contiguous()
        if yv.shape != (B,):
            raise ValueError("y must be [B], got %s" % (tuple(yv.shape),))
        dims = plan.dims(B, model.training)
        key = (B, bool(model.training), dims.obprop_mode, dev.index)
        ws = cl.scratch("_dp_workspace", key, lib.rd_workspace_bytes(C.byref(dims)))
        f32 = dict(device=dev, dtype=torch.float32)
        logits, dlog, loss = torch.empty(B, plan.n_classes, **f32), torch.empty(B, plan.n_classes, **f32), torch.empty(1, **f32)
        st = L.stream_ptr(dev)
        L.check(lib.rd_raindrop_v2_fwd(C.byref(dims), C.byref(cl.params), cl.x.data_ptr(), L.ptr(cl.st), cl.tm.data_ptr(),
                                       cl.ln.data_ptr(), plan.node_scale.data_ptr(), L.ptr(plan.rng_state), ws.data_ptr(),
                                       logits.data_ptr(), yv.data_ptr(), loss.data_ptr(), dlog.data_ptr(), st),
                "rd_raindrop_v2_fwd")
        nbytes = lib.rd_dp_scratch_bytes(C.byref(dims))
        scratch = cl.scratch("_dp_scratch", key, nbytes)
        sq = torch.empty(B, len(plan.fields), dtype=torch.float64, device=dev)
        L.check(lib.rd_raindrop_v2_per_sample_grad_sqnorms(C.byref(dims), C.byref(cl.params), L.ptr(cl.st), cl.ln.data_ptr(),
                                                           plan.node_scale.data_ptr(), ws.data_ptr(), dlog.data_ptr(),
                                                           scratch.data_ptr(), sq.data_ptr(), st),
                "rd_raindrop_v2_per_sample_grad_sqnorms")
    return sq * float(B * B)      # the kernels' norms are of grad(l_b / B)


class DPTrainStep(TrainStep):
    """One DP-SGD step on static device buffers: forward, per-sample gradient norms, clipping of d(loss)/d(logits), the
    backward of TrainStep on the clipped d_logits, Gaussian noise, Adam -- all on the device and CUDA-graph capturable.

    batch_capacity: B slots; `weight` [B] (float32, 1 = in the batch, 0 = empty slot, default all 1) rides with the
    batch.  max_grad_norm: C.  noise_multiplier: sigma.  expected_batch_size: L = q n_train.  noise_seed: the Philox seed
    of the noise (default: 64 bits from os.urandom); the noise key {seed, step} lives on the device and every step
    advances it.  The key is part of the training state: a run resumed with the same noise_seed must restore its step
    (noise_key_state() / set_noise_key()), or it replays the noise of the earlier steps, which voids the guarantee.  After a step, `loss` is the mean cross-entropy over the slots with weight 1, `clip_factors` [B] the
    c_b, `sqnorms` the per-sample squared norms per trained tensor (of grad(l_b / B); per_sample_sqnorms() scales them to
    grad l_b).  One GPU only: data-parallel DP-SGD is not supported."""

    def __init__(self, model, batch_capacity, max_grad_norm, noise_multiplier, expected_batch_size, lr=1e-4,
                 noise_seed=None, use_graph=True, betas=(0.9, 0.999), eps=1e-8, group=None):
        if dist.is_initialized() and dist.get_world_size(group) > 1:
            raise L.RaindropB200Error("DPTrainStep runs on one GPU; data-parallel DP-SGD is not supported")
        max_grad_norm, noise_multiplier, expected_batch_size = float(max_grad_norm), float(noise_multiplier), float(expected_batch_size)
        if not max_grad_norm > 0 or not noise_multiplier >= 0 or not expected_batch_size > 0:
            raise ValueError("max_grad_norm and expected_batch_size must be > 0 and noise_multiplier >= 0")
        super().__init__(model, batch_capacity, lr=lr, betas=betas, eps=eps, group=group, use_graph=use_graph,
                         distributed=False)
        self.max_grad_norm, self.noise_multiplier, self.expected_batch_size = max_grad_norm, noise_multiplier, expected_batch_size
        dev, lib = self.device, self.lib
        self.weight = torch.ones(self.B, dtype=torch.float32, device=dev)
        self.clip_factors = torch.ones(self.B, dtype=torch.float32, device=dev)
        self.sqnorms = torch.zeros(self.B, len(self.plan.fields), dtype=torch.float64, device=dev)
        self.dp_scratch = torch.empty(lib.rd_dp_scratch_bytes(C.byref(self.dims)) // 4, dtype=torch.float32, device=dev)
        seed = int.from_bytes(os.urandom(8), "little") if noise_seed is None else int(noise_seed)
        if not 0 <= seed < 1 << 64:
            raise ValueError("noise_seed must be in [0, 2^64)")
        self.noise_key = torch.tensor(np.array([seed, 0, 0], dtype=np.uint64).view(np.int64), device=dev)
        params = model.used_parameters()
        n = len(params)
        self._noise_off = (C.c_int64 * n)(*self.offsets)
        self._noise_numel = (C.c_int64 * n)(*[p.numel() for p in params])
        self.noise_std = noise_multiplier * max_grad_norm / expected_batch_size

    def load_batch(self, batch, non_blocking=True):
        """TrainStep.load_batch plus the slot weights batch["weight"] (default: every slot in the batch)."""
        super().load_batch(batch, non_blocking)
        if batch.get("weight") is not None:
            self.weight.copy_(torch.as_tensor(batch["weight"]), non_blocking=non_blocking)
        else:
            self.weight.fill_(1.0)

    def _state(self):
        return super()._state() + (self.noise_key, self.clip_factors, self.sqnorms)

    def _norm_pass(self, st):
        """Stage 2: the per-sample squared norms of the forward in the workspace, into self.sqnorms."""
        L.check(self.lib.rd_raindrop_v2_per_sample_grad_sqnorms(C.byref(self.dims), C.byref(self.P), L.ptr(self.static),
                                                                self.lengths.data_ptr(), self.plan.node_scale.data_ptr(),
                                                                self.ws.data_ptr(), self.d_logits.data_ptr(),
                                                                self.dp_scratch.data_ptr(), self.sqnorms.data_ptr(), st),
                "rd_raindrop_v2_per_sample_grad_sqnorms")

    def _enqueue(self):
        lib, st = self.lib, L.stream_ptr(self.device)
        self._forward(st)
        self._norm_pass(st)
        L.check(lib.rd_dp_clip_scale(C.byref(self.dims), self.ws.data_ptr(), self.sqnorms.data_ptr(), self.weight.data_ptr(),
                                     self.max_grad_norm, self.expected_batch_size, self.d_logits.data_ptr(),
                                     self.clip_factors.data_ptr(), self.loss.data_ptr(), st),
                "rd_dp_clip_scale")
        self._bwd(L.BWD_ALL, st)
        L.check(lib.rd_dp_add_noise(self.flat_g.data_ptr(), self.flat_g.numel(), self._noise_off, self._noise_numel,
                                    len(self.offsets), self.noise_std, self.noise_key.data_ptr(), st),
                "rd_dp_add_noise")
        self._adam(st)

    def noise_key_state(self):
        """(seed, step) of the noise stream, to be saved with a checkpoint (reads the device key: synchronises)."""
        seed, step, _ = (int(v) for v in self.noise_key.cpu().numpy().view(np.uint64))
        return seed, step

    def set_noise_key(self, seed, step):
        """Restores a saved noise_key_state(); the next step draws the noise of that step."""
        seed, step = int(seed), int(step)
        if not (0 <= seed < 1 << 64 and 0 <= step < 1 << 64):
            raise ValueError("seed and step must be in [0, 2^64)")
        self.noise_key.copy_(torch.tensor(np.array([seed, step, 0], dtype=np.uint64).view(np.int64)))

    def per_sample_sqnorms(self):
        """[B, n_fields] float64: ||grad l_b||^2 per trained tensor of the last step (columns: sqnorm_fields)."""
        return self.sqnorms * float(self.B * self.B)

    def clipped_fraction(self):
        """Fraction of the last step's weight-1 slots whose gradient was clipped (c_b < 1), as a device scalar."""
        w = self.weight > 0
        return ((self.clip_factors < 1) & w).sum() / w.sum().clamp(min=1)
