"""Certified robustness of Raindrop_v2 by randomized smoothing (Cohen, Rosenfeld & Kolter, ICML 2019): Monte Carlo
class votes under Gaussian noise computed on the device in one call per batch (rd_raindrop_v2_smooth_counts), Cohen's
PREDICT and CERTIFY on the host, and Gaussian-augmentation training as a TrainStep whose whole step is one CUDA graph.

    res = certify(model.eval(), src, static, times, lengths, sigma=0.25)      # n0 = 100, n = 100,000, alpha = 0.001
    certified = (res.prediction == y) & (res.radius >= 0.5)                   # provably correct within L2 radius 0.5
    pred = predict(model.eval(), src, static, times, lengths, sigma=0.25)     # -1: abstain

    step = SmoothingTrainStep(model.train(), batch_size=128, sigma=0.25)      # train on x + sigma z
    step.load_batch(batch)
    step.step()

The smoothed classifier g(x) = argmax_c P(f(x + sigma z) = c) adds noise on the threat model of adversarial.pgd: only the
value half of src, only at observed cells (mask src[..., N:] > 0; padded rows have mask 0), optionally restricted to
some sensors, plus the static vector when perturb_static.  The mask half, times and lengths never change.  sigma and
the certified radius are in the units the model sees (per-feature standard deviations after normalisation): a radius r
of sample b certifies that g's prediction does not change under any perturbation delta of S_b with ||delta||_2 < r, the
threat model of pgd(norm="l2").  Replicate m of a call with key (seed, step) draws its noise at Philox key
(seed, step + m), so counts over n = a + b replicates at step s are the counts of a at s plus those of b at s + a.
"""
import ctypes as C
import math
import os
from dataclasses import dataclass

import numpy as np
import torch
import torch.distributed as dist

from . import lib as L
from .adversarial import _check_key, _sensor_mask
from .attribution import _Call, _check_call
from .train import TrainStep
from .uncertainty import _device_key


@dataclass
class CertifyResult:
    """Cohen's CERTIFY per sample (host numpy arrays, float64 statistics): prediction [B] int64 (c_A, or -1 = abstain);
    radius [B] float64 (sigma Phi^-1(p_lower), -1 when abstaining); p_lower [B] the one-sided Clopper-Pearson lower
    bound of P(f(x + sigma z) = c_A); counts0 [B, C] the selection votes and counts [B, C] the estimation votes (int64
    device tensors)."""
    prediction: object
    radius: object
    p_lower: object
    counts0: object
    counts: object


def _check_sigma(sigma):
    sigma = float(sigma)
    if not (math.isfinite(sigma) and sigma >= 0):
        raise ValueError("sigma must be finite and >= 0, got %r" % sigma)
    return sigma


def _check_alpha(alpha):
    alpha = float(alpha)
    if not 0.0 < alpha < 1.0:
        raise ValueError("alpha must lie in (0, 1), got %r" % alpha)
    return alpha


def _check_n(name, n):
    n = int(n)
    if not 1 <= n < 1 << 31:
        raise ValueError("%s must be in [1, 2^31), got %d" % (name, n))
    return n


def _counts(counts):
    c = counts.detach().cpu().numpy() if torch.is_tensor(counts) else np.asarray(counts)
    if c.ndim != 2 or c.shape[1] < 1:
        raise ValueError("counts must be [B, C >= 1], got shape %s" % (c.shape,))
    if not np.issubdtype(c.dtype, np.integer) or (c < 0).any():
        raise ValueError("counts must be non-negative integers")
    return c.astype(np.int64)


def smooth_counts(model, src, static, times, lengths, *, sigma, n_samples, seed=0, step=0, sensors=None,
                  perturb_static=False, internal_batch_size=None):
    """Votes of the smoothed classifier: counts [B, C] int64 on the model's device, counts[b, c] = how many of n_samples
    noisy replicates x_b + sigma z of sample b the eval-mode model classifies as c (first maximum of the logits; a
    replicate with a non-finite logit votes for no class, so a row sums to at most n_samples).

    sigma:      the noise level, finite and >= 0, in normalised units.  n_samples: n >= 1 replicates per sample.
    seed, step: replicate m draws its noise at Philox key (seed, step + m), indexed by (sample, t, sensor): a sample's
                counts depend on neither B nor the chunking.  The model's dropout stream is neither read nor advanced.
    sensors:    None (every sensor) or a bool [d_inp]: only those sensors' observed cells get noise.
    perturb_static: noise on the static vector too (needs a model with a static branch).
    internal_batch_size: (replicate, sample) rows per chunk, i.e. max(1, internal_batch_size // B) replicates per chunk.
                Default: the largest chunk whose scratch fits in 1 GiB.  The counts do not depend on it once
                model._plan.obprop_mode is pinned (mode 0 picks the ob-prop arithmetic from the chunk's row count).

    Stream-ordered and sync-free apart from the host checks; changes neither the parameters, their .grad, the model's
    rng state nor a bound FlatAdam, and can be captured in a CUDA graph (after an eager call with the same key and
    shapes).  Raises ValueError for a model in training mode or invalid arguments, and RaindropB200Error without CUDA."""
    _check_call("smooth_counts", model, src, static, None, internal_batch_size)
    sigma = _check_sigma(sigma)
    n_samples = _check_n("n_samples", n_samples)
    seed, step = _check_key(seed, step)
    if step + n_samples > 1 << 64:
        raise ValueError("step + n_samples must be <= 2^64")
    if perturb_static and not model.static:
        raise ValueError("perturb_static needs a model with a static branch")
    plan = model._plan
    if sensors is not None:
        _sensor_mask(sensors, plan.N, "cpu")          # shape and dtype checked before anything touches the device
    with torch.no_grad():
        cl = _Call(model, src, static, times, lengths, None, False)
        lib, B, dev = cl.lib, src.shape[1], cl.device
        sens = _sensor_mask(sensors, plan.N, dev)
        dims = plan.dims(B, False)
        cc, scratch = cl.chunk_scratch("_smooth_scratch", "rd_smooth_scratch_bytes", dims, n_samples, internal_batch_size)
        key = _device_key(plan, seed, step, dev)
        counts = torch.empty(B, plan.n_classes, dtype=torch.int64, device=dev)
        L.check(lib.rd_raindrop_v2_smooth_counts(C.byref(dims), C.byref(cl.params), cl.x.data_ptr(), L.ptr(cl.st),
                                                 cl.tm.data_ptr(), cl.ln.data_ptr(), plan.node_scale.data_ptr(),
                                                 L.ptr(sens), int(bool(perturb_static)), sigma, key.data_ptr(), n_samples,
                                                 cc, scratch.data_ptr(), counts.data_ptr(), L.stream_ptr(dev)),
                "rd_raindrop_v2_smooth_counts")
    return counts


def predict_from_counts(counts, alpha=0.001):
    """Cohen's PREDICT from votes counts [B, C] (tensor or array), in float64 on the host: the top class c_A (ties: the
    lowest index) when the two-sided binomial test of n_A against n_A + n_B at p = 1/2 (n_B the runner-up's count) has
    p-value <= alpha, else -1 (abstain).  Returns int64 [B]."""
    from scipy.stats import binomtest
    c = _counts(counts)
    alpha = _check_alpha(alpha)
    top = np.argmax(c, axis=1)
    out = np.full(c.shape[0], -1, dtype=np.int64)
    for b in range(c.shape[0]):
        nA = int(c[b, top[b]])
        nB = int(np.delete(c[b], top[b]).max()) if c.shape[1] > 1 else 0
        if nA + nB > 0 and binomtest(nA, nA + nB, 0.5).pvalue <= alpha:
            out[b] = top[b]
    return out


def selection_lower_bound(counts0, counts, alpha, n=None):
    """The step CERTIFY shares between smoothing and ablation, in float64 on the host: c_A = argmax counts0 (ties: the
    lowest index) and p_lower = the one-sided (1 - alpha) Clopper-Pearson lower bound beta.ppf(alpha, k, n - k + 1) of
    P(f = c_A) from k = counts[b, c_A] of n draws (0 for k = 0).  n: the estimation draws per sample (default: the row
    sums of counts; give it when replicates may have voted for no class, so that they count against c_A).  alpha is
    checked by the caller.  Returns (c_A int64 [B], p_lower float64 [B])."""
    from scipy.stats import beta
    c0, c = _counts(counts0), _counts(counts)
    if c0.shape != c.shape:
        raise ValueError("counts0 and counts must have the same shape, got %s and %s" % (c0.shape, c.shape))
    ca = np.argmax(c0, axis=1)
    k = c[np.arange(c.shape[0]), ca].astype(np.float64)
    nn = c.sum(axis=1) if n is None else np.broadcast_to(np.asarray(n, dtype=np.int64), k.shape)
    if (nn < c.sum(axis=1)).any() or (nn < 1).any():
        raise ValueError("n must be >= 1 and at least each row's vote count")
    nn = nn.astype(np.float64)
    return ca, np.where(k > 0, beta.ppf(alpha, np.maximum(k, 1.0), nn - k + 1.0), 0.0)


def certify_from_counts(counts0, counts, sigma, alpha=0.001, n=None):
    """Cohen's CERTIFY from selection votes counts0 and estimation votes counts ([B, C], tensors or arrays), in float64
    on the host: c_A and p_lower as selection_lower_bound computes them, and radius = sigma Phi^-1(p_lower), or
    prediction -1 and radius -1 when p_lower < 1/2.  n: the estimation draws per sample (default: the row sums of
    counts).  Returns (prediction int64 [B], radius float64 [B], p_lower float64 [B])."""
    from scipy.stats import norm
    sigma, alpha = _check_sigma(sigma), _check_alpha(alpha)
    ca, p_lower = selection_lower_bound(counts0, counts, alpha, n)
    ok = p_lower >= 0.5
    radius = np.where(ok, sigma * norm.ppf(np.where(ok, p_lower, 0.5)), -1.0)
    return np.where(ok, ca, -1).astype(np.int64), radius.astype(np.float64), p_lower.astype(np.float64)


def predict(model, src, static, times, lengths, *, sigma, n_samples=1000, alpha=0.001, seed=0, step=0, sensors=None,
            perturb_static=False, internal_batch_size=None):
    """Cohen's PREDICT of the smoothed classifier: predict_from_counts of smooth_counts (arguments as there).  Returns
    int64 [B] on the host: the class, or -1 (abstain).  The probability of returning a class other than g(x) is at
    most alpha."""
    alpha = _check_alpha(alpha)
    counts = smooth_counts(model, src, static, times, lengths, sigma=sigma, n_samples=n_samples, seed=seed, step=step,
                           sensors=sensors, perturb_static=perturb_static, internal_batch_size=internal_batch_size)
    return predict_from_counts(counts, alpha)


def certify(model, src, static, times, lengths, *, sigma, n0=100, n_samples=100_000, alpha=0.001, seed=0, step=0,
            sensors=None, perturb_static=False, internal_batch_size=None):
    """Cohen's CERTIFY of the smoothed classifier.  n0 selection replicates at key (seed, step) pick c_A; n_samples
    estimation replicates at (seed, step + n0) -- disjoint noise -- bound P(f(x + sigma z) = c_A) from below, and
    certify_from_counts turns the bound into an L2 radius over the perturbable set S_b in normalised units (the threat
    model of pgd(norm="l2")).  With probability >= 1 - alpha over the noise, a sample that does not abstain has
    g(x + delta) = prediction for every delta on S_b with ||delta||_2 < radius.  Other arguments as smooth_counts.
    Returns a CertifyResult."""
    alpha = _check_alpha(alpha)
    n0 = _check_n("n0", n0)
    n_samples = _check_n("n_samples", n_samples)
    seed, step = _check_key(seed, step)
    kw = dict(sigma=sigma, seed=seed, sensors=sensors, perturb_static=perturb_static,
              internal_batch_size=internal_batch_size)
    counts0 = smooth_counts(model, src, static, times, lengths, n_samples=n0, step=step, **kw)
    counts = smooth_counts(model, src, static, times, lengths, n_samples=n_samples, step=step + n0, **kw)
    pred, radius, p_lower = certify_from_counts(counts0, counts, sigma, alpha, n=n_samples)
    return CertifyResult(pred, radius, p_lower, counts0, counts)


class AugmentedTrainStep(TrainStep):
    """A TrainStep that trains on a copy of the loaded batch augmented on the device every step (Gaussian noise,
    random ablation), the whole step one CUDA graph.  The clean batch goes where TrainStep keeps it (load_batch,
    DeviceDataset.fill); the augmented copy lands in noisy_src / noisy_static, which the training forward reads.  The
    augmentation is drawn at a device key {seed, step} that every step advances by one, so a resumed run restores it
    with noise_key_state() / set_noise_key().  A subclass checks its arguments and refuse_distributed() before calling
    __init__ (which touches the model), and implements _augment(stream).  One GPU only."""

    augmentation = None     # the kind of training, in the one-GPU error

    @classmethod
    def refuse_distributed(cls, group):
        if dist.is_initialized() and dist.get_world_size(group) > 1:
            raise L.RaindropB200Error("%s runs on one GPU; data-parallel %s training is not supported"
                                      % (cls.__name__, cls.augmentation))

    def __init__(self, model, batch_size, noise_seed, lr, use_graph, betas, adam_eps, group):
        seed = int.from_bytes(os.urandom(8), "little") if noise_seed is None else int(noise_seed)
        _check_key(seed, 0)
        super().__init__(model, batch_size, lr=lr, betas=betas, eps=adam_eps, group=group, use_graph=use_graph,
                         distributed=False)
        self.noise_dims = self.plan.dims(self.B, False)
        self.noisy_src = torch.zeros_like(self.src)
        self.noisy_static = torch.zeros_like(self.static) if self.static is not None else None
        self.noise_key = torch.tensor(np.array([seed, 0], dtype=np.uint64).view(np.int64), device=self.device)

    def _inputs(self):
        return self.noisy_src, self.noisy_static, self.times, self.lengths

    def _state(self):
        extra = (self.noise_key, self.noisy_src) + ((self.noisy_static,) if self.noisy_static is not None else ())
        return super()._state() + extra

    def _augment(self, st):
        raise NotImplementedError

    def _enqueue(self):
        self._augment(L.stream_ptr(self.device))
        self.noise_key[1:].add_(1)
        super()._enqueue()

    def noise_key_state(self):
        """(seed, step) of the noise stream, to be saved with a checkpoint (reads the device key: synchronises)."""
        seed, step = (int(v) for v in self.noise_key.cpu().numpy().view(np.uint64))
        return seed, step

    def set_noise_key(self, seed, step):
        """Restores a saved noise_key_state(); the next step draws the noise of that step."""
        seed, step = _check_key(seed, step)
        self.noise_key.copy_(torch.tensor(np.array([seed, step], dtype=np.uint64).view(np.int64)))


class SmoothingTrainStep(AugmentedTrainStep):
    """Gaussian data augmentation (Cohen et al. 2019; Lecuyer et al. 2019) on static device buffers: each step draws
    x + sigma z for the loaded batch with smooth_counts' noise (one replicate at the device key {seed, step}, on the
    same perturbable set), then runs TrainStep's forward, backward and Adam on the noisy copy -- all on the device, one
    CUDA graph per step.  A model trained this way keeps its accuracy under the noise that certify adds.

    The noisy copy lands in noisy_src / noisy_static (AugmentedTrainStep).  noise_seed: the Philox seed (default: 64
    bits from os.urandom); save and restore the key with noise_key_state() / set_noise_key().  At sigma = 0 a step is
    TrainStep's bit for bit.  adam_eps is Adam's epsilon.  One GPU only."""

    augmentation = "smoothing"

    def __init__(self, model, batch_size, sigma, sensors=None, perturb_static=False, noise_seed=None, lr=1e-4,
                 use_graph=True, betas=(0.9, 0.999), adam_eps=1e-8, group=None):
        self.refuse_distributed(group)
        self.sigma = _check_sigma(sigma)
        self.perturb_static = bool(perturb_static)
        if self.perturb_static and not model.static:
            raise ValueError("perturb_static needs a model with a static branch")
        if sensors is not None:
            _sensor_mask(sensors, model._plan.N, "cpu")
        super().__init__(model, batch_size, noise_seed, lr, use_graph, betas, adam_eps, group)
        self.sensors = _sensor_mask(sensors, self.plan.N, self.device)

    def _augment(self, st):
        L.check(self.lib.rd_debug_smoothing_inputs(C.byref(self.noise_dims), self.src.data_ptr(), L.ptr(self.static),
                                                   self.times.data_ptr(), self.lengths.data_ptr(), L.ptr(self.sensors),
                                                   int(self.perturb_static), self.sigma, self.noise_key.data_ptr(), 0, 1,
                                                   self.noisy_src.data_ptr(), L.ptr(self.noisy_static), None, None, st),
                "rd_debug_smoothing_inputs")
