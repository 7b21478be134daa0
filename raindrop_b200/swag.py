"""SWA and SWAG of Raindrop_v2 (Izmailov et al. 2018, "Averaging Weights Leads to Wider Optima"; Maddox et al. 2019,
"A Simple Baseline for Bayesian Uncertainty in Deep Learning"), and MultiSWAG (Wilson & Izmailov 2020), computed on the
device.

A SWAG posterior is collected from the training trajectory: after each epoch (or every c steps) of training at a
constant or cyclical learning rate, one launch folds the current weights theta into fp64 running moments and keeps the
last `rank` deviations theta - mean as a low-rank factor D:

    posterior = SWAG(model, rank=20)
    for epoch in range(swa_epochs):
        ...  # TrainStep.step() over the epoch, at the SWA learning rate (TrainStep.set_lr)
        posterior.collect(step)
    posterior.load_mean(model)                       # the SWA model
    res = swag_predictive(model.eval(), posterior, src, static, times, lengths, n_samples=30)
    res = swag_predictive(model, [posterior_a, posterior_b], ...)      # MultiSWAG: several independently trained runs

The posterior is N(mean, scale (diag(sq_mean - mean^2) + D D^T / (k - 1))), k = min(collected, rank) columns; scale 0.5
gives the paper's sampler.  swag_predictive averages the softmax of the eval forward over weight samples and returns the
statistics of uncertainty.mc_dropout; with scale = 0 and n_samples = 1 it is the deep ensemble of the members' SWA
weights.  The moments are kept in fp64: sq_mean - mean^2 cancels catastrophically in fp32 at the weight variances of a
converged run (a variance of 1e-8 under a weight of magnitude 1e-1 is below fp32's resolution of sq_mean).

swag_from_snapshots and swag_sample_from_state are float64 numpy restatements of the two kernels: the documented
semantics, and the oracle of the tests.
"""
import ctypes as C
import math

import numpy as np
import torch

from . import functional as RF
from . import lib as L
from .attribution import _Call, _check_call
from .influence import _bucket_length, grad_layout
from .uncertainty import MCDropoutResult, _device_key

SITE_SWAG = 102


class SWAGResult(MCDropoutResult):
    """The Bayesian model average of swag_predictive over the M = n_members * n_samples weight samples, with the field
    names and definitions of uncertainty.MCDropoutResult (fp32 tensors on the device; samples [M, B, C] only with
    return_samples)."""


def _layout_key(layout):
    return [(k, int(o), tuple(int(x) for x in s)) for k, o, s in layout]


def _check_rank(rank):
    if isinstance(rank, bool) or int(rank) != rank or not 0 <= int(rank) <= L.SWAG_MAX_RANK:
        raise ValueError("rank must be an integer in [0, %d], got %r" % (L.SWAG_MAX_RANK, rank))
    return int(rank)


def _check_scale(scale):
    s = float(scale)
    if not (math.isfinite(s) and s >= 0):
        raise ValueError("scale must be finite and >= 0, got %r" % (scale,))
    return s


def _check_key(seed, step, n):
    seed, step = int(seed), int(step)
    if not 0 <= seed < 1 << 64:
        raise ValueError("seed must be in [0, 2^64), got %d" % seed)
    if step < 0 or step + n > 1 << 64:
        raise ValueError("step must be >= 0 with step + %d <= 2^64, got %d" % (n, step))
    return seed, step


class SWAG:
    """An SWAG posterior over the trained tensors of a Raindrop_v2 (its used_parameters, in TrainStep's flat bucket
    layout `layout` = influence.grad_layout(model), n floats).  Device buffers on the model's device: mean and sq_mean
    (float64 [n]), dev (float32 [rank, n], slot c % rank holds the deviation of snapshot c); n_collected snapshots.
    rank = 0 keeps the diagonal only (SWAG-diagonal)."""

    def __init__(self, model, rank=20):
        self.rank = _check_rank(rank)
        self.layout = grad_layout(model)
        self.n = _bucket_length(self.layout)
        self.device = model.used_parameters()[0].device
        self.mean = torch.zeros(self.n, dtype=torch.float64, device=self.device)
        self.sq_mean = torch.zeros(self.n, dtype=torch.float64, device=self.device)
        self.dev = torch.zeros(self.rank, self.n, dtype=torch.float32, device=self.device)
        self.n_collected = 0

    @property
    def k(self):
        """Deviation columns that hold data: min(n_collected, rank)."""
        return min(self.n_collected, self.rank)

    def _check_model(self, model, what="model"):
        if _layout_key(grad_layout(model)) != _layout_key(self.layout):
            raise ValueError("%s's trained tensors differ from the posterior's layout" % what)

    def _bucket(self, source):
        """theta [n] fp32 on the device: TrainStep / FlatAdam's flat_p itself, or a model's used parameters packed."""
        from .models_rd import Raindrop_v2
        from .optim import FlatAdam
        from .train import TrainStep
        if isinstance(source, (TrainStep, FlatAdam)):
            self._check_model(source.model, "the source's model")
            theta = source.flat_p.detach()
        elif isinstance(source, Raindrop_v2):
            self._check_model(source)
            theta = torch.zeros(self.n, dtype=torch.float32, device=self.device)
            for (_, off, shape), p in zip(self.layout, source.used_parameters()):
                theta[off:off + math.prod(shape)].copy_(p.detach().reshape(-1))
        else:
            raise TypeError("collect takes a TrainStep, a FlatAdam or a Raindrop_v2, got %s" % type(source).__name__)
        if theta.numel() != self.n or theta.dtype != torch.float32 or theta.device != self.device:
            raise ValueError("the source's bucket is not [%d] float32 on %s" % (self.n, self.device))
        return theta

    def collect(self, source):
        """Folds the current weights of `source` (a TrainStep, a FlatAdam or the Raindrop_v2 itself) into the posterior:
        one launch on the current stream that only reads the weights, so training is unaffected bit for bit."""
        theta = self._bucket(source)
        if self.device.type != "cuda":
            raise L.RaindropB200Error("SWAG.collect needs the posterior on a CUDA device")
        lib = L.load()
        with torch.no_grad():
            L.check(lib.rd_swag_collect(theta.data_ptr(), self.n, self.n_collected, self.rank, self.mean.data_ptr(),
                                        self.sq_mean.data_ptr(), L.ptr(self.dev) if self.rank > 0 else None,
                                        L.stream_ptr(self.device)), "rd_swag_collect")
        self.n_collected += 1

    def _require_data(self):
        if self.n_collected < 1:
            raise ValueError("the SWAG posterior is empty: collect at least one snapshot first")

    def load_mean(self, model):
        """Writes fp32(mean) into the model's trained tensors: the SWA model.  Raindrop_v2 has LayerNorm and no
        BatchNorm, so the averaged weights need no statistics pass."""
        self._require_data()
        self._check_model(model)
        with torch.no_grad():
            for (_, off, shape), p in zip(self.layout, model.used_parameters()):
                p.copy_(self.mean[off:off + math.prod(shape)].view(shape).to(p.dtype))

    def sample_weights(self, seed=0, step=0, scale=0.5):
        """One weight vector of the posterior, flat fp32 [n] in the bucket layout (rd_swag_sample at key (seed, step),
        replicate 0); swag_predictive's replicate r draws sample_weights(seed, step + r, scale) of its member."""
        self._require_data()
        scale = _check_scale(scale)
        seed, step = _check_key(seed, step, 1)
        if self.device.type != "cuda":
            raise L.RaindropB200Error("SWAG.sample_weights needs the posterior on a CUDA device")
        lib = L.load()
        key = torch.tensor(np.array([seed, step], dtype=np.uint64).view(np.int64), device=self.device)
        out = torch.empty(self.n, dtype=torch.float32, device=self.device)
        L.check(lib.rd_swag_sample(self.mean.data_ptr(), self.sq_mean.data_ptr(), L.ptr(self.dev) if self.k >= 2 else None,
                                   self.n, self.k, scale, key.data_ptr(), 0, out.data_ptr(), L.stream_ptr(self.device)),
                "rd_swag_sample")
        return out

    def save(self, path):
        torch.save(dict(layout=_layout_key(self.layout), rank=self.rank, n_collected=self.n_collected,
                        mean=self.mean.cpu(), sq_mean=self.sq_mean.cpu(), dev=self.dev.cpu()), path)

    @classmethod
    def load(cls, path, model):
        """A saved posterior, on the model's device; refused when the model's trained tensors have another layout."""
        d = torch.load(path, map_location="cpu", weights_only=True)
        out = cls(model, rank=int(d["rank"]))
        if [tuple(e) for e in d["layout"]] != [(k, o, tuple(s)) for k, o, s in _layout_key(out.layout)]:
            raise ValueError("the saved SWAG posterior was collected for a model with another layout")
        out.mean.copy_(d["mean"])
        out.sq_mean.copy_(d["sq_mean"])
        out.dev.copy_(d["dev"])
        out.n_collected = int(d["n_collected"])
        return out


# ---- float64 restatements ---------------------------------------------------------------------------------------------
def swag_from_snapshots(thetas, rank):
    """(mean, sq_mean, dev, k) of rd_swag_collect over the snapshots thetas [c, n] in order, float64 numpy (dev float32
    [rank, n]): mean = (c mean + theta) / (c + 1), sq_mean likewise with theta^2, slot c % rank of dev =
    fp32(theta - mean'), k = min(c, rank)."""
    rank = _check_rank(rank)
    th = np.asarray(thetas, dtype=np.float32).astype(np.float64)
    if th.ndim != 2:
        raise ValueError("thetas must be [c, n]")
    n = th.shape[1]
    mean, sq = np.zeros(n), np.zeros(n)
    dev = np.zeros((rank, n), dtype=np.float32)
    for c in range(th.shape[0]):
        t = th[c]
        mean = (c * mean + t) / (c + 1.0)
        sq = (c * sq + t * t) / (c + 1.0)
        if rank > 0:
            dev[c % rank] = (t - mean).astype(np.float32)
    return mean, sq, dev, min(th.shape[0], rank)


def swag_normals(seed, step, idx):
    """The site-102 standard normals of element indices idx at key (seed, step), float32: Box-Muller on the Philox block's
    word pairs as rd_dp_add_noise draws them (element i: block i >> 2, words (x, y) for i & 3 in {0, 1}, (z, w) for
    {2, 3}; cosine for even i, sine for odd)."""
    from oracle.dropout_masks import philox4x32_10
    seed, step = int(seed) & 0xFFFFFFFFFFFFFFFF, int(step) & 0xFFFFFFFFFFFFFFFF
    idx = np.asarray(idx, dtype=np.uint64)
    blk = idx >> np.uint64(2)
    ctr = np.stack([blk & np.uint64(0xFFFFFFFF), blk >> np.uint64(32), np.full_like(blk, SITE_SWAG),
                    np.full_like(blk, step & 0xFFFFFFFF)], -1)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) ^ (step >> 32)], dtype=np.uint64)
    w = philox4x32_10(ctr, key).astype(np.uint64)
    hi = (idx & np.uint64(2)) != 0
    a = np.where(hi, w[..., 2], w[..., 0])
    b = np.where(hi, w[..., 3], w[..., 1])
    u1 = ((a >> np.uint64(8)).astype(np.float64) + 1.0) * (1.0 / 16777216.0)
    u2 = (b >> np.uint64(8)).astype(np.float64) * (1.0 / 16777216.0)
    r, t = np.sqrt(-2.0 * np.log(u1)), 6.283185307179586 * u2
    return np.where((idx & np.uint64(1)) != 0, r * np.sin(t), r * np.cos(t)).astype(np.float32)


def swag_sample_from_state(mean, sq_mean, dev, k, scale, seed, step, replicate=0):
    """rd_swag_sample in float64 numpy: fp32(mean + sqrt(scale) (sqrt(max(sq_mean - mean^2, 0)) z1 + [k >= 2]
    sum_{j<k} dev[j] z2_j / sqrt(k - 1))), the slot sum in slot order, z = swag_normals at key (seed, step + replicate):
    z1 = elements 0 .. n-1, z2 = elements n .. n+k-1."""
    mean = np.asarray(mean, dtype=np.float64)
    sq = np.asarray(sq_mean, dtype=np.float64)
    n, k, scale = mean.shape[0], int(k), _check_scale(scale)
    key = int(step) + int(replicate)
    z1 = swag_normals(seed, key, np.arange(n)).astype(np.float64)
    a = np.sqrt(np.maximum(sq - mean * mean, 0.0)) * z1
    if k >= 2:
        d = np.asarray(dev, dtype=np.float32)[:k].astype(np.float64)
        z2 = swag_normals(seed, key, n + np.arange(k)).astype(np.float64)
        s = np.zeros(n)
        for j in range(k):
            s = s + d[j] * z2[j]
        a = a + s / np.sqrt(float(k - 1))
    return (mean + np.sqrt(scale) * a).astype(np.float32)


# ---- the predictive ---------------------------------------------------------------------------------------------------
def _members(model, posterior):
    members = list(posterior) if isinstance(posterior, (list, tuple)) else [posterior]
    if not members:
        raise ValueError("posterior must be a SWAG or a non-empty list of them")
    for p in members:
        if not isinstance(p, SWAG):
            raise TypeError("posterior must be a SWAG or a list of SWAG, got %s" % type(p).__name__)
        p._require_data()
        p._check_model(model)
    if len({p.device for p in members}) != 1:
        raise ValueError("the members of a MultiSWAG posterior must be on one device")
    return members


def swag_predictive(model, posterior, src, static, times, lengths, n_samples=30, scale=0.5, seed=0, step=0,
                    internal_batch_size=None, return_samples=False):
    """SWAGResult of the batch under an SWAG posterior, or MultiSWAG under a list of them: replicate
    r = member * n_samples + s is the eval forward of the batch with the weights member.sample_weights(seed, step + r,
    scale), and the replicates are reduced as mc_dropout reduces its own (rd_raindrop_v2_swag_predictive, one call).

    internal_batch_size: samples per forward chunk (default: the largest chunk <= B whose scratch fits in 1 GiB).  The
    result is bitwise independent of it, except that obprop_mode 0 (auto) picks the ob-prop arithmetic from the chunk's
    row count: pin model._plan.obprop_mode for results independent of it.

    Eval arithmetic whatever the model's mode; leaves the mode, the parameters, their .grad, the dropout counter and any
    bound FlatAdam / TrainStep unchanged.  Runs under no_grad, stream-ordered and sync-free, and can be captured in a
    CUDA graph (after an eager call with the same key and shapes).  Raises RaindropB200Error without CUDA or without the
    built library."""
    _check_call("swag_predictive", model, src, static, None, internal_batch_size, train_ok=True)
    members = _members(model, posterior)
    if isinstance(n_samples, bool) or int(n_samples) != n_samples or not 1 <= int(n_samples) <= 0x7FFFFFFF:
        raise ValueError("n_samples must be an integer in [1, 2^31), got %r" % (n_samples,))
    n_samples = int(n_samples)
    M = n_samples * len(members)
    if M > 0x7FFFFFFF:
        raise ValueError("n_samples * members = %d must be < 2^31" % M)
    scale = _check_scale(scale)
    seed, step = _check_key(seed, step, M)
    plan = model._plan
    with torch.no_grad():
        cl = _Call(model, src, static, times, lengths, None, False)
        lib, B, dev = cl.lib, src.shape[1], cl.device
        if members[0].device != dev:
            raise ValueError("the posterior is on %s, the inputs on %s" % (members[0].device, dev))
        dims = plan.dims(B, False)
        rpc, scratch = cl.chunk_scratch("_swag_scratch", "rd_swag_predictive_scratch_bytes", dims, B,
                                        internal_batch_size, per_sample=True)
        n = members[0].n
        theta = cl.scratch("_swag_theta", (n, dev.index), 4 * n)
        params = L.RdParams()
        params.R_u = plan.R_u.data_ptr()
        for (_, path), (_, off, _) in zip(plan.fields, members[0].layout):
            RF._set_field(params, path, theta.data_ptr() + 4 * off)
        table = (L.RdSwagMember * len(members))()
        for t, p in zip(table, members):
            t.mean, t.sq_mean, t.k = p.mean.data_ptr(), p.sq_mean.data_ptr(), p.k
            t.dev = p.dev.data_ptr() if p.k >= 2 else None
        key = _device_key(plan, seed, step, dev)
        f32 = dict(device=dev, dtype=torch.float32)
        mean = torch.empty(B, plan.n_classes, **f32)
        var = torch.empty(B, plan.n_classes, **f32)
        ent = torch.empty(3, B, **f32)
        samples = torch.empty(M, B, plan.n_classes, **f32) if return_samples else None
        L.check(lib.rd_raindrop_v2_swag_predictive(C.byref(dims), C.byref(params), cl.x.data_ptr(), L.ptr(cl.st),
                                                   cl.tm.data_ptr(), cl.ln.data_ptr(), plan.node_scale.data_ptr(), table,
                                                   len(members), scale, key.data_ptr(), n_samples, theta.data_ptr(), n,
                                                   rpc, scratch.data_ptr(), mean.data_ptr(), var.data_ptr(),
                                                   ent.data_ptr(), L.ptr(samples), L.stream_ptr(dev)),
                "rd_raindrop_v2_swag_predictive")
    return SWAGResult(mean, var, ent[0], ent[1], ent[2], samples)
