"""Monte Carlo dropout predictive uncertainty of Raindrop_v2, computed on the device in one call per batch
(rd_raindrop_v2_mc_dropout).

Raindrop_v2 is trained with dropout (the lift, and per encoder layer the attention probabilities, dropout1, the FFN and
dropout2).  Monte Carlo dropout keeps those masks active at inference and averages M stochastic forwards; how much the
replicates disagree is the model's uncertainty, with no retraining:

    res = mc_dropout(model, src, static, times, lengths, n_samples=30)
    pred = res.mean_probs.argmax(dim=1)
    keep = res.mutual_information.argsort()[: int(0.8 * B)]     # the 80 % of samples the model is surest about

Replicate m of a call with key (seed, step) is exactly the training-mode forward of the batch at dropout key
(seed, step + m) -- the forward Raindrop_v2 runs in train() mode with plan.rng_state = (seed, step + m) -- and its masks
are the documented Philox stream (oracle/dropout_masks.py restates it).  The model's own counter is never advanced.
"""
import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from . import lib as L
from .attribution import _Call, _check_call


@dataclass
class MCDropoutResult:
    """Per-sample statistics over the M replicates, p_m = softmax(logits_m) (fp64 arithmetic):
    mean_probs [B, C] = mean p_m; variance [B, C] = sample variance of p_m (divisor M - 1, 0 when M = 1);
    predictive_entropy [B] = H(mean p); expected_entropy [B] = mean H(p_m); mutual_information [B] = their difference
    (natural log, 0 log 0 = 0); samples [M, B, C] = the replicates' logits, when requested."""
    mean_probs: object
    variance: object
    predictive_entropy: object
    expected_entropy: object
    mutual_information: object
    samples: object = None


def _check_logits(logits):
    x = logits.detach().cpu().double().numpy() if torch.is_tensor(logits) else np.asarray(logits, dtype=np.float64)
    if x.ndim != 3 or min(x.shape) < 1:
        raise ValueError("logits must be [M >= 1, B >= 1, C >= 1], got shape %s" % (x.shape,))
    if not np.all(np.isfinite(x)):
        raise ValueError("logits must be finite")
    return x


def mc_dropout_from_logits(logits):
    """The statistics of mc_dropout from per-replicate logits [M, B, C] (tensor or array), in float64 on the host.
    Returns an MCDropoutResult of float64 numpy arrays, `samples` the logits themselves."""
    x = _check_logits(logits)
    M = x.shape[0]
    mx = x.max(axis=2, keepdims=True)
    lp = (x - mx) - np.log(np.exp(x - mx).sum(axis=2, keepdims=True))
    p = np.exp(lp)
    h = -(p * lp).sum(axis=2)                               # [M, B]; p = 0 contributes 0 (lp is finite)
    mean = p.mean(axis=0)
    var = p.var(axis=0, ddof=1) if M > 1 else np.zeros_like(mean)
    pos = mean > 0
    pred = -np.where(pos, mean * np.log(np.where(pos, mean, 1.0)), 0.0).sum(axis=1)
    expected = h.mean(axis=0)
    return MCDropoutResult(mean, var, pred, expected, pred - expected, x)


def _device_key(plan, seed, step, device):
    """Device uint64 {seed, step} (held as int64), cached per plan in one entry that another key replaces: a CUDA-graph
    capture after an eager call with the same key copies nothing.  A key read by a call under capture is held for the
    plan's lifetime, so the graph's replays stay valid after later calls replace the entry."""
    k = (seed, step, device.index)
    cached = plan.__dict__.get("_mc_key")
    if cached is None or cached[0] != k:
        cached = plan.__dict__["_mc_key"] = (k, torch.tensor(np.array([seed, step], dtype=np.uint64).view(np.int64),
                                                             device=device))
    got = cached[1]
    if device.type == "cuda" and torch.cuda.is_current_stream_capturing():
        held = plan.__dict__.setdefault("_mc_keys_captured", [])
        if not any(t is got for t in held):
            held.append(got)
    return got


def mc_dropout(model, src, static, times, lengths, n_samples=30, seed=None, step=0, internal_batch_size=None,
               return_samples=False):
    """Monte Carlo dropout of a Raindrop_v2: n_samples training-mode forwards of the batch, replicate m at dropout key
    (seed, step + m), reduced to per-sample statistics on the device.  Returns an MCDropoutResult of fp32 tensors on the
    model's device (`samples` [M, B, C] only with return_samples).

    seed:     the Philox seed (0 <= seed < 2^64); None = the model's own dropout seed.  step: the first replicate's step
              counter (0 <= step, step + n_samples <= 2^64).
    internal_batch_size: (replicate, sample) rows per chunk, i.e. max(1, internal_batch_size // B) replicates per chunk.
              Default: the largest chunk whose scratch fits in 1 GiB.  The result does not depend on the chunking,
              except that obprop_mode 0 (auto) picks the ob-prop arithmetic from the chunk's row count: pin
              model._plan.obprop_mode for results independent of it.

    Works in train() and eval() mode alike and leaves the mode, the parameters, their .grad and the model's dropout
    counter unchanged; runs under no_grad, stream-ordered and sync-free, and can be captured in a CUDA graph (after an
    eager call with the same key and shapes).  Raises RaindropB200Error without CUDA or without the built library."""
    _check_call("mc_dropout", model, src, static, None, internal_batch_size, train_ok=True)
    n_samples = int(n_samples)
    if n_samples < 1 or n_samples > 0x7FFFFFFF:
        raise ValueError("n_samples must be in [1, 2^31), got %d" % n_samples)
    seed = model._seed if seed is None else int(seed)
    step = int(step)
    if not 0 <= seed < 1 << 64:
        raise ValueError("seed must be in [0, 2^64), got %d" % seed)
    if step < 0 or step + n_samples > 1 << 64:
        raise ValueError("step must be >= 0 with step + n_samples <= 2^64, got %d" % step)
    plan = model._plan
    with torch.no_grad():
        cl = _Call(model, src, static, times, lengths, None, False)
        lib, B = cl.lib, src.shape[1]
        dims = plan.dims(B, True)
        cc, scratch = cl.chunk_scratch("_mc_scratch", "rd_mc_dropout_scratch_bytes", dims, n_samples, internal_batch_size)
        key = _device_key(plan, seed, step, cl.device)
        f32 = dict(device=cl.device, dtype=torch.float32)
        mean = torch.empty(B, plan.n_classes, **f32)
        var = torch.empty(B, plan.n_classes, **f32)
        ent = torch.empty(3, B, **f32)
        samples = torch.empty(n_samples, B, plan.n_classes, **f32) if return_samples else None
        L.check(lib.rd_raindrop_v2_mc_dropout(C.byref(dims), C.byref(cl.params), cl.x.data_ptr(), L.ptr(cl.st),
                                              cl.tm.data_ptr(), cl.ln.data_ptr(), plan.node_scale.data_ptr(),
                                              key.data_ptr(), n_samples, cc, scratch.data_ptr(), mean.data_ptr(),
                                              var.data_ptr(), ent.data_ptr(), L.ptr(samples), L.stream_ptr(cl.device)),
                "rd_raindrop_v2_mc_dropout")
    return MCDropoutResult(mean, var, ent[0], ent[1], ent[2], samples)
