"""Batch active learning for Raindrop_v2: which records of an unlabelled pool to label next, computed on the device.

Labels of P12 / P19 stays are a clinician's review of a whole stay, so a labelling round asks for a batch of k.  Taking
the k largest single-point BALD scores picks near-duplicates; the two standard remedies are here:

    logits = pool_logits(model.eval(), (pool_ds, pool_idx), n_samples=100)        # [M, N, C] over the pool
    res = batch_bald(logits, k=100)                                               # Kirsch et al. 2019
    res = badge(model, (pool_ds, pool_idx), k=100)                                # Ash et al. 2020

batch_bald   greedy BatchBALD: pick i maximises the joint mutual information of the batch, H(y_A, y_n) minus the sum of
             the expected conditional entropies, exactly while C^|A| <= n_configs and by Kirsch's importance-weighted
             estimate over n_configs sampled configurations beyond (rd_batch_bald).
badge        k-means++ seeding over the last-layer gradient embeddings (p - e_yhat) (x) [h; 1], h = the head's hidden
             activation, with distances in factorised form (rd_badge).
pool_logits  the posterior replicates' logits over a whole pool from mc_dropout, swag_predictive or
             laplace_predictive(link="mc"); it adds no kernel.

Both acquisitions are one stream-ordered call whose greedy loop never synchronises with the host, capturable in a CUDA
graph after an eager call with the same key and shapes, and bitwise independent of internal_batch_size.
oracle/active_oracle.py restates both in numpy float64.
"""
from dataclasses import dataclass

import numpy as np
import torch

from . import lib as L
from .influence import _check_batch_size, _check_data, _source

DEFAULT_SCRATCH_BYTES = 1 << 30
FEATURE_BLOCK = 4096        # pool records per ood.features call of badge


@dataclass
class BatchBALDResult:
    """indices [k] int64: the picks in order; scores [k] float64: the estimated joint mutual information of the batch
    after each pick; exact [k] bool: which picks enumerated every configuration; bald [N] float64: the single-point
    mutual information (scores[0] == bald[indices[0]])."""
    indices: object
    scores: object
    exact: object
    bald: object


@dataclass
class BadgeResult:
    """indices [k] int64: the picks in order; d2 [k] float64: each pick's squared distance to the nearest earlier pick
    at the time it was drawn (inf for the first, which is the largest-norm embedding)."""
    indices: object
    d2: object


def _int(x, what, lo, hi):
    if isinstance(x, bool) or not isinstance(x, (int, np.integer)) or not lo <= int(x) <= hi:
        raise ValueError("%s must be an integer in [%d, %d], got %r" % (what, lo, hi, x))
    return int(x)


def _key(seed, step):
    return _int(seed, "seed", 0, (1 << 64) - 1), _int(step, "step", 0, (1 << 64) - 1)


def _cuda_tensor(x, what):
    if not torch.is_tensor(x):
        raise TypeError("%s must be a torch tensor" % what)
    if not torch.cuda.is_available() or x.device.type != "cuda":
        raise L.RaindropB200Error("%s needs CUDA: pass tensors on a CUDA device (there is no CPU path)" % what)
    return x.detach().to(torch.float32).contiguous()


def _check_finite(x, what):
    """One host synchronisation, skipped under CUDA-graph capture (where the eager call with the same inputs has
    already checked them)."""
    if x.is_cuda and torch.cuda.is_current_stream_capturing():
        return
    if not bool(torch.isfinite(x).all()):
        raise ValueError("%s must be finite" % what)


def batch_bald(logits, k, n_configs=10_000, seed=0, step=0, internal_batch_size=None):
    """Greedy BatchBALD over posterior replicates' logits [M, N, C] (pool_logits, or samples of mc_dropout,
    swag_predictive or laplace_predictive(link="mc")).  Returns a BatchBALDResult of device tensors.

    Pick i, with the chosen set A (|A| = i), is the unchosen n maximising H(y_A, y_n) - sum_{a in A u {n}} E_m H(y_a |
    theta_m), ties to the lowest index.  The joint entropy is exact while C^i <= n_configs; beyond that it is estimated
    from n_configs configurations drawn from the mixture at Philox key (seed, step) (see rd_batch_bald).  The first pick
    is the BALD argmax and scores[0] its mutual information.

    internal_batch_size: candidates per joint-entropy launch (default: the largest chunk whose scratch fits in 1 GiB
    beyond the fixed part); the result is bitwise independent of it.  Limits, refused with ValueError before any device
    work: 2 <= C <= 8, M <= 1024, n_configs <= 65536, 1 <= k <= N, finite logits.  Stream-ordered, no host
    synchronisation after the checks; raises RaindropB200Error without CUDA or the built library."""
    if not torch.is_tensor(logits) or logits.dim() != 3:
        raise ValueError("logits must be a tensor [M, N, C]")
    M, N, C = (int(s) for s in logits.shape)
    if not 2 <= C <= L.ACTIVE_MAX_CLASSES:
        raise ValueError("batch_bald supports 2 to %d classes, got %d" % (L.ACTIVE_MAX_CLASSES, C))
    if not 1 <= M <= L.ACTIVE_MAX_REPLICATES:
        raise ValueError("batch_bald supports 1 to %d replicates, got %d" % (L.ACTIVE_MAX_REPLICATES, M))
    if N < 1:
        raise ValueError("the pool is empty")
    k = _int(k, "k", 1, N)
    n_configs = _int(n_configs, "n_configs", 1, L.ACTIVE_MAX_CONFIGS)
    seed, step = _key(seed, step)
    _check_batch_size(internal_batch_size)
    x = _cuda_tensor(logits, "batch_bald")
    _check_finite(x, "logits")
    lib = L.load()
    if internal_batch_size is None:         # the partial sums: 8 bytes per (64 configurations, candidate)
        chunk = int(min(N, max(1, DEFAULT_SCRATCH_BYTES // (8 * ((n_configs + 63) // 64)))))
    else:
        chunk = int(min(N, int(internal_batch_size)))
    nb = lib.rd_batch_bald_scratch_bytes(N, M, C, n_configs, chunk)
    if nb == 0:
        L.check(-2, "rd_batch_bald_scratch_bytes")
    dev = x.device
    with torch.cuda.device(dev):
        scratch = torch.empty((nb + 255) // 256 * 32, dtype=torch.float64, device=dev)
        idx = torch.empty(k, dtype=torch.int64, device=dev)
        scores = torch.empty(k, dtype=torch.float64, device=dev)
        exact = torch.empty(k, dtype=torch.bool, device=dev)
        bald = torch.empty(N, dtype=torch.float64, device=dev)
        L.check(lib.rd_batch_bald(x.data_ptr(), N, M, C, k, n_configs, seed, step, chunk, scratch.data_ptr(),
                                  idx.data_ptr(), scores.data_ptr(), exact.data_ptr(), bald.data_ptr(),
                                  L.stream_ptr(dev)), "rd_batch_bald")
    return BatchBALDResult(idx, scores, exact, bald)


def badge_from_features(hidden, logits, k, seed=0, step=0):
    """BADGE's k-means++ seeding over the gradient embeddings (p_n - e_yhat_n) (x) [h_n; 1] of hidden [N, F] and logits
    [N, C] (device tensors).  The first centre is the largest-norm embedding; each later one is drawn with probability
    proportional to D^2, its squared distance to the nearest centre, by one fp64 uniform from Philox at (seed, step,
    pick).  Returns a BadgeResult of device tensors.  Limits as batch_bald (C <= 8, 1 <= k <= N, finite inputs)."""
    if not torch.is_tensor(hidden) or hidden.dim() != 2 or not torch.is_tensor(logits) or logits.dim() != 2:
        raise ValueError("hidden must be a tensor [N, F] and logits a tensor [N, C]")
    N, F = (int(s) for s in hidden.shape)
    C = int(logits.shape[1])
    if int(logits.shape[0]) != N:
        raise ValueError("hidden has %d rows, logits %d" % (N, int(logits.shape[0])))
    if not 2 <= C <= L.ACTIVE_MAX_CLASSES:
        raise ValueError("badge supports 2 to %d classes, got %d" % (L.ACTIVE_MAX_CLASSES, C))
    if N < 1 or F < 1:
        raise ValueError("hidden must be non-empty, got %s" % ((N, F),))
    k = _int(k, "k", 1, N)
    seed, step = _key(seed, step)
    h = _cuda_tensor(hidden, "badge")
    z = _cuda_tensor(logits, "badge")
    if h.device != z.device:
        raise ValueError("hidden is on %s, logits on %s" % (h.device, z.device))
    _check_finite(h, "hidden")
    _check_finite(z, "logits")
    lib = L.load()
    nb = lib.rd_badge_scratch_bytes(N, F, C)
    if nb == 0:
        L.check(-2, "rd_badge_scratch_bytes")
    dev = h.device
    with torch.cuda.device(dev):
        scratch = torch.empty((nb + 255) // 256 * 32, dtype=torch.float64, device=dev)
        idx = torch.empty(k, dtype=torch.int64, device=dev)
        d2 = torch.empty(k, dtype=torch.float64, device=dev)
        L.check(lib.rd_badge(h.data_ptr(), z.data_ptr(), N, F, C, k, seed, step, scratch.data_ptr(), idx.data_ptr(),
                             d2.data_ptr(), L.stream_ptr(dev)), "rd_badge")
    return BadgeResult(idx, d2)


def _pool(model, pool, what):
    _check_data(model, pool, what, allow_none_y=True, unlabelled=True)
    n, fetch = _source(pool, what, unlabelled=True)
    if n < 1:
        raise ValueError("%s holds no records" % what)
    return n, fetch


def _batches(n, batch_size):
    batch_size = _int(batch_size, "batch_size", 1, 1 << 31)
    return [(i0, min(n, i0 + batch_size)) for i0 in range(0, n, batch_size)]


def badge(model, pool, k, seed=0, step=0, internal_batch_size=None):
    """BADGE over an unlabelled pool: the head's hidden activation h = relu(mlp_static.0(x)) and the logits of eval
    forwards (ood.features(layer="hidden") over blocks of FEATURE_BLOCK records), then badge_from_features.  pool: a dict (src,
    static, times, lengths), a DeviceDataset (labels not needed) or (DeviceDataset, indices).  internal_batch_size is
    the forward chunk of ood.features.  Eval mode only; the model is not changed."""
    from .ood import features
    n, fetch = _pool(model, pool, "pool")
    k = _int(k, "k", 1, n)
    _key(seed, step)
    hs, zs = [], []
    for i0, i1 in _batches(n, FEATURE_BLOCK):
        src, static, times, lengths, _ = fetch(i0, i1)
        h, z = features(model, src, static, times, lengths, "hidden", internal_batch_size)
        hs.append(h)
        zs.append(z)
    h = torch.cat(hs) if len(hs) > 1 else hs[0]
    z = torch.cat(zs) if len(zs) > 1 else zs[0]
    return badge_from_features(h, z, k, seed, step)


def pool_logits(model, pool, posterior=None, n_samples=100, seed=None, step=0, batch_size=1024,
                internal_batch_size=None):
    """Posterior replicates' logits [M, N, C] (fp32, on the model's device) over a whole pool, for batch_bald.

    pool: a dict (src, static, times, lengths; no labels needed), a DeviceDataset or (DeviceDataset, indices).
    posterior: None = Monte Carlo dropout (mc_dropout, M = n_samples); a SWAG or a list of them = swag_predictive
    (M = n_samples * members); a LaplaceApproximation = laplace_predictive(link="mc").  seed None = the model's dropout
    seed for mc_dropout and 0 for the others.

    The pool is cut into batches of batch_size records, and replicate m of every batch uses the key the wrapped call
    documents (mc_dropout: dropout key (seed, step + m)).  Dropout masks are drawn per row of the batch a record sits in,
    so for mc_dropout batch_size is part of the key: the result is deterministic for a given batch_size.
    internal_batch_size is passed to the wrapped call.  Eval mode only; the model is not changed."""
    from .laplace import LaplaceApproximation, laplace_predictive
    from .swag import SWAG, swag_predictive
    from .uncertainty import mc_dropout
    n, fetch = _pool(model, pool, "pool")
    n_samples = _int(n_samples, "n_samples", 1, 0x7FFFFFFF)
    if posterior is None:
        run = lambda b, s: mc_dropout(model, *b, n_samples=n_samples, seed=s, step=step,
                                      internal_batch_size=internal_batch_size, return_samples=True)
    elif isinstance(posterior, LaplaceApproximation):
        run = lambda b, s: laplace_predictive(model, posterior, *b, link="mc", n_samples=n_samples,
                                              seed=0 if s is None else s, step=step,
                                              internal_batch_size=internal_batch_size, return_samples=True)
    elif isinstance(posterior, SWAG) or (isinstance(posterior, (list, tuple)) and posterior
                                         and all(isinstance(p, SWAG) for p in posterior)):
        run = lambda b, s: swag_predictive(model, posterior, *b, n_samples=n_samples, seed=0 if s is None else s,
                                           step=step, internal_batch_size=internal_batch_size, return_samples=True)
    else:
        raise TypeError("posterior must be None, a SWAG, a list of SWAG or a LaplaceApproximation, got %s"
                        % type(posterior).__name__)
    parts = []
    for i0, i1 in _batches(n, batch_size):
        src, static, times, lengths, _ = fetch(i0, i1)
        parts.append(run((src, static, times, lengths), seed).samples)
    return torch.cat(parts, dim=1) if len(parts) > 1 else parts[0]
