"""Laplace approximation of Raindrop_v2 (MacKay 1992; Ritter et al. 2018; Daxberger et al. 2021, "Laplace Redux"):
post-hoc predictive uncertainty of a trained checkpoint, with no retraining, computed on the device.

The posterior over the selected parameters is N(theta*, H^-1) with H = n F + delta I, F the EK-FAC Fisher of the
training set (influence.ekfac_factors).  In the Kronecker eigenbasis H is diagonal, n Lambda_j + delta.  The linearised
(GLM) predictive of sample b is a Gaussian over its logits, f ~ N(f(x_b; theta*), Sigma_b), with

    Sigma_b[c, c'] = sum_j J~_{b,c,j} J~_{b,c',j} / (n Lambda_j + delta)

and J~_{b,c} the gradient of logit c rotated into the eigenbasis (rd_raindrop_v2_laplace_logit_cov).  The prior
precision delta maximises the log marginal likelihood, closed-form in the same basis:

    log Z(delta) = sum_b log p(y_b | x_b, theta*) - (delta / 2) ||theta*||^2 + (P / 2) log delta
                   - 1/2 sum_j log(n Lambda_j + delta)

    la = laplace_fit(model.eval(), DeviceDataset(P, Pstatic, Ptime, y))
    res = laplace_predictive(model, la, src, static, times, lengths, link="probit")
    keep = res.predictive_entropy.argsort()[: int(0.8 * B)]      # the 80 % of samples the model is surest about

link "probit" maps (f, Sigma) to probabilities with the probit approximation, softmax(f_c / sqrt(1 + pi/8 Sigma_cc));
link "mc" draws n_samples logit vectors per sample (rd_laplace_predictive_mc) and reduces them as mc_dropout does.
"""
import ctypes as C
import math
from dataclasses import dataclass

import numpy as np
import torch

from . import lib as L
from .attribution import DEFAULT_SCRATCH_BYTES, _Call, _check_call, _largest_chunk
from .influence import (EKFACFactors, _Weights, _bucket_length, _check_batch_size, _check_data, _check_factors, _dims,
                        _offsets, _row_batch, _selected, _source, ekfac_factors, ekfac_rotate, ekfac_weights,
                        grad_layout)
from .uncertainty import _device_key

LINKS = ("probit", "mc")


def _selected_columns(layout_shapes, fields):
    """int64 numpy: the bucket columns of the selected fields (no padding)."""
    sel = _selected([(k, o, s) for (k, s), o in zip(layout_shapes, _offsets(layout_shapes))],
                    None if fields is None else list(fields))
    return np.concatenate([np.arange(o, o + math.prod(s), dtype=np.int64)
                           for (k, s), o in zip(layout_shapes, _offsets(layout_shapes)) if k in sel])


def _check_delta(delta, what="prior_precision"):
    if isinstance(delta, bool) or not isinstance(delta, (int, float, np.floating, np.integer)):
        raise ValueError("%s must be a positive float" % what)
    d = float(delta)
    if not (math.isfinite(d) and d > 0):
        raise ValueError("%s must be a finite float > 0, got %r" % (what, delta))
    return d


def log_marginal_likelihood(delta, n_lambda, theta_sqnorm, train_loglik):
    """log Z(delta) in float64 over the selected parameters; n_lambda = n Lambda_j of each of them."""
    d = _check_delta(delta, "delta")
    nl = np.asarray(n_lambda, dtype=np.float64)
    return float(train_loglik - 0.5 * d * theta_sqnorm + 0.5 * nl.size * math.log(d) - 0.5 * np.log(nl + d).sum())


def fit_prior_precision(n_lambda, theta_sqnorm):
    """The delta maximising log Z: the root of the stationarity condition delta ||theta*||^2 = gamma(delta),
    gamma = sum_j n Lambda_j / (n Lambda_j + delta) (MacKay's effective number of parameters).  In u = log delta,
    d log Z / du = (gamma - delta ||theta*||^2) / 2 decreases strictly, so the root is unique; it is found by Newton's
    method in u kept inside a bracket that bisection shrinks whenever a Newton step leaves it (float64, host)."""
    nl = np.asarray(n_lambda, dtype=np.float64)
    m = float(theta_sqnorm)
    gmax = float(np.count_nonzero(nl > 0))
    if not m > 0:
        raise ValueError("||theta*||^2 = 0 over the selected fields: log Z grows without bound in the prior precision")
    if gmax == 0:
        raise ValueError("every eigenvalue is 0 over the selected fields: log Z has no maximum in the prior precision")

    def g(u):
        d = math.exp(u)
        r = nl / (nl + d)
        return float(r.sum()) - d * m, -float((r * (1.0 - r)).sum()) - d * m

    hi = math.log(gmax / m)               # g(hi) = sum r - gmax < 0
    lo = hi - 1.0
    while g(lo)[0] <= 0:
        lo = hi - 2.0 * (hi - lo)
    u = 0.5 * (lo + hi)
    for _ in range(200):
        gu, dg = g(u)
        if gu > 0:
            lo = u
        else:
            hi = u
        if gu == 0 or hi - lo <= 4 * np.finfo(np.float64).eps * max(1.0, abs(u)):
            break
        nu = u - gu / dg
        u = nu if lo < nu < hi else 0.5 * (lo + hi)
    return math.exp(u)


@dataclass
class LaplaceApproximation:
    """A fitted Laplace approximation (laplace_fit): the EK-FAC factors of the training set, the prior precision delta,
    n training samples, P selected parameters, sum_b log p(y_b | x_b, theta*) over the training set and ||theta*||^2
    over the selected fields.  save / load keep everything; a loaded approximation is refused for other weights by the
    factors' fingerprint."""
    factors: EKFACFactors
    prior_precision: float
    n: int
    n_params: int
    train_loglik: float
    theta_sqnorm: float

    def _n_lambda(self):
        cols = _selected_columns(self.factors.layout, self.factors.fields)
        return self.n * self.factors.eigenvalues.detach().cpu().double().numpy()[cols]

    def log_marginal_likelihood(self, delta=None):
        """log Z at delta (default: the fitted prior precision)."""
        return log_marginal_likelihood(self.prior_precision if delta is None else delta, self._n_lambda(),
                                       self.theta_sqnorm, self.train_loglik)

    def save(self, path):
        torch.save(dict(factors=self.factors._state(), prior_precision=self.prior_precision, n=self.n,
                        n_params=self.n_params, train_loglik=self.train_loglik, theta_sqnorm=self.theta_sqnorm), path)

    @classmethod
    def load(cls, path, map_location=None):
        d = torch.load(path, map_location=map_location, weights_only=True)
        return cls(factors=EKFACFactors._from_state(d["factors"]), prior_precision=float(d["prior_precision"]),
                   n=int(d["n"]), n_params=int(d["n_params"]), train_loglik=float(d["train_loglik"]),
                   theta_sqnorm=float(d["theta_sqnorm"]))


@dataclass
class LaplaceResult:
    """The predictive of laplace_predictive, with the field names of uncertainty.MCDropoutResult (fp32 tensors on the
    device; None where the link does not define them):
      mean_probs [B, C]; predictive_entropy [B] = H(mean_probs) (both links);
      variance [B, C], expected_entropy [B], mutual_information [B] (link "mc"); samples [M, B, C] (mc, return_samples);
      mean_logits [B, C] = f(x_b; theta*) (fp32) and logit_cov [B, C, C] = Sigma_b (fp64) (both links)."""
    mean_probs: object
    variance: object
    predictive_entropy: object
    expected_entropy: object
    mutual_information: object
    samples: object
    mean_logits: object
    logit_cov: object


def probit_predictive(mean_logits, logit_cov):
    """(mean_probs, predictive_entropy) of the probit link in float64 torch arithmetic on the inputs' device:
    softmax(mu_c / sqrt(1 + pi/8 Sigma_cc)) and its entropy (natural log, 0 log 0 = 0)."""
    mu = torch.as_tensor(mean_logits).double()
    var = torch.as_tensor(logit_cov).double().diagonal(dim1=1, dim2=2)
    p = torch.softmax(mu / torch.sqrt(1.0 + (math.pi / 8.0) * var), dim=1)
    h = -torch.where(p > 0, p * torch.log(torch.where(p > 0, p, torch.ones_like(p))), torch.zeros_like(p)).sum(dim=1)
    return p, h


def laplace_from_grads(J, factors, prior_precision):
    """float64 numpy restatement of the logit covariance: J [B, C, bucket] plain Jacobian rows (the gradient of each
    logit), rotated with the factors' float64 bases (influence.ekfac_rotate) and contracted with
    w = 1 / (n Lambda + delta) -> Sigma [B, C, C]."""
    J = np.asarray(J, dtype=np.float64)
    d = _check_delta(prior_precision)
    w = ekfac_weights(factors, damping=d / factors.n) / factors.n
    if J.ndim != 3 or J.shape[2] != w.shape[0]:
        raise ValueError("J must be [B, C, %d], got %s" % (w.shape[0], J.shape))
    Jr = ekfac_rotate(J.reshape(-1, J.shape[2]), factors).reshape(J.shape)
    return np.einsum("bcj,j,bdj->bcd", Jr, w, Jr)


def _fields_sqnorm(model, fields):
    """(||theta||^2 in float64, P) over the selected fields."""
    sel = _selected(grad_layout(model), None if fields is None else list(fields))
    sq, P = 0.0, 0
    for (key, _), p in zip(model._plan.fields, model.used_parameters()):
        if key in sel:
            sq += float(p.detach().double().pow(2).sum())
            P += p.numel()
    return sq, P


def _forward(model, src, static, times, lengths, y=None):
    """One eval forward of a batch in the rows' arithmetic (influence._dims) -> (call, dims, workspace, logits, loss)."""
    cl = _Call(model, src, static, times, lengths, None, False)
    lib, plan, dev = cl.lib, cl.plan, cl.device
    B = cl.x.shape[1]
    dims = _dims(plan, B)
    ws = cl.scratch("_psg_workspace", (B, dims.obprop_mode, dev.index), lib.rd_workspace_bytes(C.byref(dims)))
    f32 = dict(device=dev, dtype=torch.float32)
    logits = torch.empty(B, plan.n_classes, **f32)
    loss = dlog = None
    if y is not None:
        y = y.to(device=dev, dtype=torch.int64).contiguous()
        loss, dlog = torch.empty(1, **f32), torch.empty(B, plan.n_classes, **f32)
    L.check(lib.rd_raindrop_v2_fwd(C.byref(dims), C.byref(cl.params), cl.x.data_ptr(), L.ptr(cl.st), cl.tm.data_ptr(),
                                   cl.ln.data_ptr(), plan.node_scale.data_ptr(), L.ptr(plan.rng_state), ws.data_ptr(),
                                   logits.data_ptr(), L.ptr(y), L.ptr(loss), L.ptr(dlog), L.stream_ptr(dev)),
            "rd_raindrop_v2_fwd")
    return cl, dims, ws, logits, loss


def _train_loglik(model, train):
    """sum_b log p(y_b | x_b, theta*) over `train` with its labels: -B * the fused mean loss of rd_raindrop_v2_fwd per
    batch of tracin's row batch, added in fp64 on the device (one host sync)."""
    n, fetch = _source(train, "train")
    lib = L.load()
    R = _row_batch(lib, model._plan, _bucket_length(grad_layout(model)))
    total = None
    for s0 in range(0, n, R):
        src, static, times, lengths, y = fetch(s0, min(n, s0 + R))
        _, _, _, _, loss = _forward(model, src, static, times, lengths, y)
        t = -loss.double() * src.shape[1]
        total = t if total is None else total + t
    return 0.0 if total is None else float(total.item())


def laplace_fit(model, train, fisher="true", seed=0, fields=None, prior_precision=None, internal_batch_size=None):
    """LaplaceApproximation of the model's current weights from `train` (influence.tracin's train argument, with
    labels): the EK-FAC factors (influence.ekfac_factors with fisher, seed, fields, internal_batch_size), one eval pass
    for the training log-likelihood, ||theta*||^2 over the selected fields and, with prior_precision None, the delta
    maximising the log marginal likelihood (fit_prior_precision).  fields: a subnetwork at EK-FAC block granularity
    (a linear layer's weight and bias together); parameters outside it stay at theta*.  Eval mode only; the weights,
    the mode and the dropout counter are restored."""
    if prior_precision is not None:
        prior_precision = _check_delta(prior_precision)
    _check_data(model, train, "train", allow_none_y=False)
    if isinstance(train, dict) and train.get("y") is None:
        raise ValueError("train needs its labels y (the log-likelihood term of log Z)")
    factors = ekfac_factors(model, train, fisher=fisher, seed=seed, fields=fields, internal_batch_size=internal_batch_size)
    if factors.n < 1:
        raise ValueError("train holds no samples")
    with torch.no_grad(), _Weights(model):
        ll = _train_loglik(model, train)
    sq, P = _fields_sqnorm(model, fields)
    la = LaplaceApproximation(factors=factors, prior_precision=1.0, n=factors.n, n_params=P, train_loglik=ll,
                              theta_sqnorm=sq)
    la.prior_precision = prior_precision if prior_precision is not None else fit_prior_precision(la._n_lambda(), sq)
    return la


def _cov_batch(lib, plan, cap=DEFAULT_SCRATCH_BYTES):
    """Samples per covariance call: a power of two <= 128 whose forward workspace and covariance scratch fit in `cap`
    (it depends on the model alone; at least 1)."""
    r = 128
    while r > 1 and (lib.rd_workspace_bytes(C.byref(_dims(plan, r))) +
                     lib.rd_laplace_logit_cov_scratch_bytes(C.byref(_dims(plan, r)))) > cap:
        r //= 2
    return r


def laplace_predictive(model, la, src, static, times, lengths, link="probit", n_samples=100, seed=0, step=0,
                       internal_batch_size=None, return_samples=False):
    """LaplaceResult of the batch under the linearised Laplace posterior `la` (laplace_fit).  One eval forward gives
    mu = f(x; theta*); rd_raindrop_v2_laplace_logit_cov gives Sigma_b, in calls of at most internal_batch_size samples
    (default: the largest power of two <= 128 whose buffers fit in 1 GiB), with w = 1 / (n Lambda + delta).
    link "probit": probit_predictive(mu, Sigma).  link "mc": n_samples draws f = mu + L eps per sample
    (rd_laplace_predictive_mc; replicate m at Philox key (seed, step + m), site 99), reduced as mc_dropout reduces its
    replicates, in chunks of max(1, internal_batch_size // B) replicates (default: the largest whose scratch fits in
    1 GiB); the result is bitwise the same for any chunking.  Eval mode only; the parameters, their .grad, the mode and
    the dropout counter are left as they were.  An approximation fitted to other weights is refused on the host.
    Raises RaindropB200Error without CUDA or without the built library."""
    if not isinstance(la, LaplaceApproximation):
        raise TypeError("la must be a LaplaceApproximation (laplace_fit)")
    if link not in LINKS:
        raise ValueError("link must be one of %s, got %r" % (LINKS, link))
    if isinstance(n_samples, bool) or int(n_samples) != n_samples or not 1 <= int(n_samples) <= 0x7FFFFFFF:
        raise ValueError("n_samples must be an integer in [1, 2^31), got %r" % (n_samples,))
    n_samples, seed, step = int(n_samples), int(seed), int(step)
    if not 0 <= seed < 1 << 64:
        raise ValueError("seed must be in [0, 2^64), got %d" % seed)
    if step < 0 or step + n_samples > 1 << 64:
        raise ValueError("step must be >= 0 with step + n_samples <= 2^64, got %d" % step)
    _check_batch_size(internal_batch_size)
    _check_call("laplace_predictive", model, src, static, None, internal_batch_size)
    _check_data(model, dict(src=src, static=static, times=times, lengths=lengths, y=None), "laplace_predictive",
                allow_none_y=True)
    plan = model._plan
    if plan.n_classes > L.LAPLACE_MAX_CLASSES:
        raise ValueError("laplace_predictive supports at most %d classes, the model has %d"
                         % (L.LAPLACE_MAX_CLASSES, plan.n_classes))
    _check_factors(model, la.factors)
    B, ncls = src.shape[1], plan.n_classes
    if B < 1:
        raise ValueError("the batch is empty")
    f = la.factors
    with torch.no_grad(), _Weights(model):
        cl, _, _, mu, _ = _forward(model, src, static, times, lengths)
        mu = mu.clone()
        lib, dev = cl.lib, cl.device
        st = L.stream_ptr(dev)
        w = torch.from_numpy(ekfac_weights(f, damping=la.prior_precision / la.n) / la.n).to(device=dev,
                                                                                            dtype=torch.float32)
        bases = f.bases_flat.to(device=dev, dtype=torch.float32).contiguous()
        Rc = _cov_batch(lib, plan) if internal_batch_size is None else int(internal_batch_size)
        cov = torch.empty(B, ncls, ncls, dtype=torch.float64, device=dev)
        for b0 in range(0, B, Rc):
            b1 = min(B, b0 + Rc)
            sl = slice(b0, b1)
            ccl, dims, ws, _, _ = _forward(model, src[:, sl], None if static is None else static[sl], times[:, sl],
                                           lengths[sl])
            nb = lib.rd_laplace_logit_cov_scratch_bytes(C.byref(dims))
            if nb == 0:
                L.check(-2, "rd_laplace_logit_cov_scratch_bytes")
            scratch = ccl.scratch("_laplace_cov_scratch", (b1 - b0, dims.obprop_mode, dev.index), nb)
            L.check(lib.rd_raindrop_v2_laplace_logit_cov(C.byref(dims), C.byref(ccl.params), L.ptr(ccl.st),
                                                         ccl.ln.data_ptr(), plan.node_scale.data_ptr(), ws.data_ptr(),
                                                         bases.data_ptr(), w.data_ptr(), scratch.data_ptr(),
                                                         cov[b0].data_ptr(), st), "rd_raindrop_v2_laplace_logit_cov")
        if link == "probit":
            p, h = probit_predictive(mu, cov)
            return LaplaceResult(p.float(), None, h.float(), None, None, None, mu, cov)
        if internal_batch_size is None:
            spc = _largest_chunk(lambda c: lib.rd_laplace_sample_scratch_bytes(B, ncls, c), n_samples, DEFAULT_SCRATCH_BYTES)
        else:
            spc = min(n_samples, max(1, int(internal_batch_size) // B))
        nb = lib.rd_laplace_sample_scratch_bytes(B, ncls, spc)
        if nb == 0:
            L.check(-2, "rd_laplace_sample_scratch_bytes")
        scratch = torch.empty((nb + 7) // 8, dtype=torch.float64, device=dev)
        key = _device_key(plan, seed, step, dev)
        f32 = dict(device=dev, dtype=torch.float32)
        mean, var, ent = torch.empty(B, ncls, **f32), torch.empty(B, ncls, **f32), torch.empty(3, B, **f32)
        samples = torch.empty(n_samples, B, ncls, **f32) if return_samples else None
        L.check(lib.rd_laplace_predictive_mc(mu.data_ptr(), cov.data_ptr(), B, ncls, key.data_ptr(), n_samples, spc,
                                             scratch.data_ptr(), mean.data_ptr(), var.data_ptr(), ent.data_ptr(),
                                             L.ptr(samples), st), "rd_laplace_predictive_mc")
    return LaplaceResult(mean, var, ent[0], ent[1], ent[2], samples, mu, cov)
