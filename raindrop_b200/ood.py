"""Out-of-distribution detection for Raindrop_v2: post-hoc scores on the features of a trained eval-mode model, with no
retraining, computed on the device.  Every score is oriented so that larger means more likely out of distribution.

    det = ood_fit(model.eval(), DeviceDataset(P, Pstatic, Ptime, y))      # one pass over the training set
    res = ood_scores(model, det, src, static, times, lengths, k=50)
    tau = ood_threshold(ood_scores(model, det, *val_in).mahalanobis)     # 95 % of in-distribution samples pass
    flagged = res.mahalanobis > tau

Scores (rd_raindrop_v2_ood_scores):
  msp          -max_c softmax(logits)_c (Hendrycks & Gimpel 2017)
  energy       -T logsumexp(logits / T) (Liu et al. 2020)
  mahalanobis  min_c (f - mu_c)^T Sigma^+ (f - mu_c) with the class means mu_c and the tied within-class covariance Sigma
               of the training features (Lee et al. 2018); mahalanobis_class is the argmin
  knn          the squared distance 2 - 2 s_(k) of the L2-normalised feature to its k-th nearest normalised training
               feature (Sun et al. 2022); knn_index the k neighbours
Features f: layer "hidden" (default) is relu(mlp_static.0(feat)), the penultimate activation; "pooled" is
cat(pooled, emb(static)), the head's input.  Sigma^+ is the pseudo-inverse from a float64 eigendecomposition: eigenvalues
<= 1e-6 lambda_max count as null (dead ReLU units make Sigma singular).  With W = V_r Lambda_r^-1/2 the distance is
||(f - mu) W - (mu_c - mu) W||^2, mu the mean of all training features: the device computes (f - mu) W on the tensor
cores, centring first so that the large mean stays out of the amplified near-null directions.
"""
import ctypes as C
import math
from dataclasses import dataclass

import numpy as np
import torch

from . import lib as L
from .attribution import _Call, _check_call
from .influence import _check_batch_size, _check_data, _fingerprint, _source

LAYERS = {"pooled": L.OOD_POOLED, "hidden": L.OOD_HIDDEN}
NULL_RTOL = 1e-6            # eigenvalues <= NULL_RTOL * lambda_max of the tied covariance count as null
FIT_BLOCK = 4096            # training samples per features call of ood_fit


def _layer(layer):
    if layer not in LAYERS:
        raise ValueError("layer must be one of %s, got %r" % (tuple(LAYERS), layer))
    return LAYERS[layer]


def _pad4(n):
    return (int(n) + 3) // 4 * 4


def _feature_width(plan):
    return plan.N * plan.d_ob + L.RD_D_PE + (plan.N if plan.d_static > 0 else 0)


def features(model, src, static, times, lengths, layer="hidden", internal_batch_size=None):
    """(feats [B, Df], logits [B, C]) fp32 on the model's device: the chosen layer's rows of eval forwards
    (rd_raindrop_v2_features) over chunks of internal_batch_size samples (default: the largest whose scratch fits in
    1 GiB), bitwise what the forward writes into its workspace.  The parameters, their .grad and the dropout counter
    are left untouched.  Raises ValueError for a model in training mode, RaindropB200Error without CUDA."""
    lay = _layer(layer)
    _check_call("features", model, src, static, None, internal_batch_size)
    with torch.no_grad():
        cl = _Call(model, src, static, times, lengths, None, False)
        plan, B, dev = cl.plan, src.shape[1], cl.device
        dims = plan.dims(B, False)
        spc, scratch = cl.chunk_scratch("_ood_feat_scratch", "rd_ood_features_scratch_bytes", dims, B,
                                        internal_batch_size, per_sample=True)
        f32 = dict(device=dev, dtype=torch.float32)
        feats = torch.empty(B, _feature_width(plan), **f32)
        logits = torch.empty(B, plan.n_classes, **f32)
        L.check(cl.lib.rd_raindrop_v2_features(C.byref(dims), C.byref(cl.params), cl.x.data_ptr(), L.ptr(cl.st),
                                               cl.tm.data_ptr(), cl.ln.data_ptr(), plan.node_scale.data_ptr(), lay, spc,
                                               scratch.data_ptr(), feats.data_ptr(), logits.data_ptr(),
                                               L.stream_ptr(dev)), "rd_raindrop_v2_features")
    return feats, logits


def fit_from_moments(class_sums, class_counts, gram):
    """The host half of the fit, in float64: (class means [C, F], global mean [F], W [F, r], class_proj [C, r]) from the
    moments rd_feature_moments returns.  S = gram - sum_c n_c mu_c mu_c^T, Sigma = S / n, Sigma = V Lambda V^T, W the
    columns v_j / sqrt(lambda_j) with lambda_j > NULL_RTOL * lambda_max, class_proj[c] = (mu_c - mu) W.  A class with no
    sample has NaN mean and projection (it never wins the minimum).  Raises ValueError when the features have no
    variance."""
    sums = np.asarray(class_sums, dtype=np.float64)
    counts = np.asarray(class_counts, dtype=np.int64)
    G = np.asarray(gram, dtype=np.float64)
    n = int(counts.sum())
    if n < 1:
        raise ValueError("the moments hold no samples")
    if not (np.isfinite(sums).all() and np.isfinite(G).all()):
        raise ValueError("the feature moments are not finite")
    with np.errstate(invalid="ignore", divide="ignore"):
        means = sums / counts[:, None].astype(np.float64)
    mu = sums.sum(axis=0) / n
    seen = counts > 0
    S = G - np.einsum("c,ci,cj->ij", counts[seen].astype(np.float64), means[seen], means[seen])
    Sigma = 0.5 * (S + S.T) / n
    lam, V = np.linalg.eigh(Sigma)
    if not lam.max() > 0:
        raise ValueError("the features have no within-class variance: the Mahalanobis score is undefined")
    keep = lam > NULL_RTOL * lam.max()
    W = V[:, keep] / np.sqrt(lam[keep])
    return means, mu, W, (means - mu) @ W


@dataclass
class OODDetector:
    """A fitted detector (ood_fit).  Host float64: class_means [C, F], class_counts [C], mean [F] (all training
    features), W [F, r] and class_proj [C, r].  Device: mean_dev (fp64), w_t [rp, Fp] = W^T and class_proj_dev [C, rp]
    (fp32, zero-padded to multiples of 4), and the kNN bank [round_up(n, 4), Fp] of normalised training features with
    its error-compensation remainder bank_lo (None without a bank).  fingerprint: sha256 of the weights it was fitted
    to; ood_scores refuses other weights."""
    layer: str
    n: int
    class_means: np.ndarray
    class_counts: np.ndarray
    mean: np.ndarray
    W: np.ndarray
    class_proj: np.ndarray
    mean_dev: torch.Tensor
    w_t: torch.Tensor
    class_proj_dev: torch.Tensor
    bank: object
    bank_lo: object
    n_bank: int
    fingerprint: str

    @property
    def rank(self):
        return self.W.shape[1]

    def save(self, path):
        cpu = lambda t: None if t is None else t.detach().cpu()
        torch.save(dict(layer=self.layer, n=self.n, class_means=torch.from_numpy(self.class_means),
                        class_counts=torch.from_numpy(self.class_counts), mean=torch.from_numpy(self.mean),
                        W=torch.from_numpy(self.W), class_proj=torch.from_numpy(self.class_proj), bank=cpu(self.bank),
                        bank_lo=cpu(self.bank_lo), n_bank=self.n_bank, fingerprint=self.fingerprint), path)

    @classmethod
    def load(cls, path, model=None, device=None):
        """A saved detector on `device` (default: the model's, else cuda).  With `model`, a detector fitted to other
        weights or another layer width is refused here rather than at ood_scores."""
        d = torch.load(path, map_location="cpu", weights_only=True)
        if device is None:
            device = next(model.parameters()).device if model is not None else torch.device("cuda")
        det = _detector(d["layer"], int(d["n"]), d["class_means"].numpy(), d["class_counts"].numpy(), d["mean"].numpy(),
                        d["W"].numpy(), d["class_proj"].numpy(), None, 0, str(d["fingerprint"]), device)
        if d["bank"] is not None:
            det.bank, det.bank_lo = d["bank"].to(device), d["bank_lo"].to(device)
            det.n_bank = int(d["n_bank"])
        if model is not None:
            _check_detector(model, det)
        return det


def _detector(layer, n, means, counts, mu, W, proj, bank, n_bank, fingerprint, device):
    F, r = W.shape
    C_ = proj.shape[0]
    Fp, rp = _pad4(F), _pad4(r)
    w_t = torch.zeros(rp, Fp, dtype=torch.float32)
    w_t[:r, :F] = torch.from_numpy(W.T.copy())
    pj = torch.zeros(C_, rp, dtype=torch.float32)
    pj[:, :r] = torch.from_numpy(proj)
    return OODDetector(layer=layer, n=n, class_means=means, class_counts=counts, mean=mu, W=W, class_proj=proj,
                       mean_dev=torch.from_numpy(mu).to(device), w_t=w_t.to(device), class_proj_dev=pj.to(device),
                       bank=bank, bank_lo=None, n_bank=n_bank, fingerprint=fingerprint)


def _check_detector(model, det):
    if not isinstance(det, OODDetector):
        raise TypeError("detector must be an OODDetector (ood_fit)")
    F = _feature_width(model._plan)
    if det.mean.shape != (F,) or det.class_proj.shape[0] != model._plan.n_classes:
        raise ValueError("the detector was fitted to a model of another feature width or class count")
    # hashing reads the weights back to the host: done once per state of the tensors (an in-place update bumps
    # _version), so repeated calls, and a CUDA-graph capture after an eager call, skip it
    params = model.used_parameters()
    state = tuple((p.data_ptr(), p._version) for p in params)
    if det.__dict__.get("_checked_state") == state:
        return
    fp = _fingerprint(params)
    if fp != det.fingerprint:
        raise ValueError("the detector was fitted to other weights (fingerprint %s..., the model's %s...)"
                         % (det.fingerprint[:12], fp[:12]))
    det.__dict__["_checked_state"] = state


def ood_fit(model, train, layer="hidden", knn=True, internal_batch_size=None):
    """OODDetector of the model's current weights from `train` (the forms laplace_fit takes: a dict with labels y, a
    DeviceDataset, or (DeviceDataset, indices)).  One pass: features of blocks of the training set, their moments
    accumulated on the device in float64 (rd_feature_moments, bitwise independent of the blocking), and with knn the
    normalised bank (rd_ood_prepare_bank).  The host forms the class means and the tied covariance's pseudo-inverse
    factor (fit_from_moments).  Refuses non-finite features (one host sync).  Eval mode only; the model is not
    changed."""
    lay = _layer(layer)
    _check_batch_size(internal_batch_size)
    _check_data(model, train, "ood_fit", allow_none_y=False)
    if isinstance(train, dict) and train.get("y") is None:
        raise ValueError("train needs its labels y (the class means)")
    n, fetch = _source(train, "train")
    if n < 1:
        raise ValueError("train holds no samples")
    plan = model._plan
    F, ncls = _feature_width(plan), plan.n_classes
    fp = _fingerprint(model.used_parameters())
    lib = L.load()
    with torch.no_grad():
        parts, finite, sums, counts, gram = [], [], None, None, None
        for i0 in range(0, n, FIT_BLOCK):
            src, static, times, lengths, y = fetch(i0, min(n, i0 + FIT_BLOCK))
            f, _ = features(model, src, static, times, lengths, layer, internal_batch_size)
            dev = f.device
            if sums is None:
                sums = torch.empty(ncls, F, dtype=torch.float64, device=dev)
                counts = torch.empty(ncls, dtype=torch.int64, device=dev)
                gram = torch.empty(F, F, dtype=torch.float64, device=dev)
            yd = y.to(device=dev, dtype=torch.int64).contiguous()
            L.check(lib.rd_feature_moments(f.data_ptr(), yd.data_ptr(), f.shape[0], F, ncls, int(i0 > 0),
                                           sums.data_ptr(), counts.data_ptr(), gram.data_ptr(), L.stream_ptr(dev)),
                    "rd_feature_moments")
            finite.append(torch.isfinite(f).all().reshape(1))
            if knn:
                parts.append(f)
        if not bool(torch.cat(finite).all()):
            raise ValueError("the model's %s features of the training set are not all finite" % layer)
        means, mu, W, proj = fit_from_moments(sums.cpu().numpy(), counts.cpu().numpy(), gram.cpu().numpy())
        det = _detector(layer, n, means, counts.cpu().numpy(), mu, W, proj, None, 0, fp, dev)
        if knn:
            feats = torch.cat(parts) if len(parts) > 1 else parts[0]
            Fp = _pad4(F)
            det.bank = torch.zeros(_pad4(n), Fp, dtype=torch.float32, device=dev)
            det.bank_lo = torch.zeros_like(det.bank)
            det.n_bank = n
            L.check(lib.rd_ood_prepare_bank(feats.data_ptr(), n, F, Fp, det.bank.data_ptr(), det.bank_lo.data_ptr(),
                                            L.stream_ptr(dev)), "rd_ood_prepare_bank")
    return det


@dataclass
class OODScores:
    """Per-sample scores of ood_scores (device tensors; larger = more likely out of distribution): msp [B], energy [B],
    mahalanobis [B] with mahalanobis_class [B] (int64) and the per-class distances mahalanobis_per_class [B, C], knn [B]
    with knn_index [B, k] (int64; None without a bank), logits [B, C]."""
    msp: object
    energy: object
    mahalanobis: object
    mahalanobis_class: object
    mahalanobis_per_class: object
    knn: object
    knn_index: object
    logits: object


def _check_k(k):
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= int(k) <= L.OOD_MAX_K:
        raise ValueError("k must be an integer in [1, %d], got %r" % (L.OOD_MAX_K, k))
    return int(k)


def _check_temperature(t):
    t = float(t)
    if not (math.isfinite(t) and t > 0):
        raise ValueError("temperature must be finite and > 0, got %r" % t)
    return t


def ood_scores(model, detector, src, static, times, lengths, k=50, temperature=1.0, internal_batch_size=None):
    """OODScores of a batch under `detector` (ood_fit) in one device call per batch (rd_raindrop_v2_ood_scores): per
    chunk of internal_batch_size samples (default: the largest whose scratch fits in 1 GiB) one eval forward, msp and
    energy from its logits, the Mahalanobis distances through a 3xTF32 GEMM and the k nearest bank rows through 3xTF32
    GEMMs over bank slices and a top-k selection.  Every output is bitwise independent of internal_batch_size once
    model._plan.obprop_mode is pinned.  k: 1 <= k <= min(256, bank size).  A detector fitted to other weights is
    refused.  The parameters, their .grad and the dropout counter are left untouched; the call is stream-ordered and
    can be captured in a CUDA graph (after an eager call with the same shapes)."""
    _check_call("ood_scores", model, src, static, None, internal_batch_size)
    _check_detector(model, detector)
    k = _check_k(k)
    temperature = _check_temperature(temperature)
    if detector.bank is not None and k > detector.n_bank:
        raise ValueError("k = %d exceeds the bank's %d rows" % (k, detector.n_bank))
    with torch.no_grad():
        cl = _Call(model, src, static, times, lengths, None, False)
        plan, B, dev = cl.plan, src.shape[1], cl.device
        if detector.w_t.device != dev:
            raise ValueError("the detector is on %s, the inputs on %s" % (detector.w_t.device, dev))
        has_bank = detector.bank is not None
        n_bank = detector.n_bank if has_bank else 0
        dims = plan.dims(B, False)
        spc, scratch = cl.chunk_scratch("_ood_scores_scratch", "rd_ood_scores_scratch_bytes", dims, B,
                                        internal_batch_size, detector.rank, n_bank, k, per_sample=True)
        f32 = dict(device=dev, dtype=torch.float32)
        i64 = dict(device=dev, dtype=torch.int64)
        ncls = plan.n_classes
        out = OODScores(msp=torch.empty(B, **f32), energy=torch.empty(B, **f32), mahalanobis=torch.empty(B, **f32),
                        mahalanobis_class=torch.empty(B, **i64), mahalanobis_per_class=torch.empty(B, ncls, **f32),
                        knn=torch.empty(B, **f32) if has_bank else None,
                        knn_index=torch.empty(B, k, **i64) if has_bank else None, logits=torch.empty(B, ncls, **f32))
        L.check(cl.lib.rd_raindrop_v2_ood_scores(
            C.byref(dims), C.byref(cl.params), cl.x.data_ptr(), L.ptr(cl.st), cl.tm.data_ptr(), cl.ln.data_ptr(),
            plan.node_scale.data_ptr(), LAYERS[detector.layer], detector.mean_dev.data_ptr(), detector.w_t.data_ptr(),
            detector.class_proj_dev.data_ptr(), detector.rank, L.ptr(detector.bank), L.ptr(detector.bank_lo), n_bank, k,
            temperature, spc, scratch.data_ptr(), out.logits.data_ptr(), out.msp.data_ptr(), out.energy.data_ptr(),
            out.mahalanobis.data_ptr(), out.mahalanobis_class.data_ptr(), out.mahalanobis_per_class.data_ptr(),
            L.ptr(out.knn), L.ptr(out.knn_index), L.stream_ptr(dev)), "rd_raindrop_v2_ood_scores")
    return out


def ood_scores_from_features(feats, logits, detector, k=50, temperature=1.0):
    """The float64 numpy restatement of ood_scores from given features [B, F] and logits [B, C]: the same fields as
    numpy arrays.  Mahalanobis per class as (f - mu_c)^T W W^T (f - mu_c); kNN against the detector's fp32 bank rows,
    the query normalised in float64, ties to the lower bank index."""
    f = np.asarray(torch.as_tensor(feats).detach().cpu().double())
    lg = np.asarray(torch.as_tensor(logits).detach().cpu().double())
    k, T = _check_k(k), _check_temperature(temperature)
    m = lg.max(axis=1, keepdims=True)
    msp = -1.0 / np.exp(lg - m).sum(axis=1)
    energy = -(m[:, 0] + T * np.log(np.exp((lg - m) / T).sum(axis=1)))
    diff = f[:, None, :] - detector.class_means[None, :, :]
    z = diff @ detector.W
    per = (z * z).sum(axis=2)
    per = np.where(np.isnan(per), np.inf, per)
    cls = per.argmin(axis=1)
    knn = idx = None
    if detector.bank is not None:
        if k > detector.n_bank:
            raise ValueError("k = %d exceeds the bank's %d rows" % (k, detector.n_bank))
        F = f.shape[1]
        bank = detector.bank[:detector.n_bank, :F].detach().cpu().double().numpy()
        q = f / np.maximum(np.linalg.norm(f, axis=1, keepdims=True), 1e-12)
        s = q @ bank.T
        order = np.argsort(-s, axis=1, kind="stable")        # stable: equal similarities keep index order
        idx = order[:, :k]
        knn = 2.0 - 2.0 * np.take_along_axis(s, idx[:, k - 1:k], axis=1)[:, 0]
    return OODScores(msp=msp, energy=energy, mahalanobis=per[np.arange(len(cls)), cls], mahalanobis_class=cls,
                     mahalanobis_per_class=per, knn=knn, knn_index=idx, logits=lg)


def _scores(x, what):
    a = np.asarray(torch.as_tensor(x).detach().cpu().double()).reshape(-1)
    if a.size == 0 or not np.isfinite(a).all():
        raise ValueError("%s must be non-empty and finite" % what)
    return a


def ood_threshold(score_in, tpr=0.95):
    """The threshold tau a deployment flags above: the smallest in-distribution score with at least a fraction tpr of the
    in-distribution scores <= tau (float64, host)."""
    s = np.sort(_scores(score_in, "score_in"))
    tpr = float(tpr)
    if not 0.0 < tpr <= 1.0:
        raise ValueError("tpr must lie in (0, 1], got %r" % tpr)
    need = max(1, math.ceil(tpr * s.size - 1e-9))
    return float(s[need - 1])


def _average_precision(pos, neg):
    """Average precision of ranking `pos` above `neg` (larger = positive), tied scores entering as one step."""
    s = np.concatenate([pos, neg])
    y = np.concatenate([np.ones(pos.size), np.zeros(neg.size)])
    order = np.argsort(-s, kind="stable")
    s, y = s[order], y[order]
    last = np.r_[np.nonzero(np.diff(s))[0], s.size - 1]      # the end of each group of equal scores
    tp = np.cumsum(y)[last]
    prec = tp / (last + 1.0)
    rec = tp / pos.size
    return float(np.sum(np.diff(np.r_[0.0, rec]) * prec))


def _auroc(pos, neg):
    """The probability that a `pos` score exceeds a `neg` score, ties counting 1/2 (the Mann-Whitney U statistic over
    |pos| |neg|)."""
    from scipy.stats import rankdata
    r = rankdata(np.concatenate([neg, pos]))
    u = r[neg.size:].sum() - pos.size * (pos.size + 1) / 2.0
    return float(u / (neg.size * pos.size))


def ood_metrics(score_in, score_out):
    """Detection metrics of scores on in-distribution and out-of-distribution samples (larger = OOD), float64 on the
    host: auroc (Mann-Whitney, ties count 1/2), aupr_in (in-distribution positive, ranked by -score), aupr_out (OOD
    positive) and fpr_at_95_tpr, the fraction of OOD scores <= ood_threshold(score_in, 0.95)."""
    si, so = _scores(score_in, "score_in"), _scores(score_out, "score_out")
    tau = ood_threshold(si, 0.95)
    return dict(auroc=_auroc(so, si), aupr_in=_average_precision(-si, -so),
                aupr_out=_average_precision(so, si), fpr_at_95_tpr=float(np.mean(so <= tau)))
