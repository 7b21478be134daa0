"""KNN-Shapley data valuation for Raindrop_v2: which training records help the model on held-out data and which hurt it,
computed on the device (Jia et al., VLDB 2019).

    res = knn_shapley(model.eval(), train, query=val, k=10)          # values [n_train]: larger = more helpful
    res = knn_shapley(model.eval(), train, k=10)                     # leave-one-out: no validation split needed
    suspects = res.values.argsort()[:50]                             # the lowest-valued records (likely mislabels)

Every record's value is its exact Shapley value under the utility of a k-nearest-neighbour classifier on the model's
features, averaged over the queries: no retraining and no sampling.  Features: the chosen layer's rows of eval forwards
(ood.features), L2-normalised by rd_ood_prepare_bank's rule; similarity = the fp64 dot of the normalised fp32 rows;
records ranked by similarity, descending, ties to the lower index.  For a query with label y_q and the N candidates at
ranks r = 1 .. N, m_r = 1[y(alpha_r) = y_q] and c_r = min(k, r) / (r k):
    s_r = m_r c_r - sum_{j = max(r, k) + 1}^{N} m_j / (j (j - 1))
and sum_r s_r = U_q(all) = (1/k) #{matches among the min(k, N) nearest}.  values[i] = (1/n_query) sum_q s_i^(q).
Leave-one-out mode (query=None): every training record is a query against the other n - 1, excluded from its own ranking
(its own value for that query is 0), and values[i] = (1/n) sum_{q != i} s_i^(q).

The device call (rd_knn_shapley) is stream-ordered and capturable in a CUDA graph, and its result is bitwise independent
of internal_batch_size.  oracle/valuation_oracle.py restates it in numpy float64.
"""
from dataclasses import dataclass

import numpy as np
import torch

from . import lib as L
from .active import _check_finite
from .influence import _check_batch_size, _check_data, _source

DEFAULT_SCRATCH_BYTES = 1 << 30
FEATURE_BLOCK = 4096        # records per ood.features call of knn_shapley


@dataclass
class KNNShapleyResult:
    """values [n_train] float64: each training record's mean Shapley value over the queries; utility [n_query] float64:
    each query's kNN utility U_q(all), with utility.mean() == values.sum() up to rounding; per_query [n_query, n_train]
    float64 or None: the per-query values (0 at a query's own record in leave-one-out mode).  Device tensors.  layer:
    the feature layer (None for knn_shapley_from_features)."""
    values: object
    utility: object
    per_query: object
    k: int
    layer: str
    leave_one_out: bool


def _k(k):
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= int(k) < (1 << 31):
        raise ValueError("k must be an integer >= 1, got %r" % (k,))
    return int(k)


def _feats(x, what):
    if not torch.is_tensor(x) or x.dim() != 2:
        raise ValueError("%s must be a tensor [n, F]" % what)
    if x.shape[0] < 1 or x.shape[1] < 1:
        raise ValueError("%s must be non-empty, got %s" % (what, tuple(x.shape)))
    return x


def _labels(y, n, what):
    if not torch.is_tensor(y) or y.dim() != 1 or y.shape[0] != n:
        raise ValueError("%s must be a tensor [%d] of labels" % (what, n))
    if y.is_floating_point() or y.is_complex() or y.dtype == torch.bool:
        raise ValueError("%s must hold integer labels, got %s" % (what, y.dtype))
    return y


def _device_rows(x, what):
    if not torch.cuda.is_available() or x.device.type != "cuda":
        raise L.RaindropB200Error("%s needs CUDA: pass tensors on a CUDA device (there is no CPU path)" % what)
    return x.detach().to(torch.float32).contiguous()


def _bank(lib, f, n, F, Fp):
    """The L2-normalised rows [round_up(n, 4), Fp] (rd_ood_prepare_bank; the error-compensation image is not used)."""
    bank = torch.zeros((n + 3) // 4 * 4, Fp, dtype=torch.float32, device=f.device)
    lo = torch.empty_like(bank)
    L.check(lib.rd_ood_prepare_bank(f.data_ptr(), n, F, Fp, bank.data_ptr(), lo.data_ptr(), L.stream_ptr(f.device)),
            "rd_ood_prepare_bank")
    return bank


def _chunk(lib, n, Fp, nq, internal_batch_size):
    """Queries per chunk: internal_batch_size, or the largest whose scratch fits in DEFAULT_SCRATCH_BYTES."""
    if internal_batch_size is not None:
        return int(min(nq, int(internal_batch_size), 0x7FFFFFFF))
    per = lib.rd_knn_shapley_scratch_bytes(n, Fp, 1)
    if per == 0:
        L.check(-2, "rd_knn_shapley_scratch_bytes")
    return int(max(1, min(nq, DEFAULT_SCRATCH_BYTES // per, 0x7FFFFFFF)))


def knn_shapley_from_features(train_feats, y_train, query_feats=None, y_query=None, k=10, per_query=False,
                              internal_batch_size=None):
    """KNNShapleyResult of the rows train_feats [n, F] with labels y_train [n] against query_feats [n_query, F] with
    labels y_query, or in leave-one-out mode (query_feats None: every training record a query against the others).
    Device tensors on one CUDA device; the rows are normalised on the device (rd_ood_prepare_bank).  k >= 1 (k > N is
    exact too).  internal_batch_size: queries per device chunk (default: the largest whose scratch fits in 1 GiB); the
    result is bitwise independent of it.  Refused with ValueError before any launch: shapes, labels, devices, k, fewer
    than 2 records in leave-one-out mode, non-finite features (one host synchronisation, skipped under CUDA-graph
    capture, where the eager call with the same inputs has checked them).  RaindropB200Error without CUDA."""
    k = _k(k)
    _check_batch_size(internal_batch_size)
    tf = _feats(train_feats, "train_feats")
    n, F = (int(s) for s in tf.shape)
    yt = _labels(y_train, n, "y_train")
    loo = query_feats is None
    if loo:
        if y_query is not None:
            raise ValueError("y_query needs query_feats (leave-one-out mode uses y_train)")
        if n < 2:
            raise ValueError("leave-one-out valuation needs at least 2 training records, got %d" % n)
        nq = n
    else:
        qf = _feats(query_feats, "query_feats")
        if qf.shape[1] != F:
            raise ValueError("query_feats has %d columns, train_feats %d" % (qf.shape[1], F))
        nq = int(qf.shape[0])
        if y_query is None:
            raise ValueError("query_feats needs its labels y_query")
        yq = _labels(y_query, nq, "y_query")
    if n >= (1 << 31):
        raise ValueError("at most 2^31 - 1 training records, got %d" % n)
    tensors = [tf, yt] + ([] if loo else [qf, yq])
    devs = {t.device for t in tensors}
    if len(devs) > 1:
        raise ValueError("the features and labels must be on one device, got %s" % sorted(map(str, devs)))
    t32 = _device_rows(tf, "knn_shapley")
    q32 = None if loo else _device_rows(qf, "knn_shapley")
    dev = t32.device
    _check_finite(t32, "train_feats")
    if q32 is not None:
        _check_finite(q32, "query_feats")
    lib = L.load()
    Fp = (F + 3) // 4 * 4
    qc = _chunk(lib, n, Fp, nq, internal_batch_size)
    nb = lib.rd_knn_shapley_scratch_bytes(n, Fp, qc)
    if nb == 0:
        L.check(-2, "rd_knn_shapley_scratch_bytes")
    i64 = dict(device=dev, dtype=torch.int64)
    f64 = dict(device=dev, dtype=torch.float64)
    with torch.cuda.device(dev):
        bank = _bank(lib, t32, n, F, Fp)
        queries = bank if loo else _bank(lib, q32, nq, F, Fp)
        ytd = yt.to(**i64).contiguous()
        yqd = ytd if loo else yq.to(**i64).contiguous()
        scratch = torch.empty((nb + 255) // 256 * 32, **f64)
        values = torch.empty(n, **f64)
        utility = torch.empty(nq, **f64)
        pq = torch.empty(nq, n, **f64) if per_query else None
        L.check(lib.rd_knn_shapley(bank.data_ptr(), n, Fp, ytd.data_ptr(), queries.data_ptr(), nq, yqd.data_ptr(), k,
                                   0 if loo else -1, qc, 0, scratch.data_ptr(), values.data_ptr(), L.ptr(pq),
                                   utility.data_ptr(), L.stream_ptr(dev)), "rd_knn_shapley")
        values /= nq
    return KNNShapleyResult(values=values, utility=utility, per_query=pq, k=k, layer=None, leave_one_out=loo)


def _features_of(model, data, what, layer, internal_batch_size):
    from .ood import features
    _check_data(model, data, what, allow_none_y=False)
    if isinstance(data, dict) and data.get("y") is None:
        raise ValueError("%s needs its labels y" % what)
    n, fetch = _source(data, what)
    if n < 1:
        raise ValueError("%s holds no records" % what)
    fs, ys = [], []
    for i0 in range(0, n, FEATURE_BLOCK):
        src, static, times, lengths, y = fetch(i0, min(n, i0 + FEATURE_BLOCK))
        f, _ = features(model, src, static, times, lengths, layer, internal_batch_size)
        fs.append(f)
        ys.append(y.to(device=f.device, dtype=torch.int64))
    return (torch.cat(fs) if len(fs) > 1 else fs[0]), (torch.cat(ys) if len(ys) > 1 else ys[0])


def knn_shapley(model, train, query=None, k=10, layer="hidden", per_query=False, internal_batch_size=None):
    """KNN-Shapley values of the training records of `train` against `query`, or in leave-one-out mode (query None),
    on the model's `layer` features ("hidden", the head's hidden activation, or "pooled", its input; ood.features).
    train / query: the forms ood_fit takes (a dict with labels y, a DeviceDataset, or (DeviceDataset, indices)); labels
    are required.  internal_batch_size: the forward chunk of ood.features and the queries per valuation chunk (default:
    the largest whose scratch fits in 1 GiB).  Eval mode only; the parameters, their .grad and the dropout counter are
    left untouched.  Returns a KNNShapleyResult of device tensors."""
    from .ood import _layer as check_layer
    check_layer(layer)
    k = _k(k)
    _check_batch_size(internal_batch_size)
    _check_data(model, train, "train", allow_none_y=False)
    if query is not None:
        _check_data(model, query, "query", allow_none_y=False)
    ft, yt = _features_of(model, train, "train", layer, internal_batch_size)
    fq, yq = (None, None) if query is None else _features_of(model, query, "query", layer, internal_batch_size)
    res = knn_shapley_from_features(ft, yt, fq, yq, k=k, per_query=per_query, internal_batch_size=internal_batch_size)
    res.layer = layer
    return res
