"""Out-of-distribution detection for Raindrop_v2 (raindrop_b200.ood: rd_raindrop_v2_features, rd_feature_moments,
rd_ood_prepare_bank, rd_raindrop_v2_ood_scores).

CPU: the exported symbols, the scratch queries, the host argument checks, ood_metrics / ood_threshold against scipy and
hand cases with ties, the host fit from given moments against np.linalg.pinv, ood_scores_from_features against a
brute-force float64 loop, and a save / load round trip with the refusal of other weights.  GPU: features bitwise
against the forward's workspace views and against the float64 encoder-head oracle, the moments against numpy float64
and bitwise across chunkings, every score against the float64 restatement on the device's own features, kNN ties and
tails, bitwise chunking and CUDA-graph replay without side effects (a bound FlatAdam included), non-finite features,
and full-size P19 cases whose bank is searched in one slice and in two.  Every GPU test pins plan.obprop_mode: the auto mode picks
the ob-prop arithmetic from the row count."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from helpers import build_dropin, normwise, to_dev, ws_view
from raindrop_b200 import lib as L
from raindrop_b200 import ood as OOD
from raindrop_b200.synth import make_batch, model_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXACT, FAST = 2, 1
CASES = {
    "tiny_b6": ("TINY", 6, {}),
    "tiny8_b5": ("TINY8", 5, {}),                       # no statics, 8 classes
    "p19_b9": ("P19", 9, {"first_time_zero": True}),    # padded rows
    "p12_b3": ("P12", 3, {}),                           # T = 215
    "pam_b2": ("PAM", 2, {}),                           # T = 600
}


def _width(cfg):
    d_ob = cfg["d_model"] // cfg["d_inp"]
    return cfg["d_inp"] * d_ob + 16 + (cfg["d_inp"] if cfg["static"] else 0)


# ---- CPU --------------------------------------------------------------------------------------------------------------
def test_symbols_exported():
    lib_path = os.path.join(ROOT, "raindrop_b200", "csrc", "librd_b200.so")
    out = subprocess.run(["nm", "-D", "--defined-only", lib_path], capture_output=True, text=True, check=True).stdout
    names = {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert {"rd_ood_features_scratch_bytes", "rd_raindrop_v2_features", "rd_feature_moments", "rd_ood_prepare_bank",
            "rd_ood_scores_scratch_bytes", "rd_raindrop_v2_ood_scores"} <= names


def test_scratch_queries():
    cfg = model_config("P19", dropout=0.2)
    model = build_dropin(cfg, 1, device="cpu")
    lib = L.load()
    dims = model._plan.dims(128, False)
    f1, f8 = lib.rd_ood_features_scratch_bytes(C.byref(dims), 1), lib.rd_ood_features_scratch_bytes(C.byref(dims), 8)
    assert 0 < f1 < f8
    assert lib.rd_ood_features_scratch_bytes(C.byref(dims), 0) == 0
    q = lambda *a: lib.rd_ood_scores_scratch_bytes(C.byref(dims), *a)
    base = q(0, 0, 0, 8)
    assert 0 < base < q(100, 0, 0, 8) < q(100, 1000, 50, 8)
    F = _width(cfg)
    for bad in [(0, 0, 0, 0), (-1, 0, 0, 8), (F + 1, 0, 0, 8), (10, 1000, 0, 8), (10, 1000, 257, 8), (10, 40, 41, 8),
                (10, -1, 5, 8), (10, 1 << 31, 5, 8)]:
        assert q(*bad) == 0, bad
    assert q(10, 256, 256, 8) > 0 and q(10, 5, 5, 8) > 0


def _cpu_model(name="TINY", B=4):
    cfg = model_config(name, dropout=0.2)
    return build_dropin(cfg, 3, device="cpu").eval(), make_batch(cfg, B, seed=1), cfg


def _fake_detector(cfg, n=40, knn=True, seed=0):
    """A detector fitted on the host to random features (no device)."""
    rng = np.random.default_rng(seed)
    F, Cn = _width(cfg), cfg["n_classes"]
    f = np.maximum(rng.standard_normal((n, F)), 0).astype(np.float32)
    f[:, 3] = 0                                             # a dead unit: Sigma is singular
    y = np.arange(n) % Cn
    sums = np.stack([f[y == c].astype(np.float64).sum(0) for c in range(Cn)])
    counts = np.bincount(y, minlength=Cn).astype(np.int64)
    gram = f.astype(np.float64).T @ f.astype(np.float64)
    means, mu, W, proj = OOD.fit_from_moments(sums, counts, gram)
    det = OOD._detector("hidden", n, means, counts, mu, W, proj, None, 0, "0" * 64, "cpu")
    if knn:
        q = f.astype(np.float64) / np.maximum(np.linalg.norm(f.astype(np.float64), axis=1, keepdims=True), 1e-12)
        bank = torch.zeros(OOD._pad4(n), OOD._pad4(F))
        bank[:n, :F] = torch.from_numpy(q.astype(np.float32))
        det.bank, det.bank_lo, det.n_bank = bank, torch.zeros_like(bank), n
    return det, f, y


def test_argument_validation():
    model, b, cfg = _cpu_model()
    args = (b["src"], b["static"], b["times"], b["lengths"])
    det, _, _ = _fake_detector(cfg, n=10)
    with pytest.raises(ValueError, match="layer"):
        OOD.features(model, *args, layer="logits")
    with pytest.raises(ValueError, match="eval"):
        OOD.features(model.train(), *args)
    with pytest.raises(ValueError, match="eval"):
        OOD.ood_scores(model, det, *args)
    model.eval()
    with pytest.raises(ValueError, match="internal_batch_size"):
        OOD.features(model, *args, internal_batch_size=0)
    for k in (0, 257, 1.5, True):
        with pytest.raises(ValueError, match="k must"):
            OOD._check_k(k)
    for t in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="temperature"):
            OOD._check_temperature(t)
    with pytest.raises(TypeError):
        OOD.ood_scores(model, object(), *args)
    with pytest.raises(ValueError, match="other weights"):
        OOD.ood_scores(model, det, *args)               # the fake detector's fingerprint is not the model's
    train = dict(src=b["src"], static=b["static"], times=b["times"], lengths=b["lengths"], y=None)
    with pytest.raises(ValueError, match="label"):
        OOD.ood_fit(model, train)
    with pytest.raises(ValueError, match="layer"):
        OOD.ood_fit(model, dict(train, y=b["y"]), layer="x")
    with pytest.raises(ValueError, match="eval"):
        OOD.ood_fit(model.train(), dict(train, y=b["y"]))
    model.eval()
    with pytest.raises(ValueError, match="k = 11 exceeds"):
        OOD.ood_scores_from_features(np.zeros((2, _width(cfg))), np.zeros((2, cfg["n_classes"])), det, k=11)


def test_no_cuda_raises():
    model, b, _ = _cpu_model()
    with pytest.raises(L.RaindropB200Error):
        OOD.features(model, b["src"], b["static"], b["times"], b["lengths"])


def test_non_finite_and_degenerate_moments_refused():
    lib = L.load()
    with pytest.raises(ValueError, match="not finite"):
        OOD.fit_from_moments(np.full((2, 3), np.nan), np.array([2, 2]), np.eye(3))
    with pytest.raises(ValueError, match="no within-class variance"):
        OOD.fit_from_moments(np.zeros((2, 3)), np.array([2, 2]), np.zeros((3, 3)))
    # the device bank refuses bad shapes before touching memory
    assert lib.rd_ood_prepare_bank(0, 4, 3, 4, 0, 0, 0) != 0
    assert lib.rd_ood_prepare_bank(16, 4, 3, 2, 16, 16, 0) != 0
    assert lib.rd_ood_prepare_bank(16, 0, 3, 4, 16, 16, 0) != 0


def test_threshold_and_metrics_against_scipy():
    from scipy.stats import mannwhitneyu
    rng = np.random.default_rng(4)
    for trial in range(20):
        si = rng.integers(0, 8, size=rng.integers(1, 40)).astype(np.float64)       # many ties
        so = rng.integers(2, 10, size=rng.integers(1, 40)).astype(np.float64)
        m = OOD.ood_metrics(si, so)
        u = mannwhitneyu(so, si, alternative="two-sided").statistic
        assert abs(m["auroc"] - u / (si.size * so.size)) < 1e-12
        tau = np.sort(si)[int(np.ceil(0.95 * si.size)) - 1]
        assert OOD.ood_threshold(si) == tau
        assert m["fpr_at_95_tpr"] == np.mean(so <= tau)
        # brute-force AUPR: average precision over distinct thresholds
        for pos, neg, key in ((so, si, "aupr_out"), (-si, -so, "aupr_in")):
            ap, prev = 0.0, 0.0
            for t in np.unique(np.concatenate([pos, neg]))[::-1]:
                tp, fp = (pos >= t).sum(), (neg >= t).sum()
                rec = tp / pos.size
                ap += (rec - prev) * tp / (tp + fp)
                prev = rec
            assert abs(m[key] - ap) < 1e-12, (trial, key)


def test_metrics_hand_cases():
    m = OOD.ood_metrics([0, 1], [2, 3])
    assert m == dict(auroc=1.0, aupr_in=1.0, aupr_out=1.0, fpr_at_95_tpr=0.0)
    m = OOD.ood_metrics([1, 1], [1, 1])
    assert m["auroc"] == 0.5 and m["fpr_at_95_tpr"] == 1.0 and m["aupr_out"] == 0.5
    m = OOD.ood_metrics([0, 2], [1])
    assert m["auroc"] == 0.5
    # 20 ID scores: tau is the 19th smallest; ties at tau count as accepted
    si = np.arange(20, dtype=np.float64)
    assert OOD.ood_threshold(si) == 18.0 and OOD.ood_threshold(si, 1.0) == 19.0
    assert OOD.ood_threshold([5, 5, 5, 1]) == 5.0
    assert OOD.ood_metrics(si, [18.0, 18.5, 17.0])["fpr_at_95_tpr"] == 2 / 3
    with pytest.raises(ValueError):
        OOD.ood_threshold([1.0, float("nan")])
    with pytest.raises(ValueError):
        OOD.ood_threshold([1.0], 0.0)


def test_fit_from_moments_against_pinv():
    cfg = model_config("TINY", dropout=0.2)
    det, f, y = _fake_detector(cfg, n=60)
    f64 = f.astype(np.float64)
    Cn = cfg["n_classes"]
    mu_c = np.stack([f64[y == c].mean(0) for c in range(Cn)])
    R = f64 - mu_c[y]
    Sigma = R.T @ R / len(f64)
    P = np.linalg.pinv(Sigma, rcond=1e-6, hermitian=True)
    assert np.allclose(det.class_means, mu_c, rtol=1e-12, atol=1e-12)
    assert np.allclose(det.mean, f64.mean(0), rtol=1e-12, atol=1e-12)
    WW = det.W @ det.W.T
    assert np.abs(WW - P).max() <= 1e-8 * np.abs(P).max()
    assert det.rank == np.linalg.matrix_rank(Sigma, tol=1e-6 * np.linalg.eigvalsh(Sigma).max())


def test_scores_from_features_brute_force():
    cfg = model_config("TINY", dropout=0.2)
    det, f, y = _fake_detector(cfg, n=30)
    rng = np.random.default_rng(8)
    q = np.maximum(rng.standard_normal((5, f.shape[1])), 0)
    q[1] = f[7]                                              # a query equal to a bank row
    lg = rng.standard_normal((5, cfg["n_classes"])) * 3
    k, T = 4, 1.7
    res = OOD.ood_scores_from_features(q, lg, det, k=k, temperature=T)
    P = det.W @ det.W.T
    bank = det.bank[:det.n_bank, :f.shape[1]].double().numpy()
    for b in range(5):
        p = np.exp(lg[b] - lg[b].max())
        p /= p.sum()
        assert abs(res.msp[b] + p.max()) < 1e-12
        assert abs(res.energy[b] + T * np.log(np.sum(np.exp(lg[b] / T)))) < 1e-10
        d = [(q[b] - det.class_means[c]) @ P @ (q[b] - det.class_means[c]) for c in range(cfg["n_classes"])]
        assert np.allclose(res.mahalanobis_per_class[b], d, rtol=1e-9, atol=1e-9)
        assert res.mahalanobis_class[b] == int(np.argmin(d))
        qn = q[b] / max(np.linalg.norm(q[b]), 1e-12)
        sims = [(float(qn @ bank[i]), i) for i in range(det.n_bank)]
        top = sorted(sims, key=lambda t: (-t[0], t[1]))[:k]
        assert res.knn_index[b].tolist() == [i for _, i in top]
        assert abs(res.knn[b] - (2 - 2 * top[-1][0])) < 1e-12
    assert res.knn_index[1, 0] == 7 and res.knn[1] >= 0


def test_save_load_round_trip(tmp_path):
    model, b, cfg = _cpu_model()
    det, _, _ = _fake_detector(cfg, n=12)
    det.fingerprint = OOD._fingerprint(model.used_parameters())
    p = str(tmp_path / "det.pt")
    det.save(p)
    got = OOD.OODDetector.load(p, model=model, device="cpu")
    for name in ("class_means", "class_counts", "mean", "W", "class_proj"):
        assert np.array_equal(getattr(got, name), getattr(det, name)), name
    assert torch.equal(got.bank, det.bank) and torch.equal(got.w_t, det.w_t) and got.n_bank == det.n_bank
    assert got.layer == det.layer and got.fingerprint == det.fingerprint
    other = build_dropin(cfg, 4, device="cpu").eval()
    with pytest.raises(ValueError, match="other weights"):
        OOD.OODDetector.load(p, model=other, device="cpu")
    wider = build_dropin(model_config("TINY8", dropout=0.2), 3, device="cpu").eval()
    with pytest.raises(ValueError, match="feature width"):
        OOD.OODDetector.load(p, model=wider, device="cpu")


# ---- GPU --------------------------------------------------------------------------------------------------------------
def _setup(name, mode=EXACT, wseed=9, dseed=3, B=None):
    cfg_name, B0, opts = CASES[name]
    cfg = model_config(cfg_name, dropout=0.2)
    d = to_dev(make_batch(cfg, B or B0, seed=dseed, **opts))
    model = build_dropin(cfg, wseed).eval()
    model._plan.obprop_mode = mode
    return cfg, d, model


def _args(d):
    return d["src"], d["static"], d["times"], d["lengths"]


def _train(cfg, n, seed=11, opts=None):
    t = to_dev(make_batch(cfg, n, seed=seed, **(opts or {})))
    t["y"] = torch.arange(n, device=t["src"].device) % cfg["n_classes"]
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_features_are_the_forward_workspace(name):
    cfg, d, model = _setup(name)
    plan = model._prepare(torch.device("cuda"))
    plan.debug_keep_workspace = True
    logits, _, _ = model(*_args(d))
    ws, dims = plan.last_workspace, plan.last_dims
    for layer, which in (("pooled", L.WS_FEAT), ("hidden", L.WS_HEAD_HIDDEN)):
        f, lg = OOD.features(model, *_args(d), layer=layer)
        want = ws_view(dims, ws, which).reshape(f.shape)
        assert torch.equal(f, want), layer
        assert torch.equal(lg, logits.detach()), layer
    plan.debug_keep_workspace = False


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_moments_against_numpy_and_bitwise_across_splits(name):
    cfg, _, model = _setup(name)
    n = 37
    t = _train(cfg, n)
    f, _ = OOD.features(model, t["src"], t["static"], t["times"], t["lengths"])
    lib, dev = L.load(), f.device
    F, Cn = f.shape[1], cfg["n_classes"]
    f = f.contiguous()

    def run(splits):
        s = torch.full((Cn, F), 7.0, dtype=torch.float64, device=dev)
        c = torch.full((Cn,), 5, dtype=torch.int64, device=dev)
        g = torch.full((F, F), 3.0, dtype=torch.float64, device=dev)
        for i, (a, b) in enumerate(zip(splits[:-1], splits[1:])):
            L.check(lib.rd_feature_moments(f[a].data_ptr(), t["y"][a].data_ptr(), b - a, F, Cn, int(i > 0), s.data_ptr(),
                                           c.data_ptr(), g.data_ptr(), L.stream_ptr(dev)), "rd_feature_moments")
        return s, c, g
    s, c, g = run([0, n])
    fn, y = f.double().cpu().numpy(), t["y"].cpu().numpy()
    assert c.cpu().tolist() == np.bincount(y, minlength=Cn).tolist()
    want_s = np.stack([fn[y == k].sum(0) for k in range(Cn)])
    want_g = fn.T @ fn
    assert np.abs(s.cpu().numpy() - want_s).max() <= 1e-12 * max(1.0, np.abs(want_s).max())
    assert np.abs(g.cpu().numpy() - want_g).max() <= 1e-12 * max(1.0, np.abs(want_g).max())
    for splits in ([0, 1, n], [0, 5, 6, 30, n], [0, n], list(range(n + 1))):
        s2, c2, g2 = run(splits)
        assert torch.equal(s2, s) and torch.equal(c2, c) and torch.equal(g2, g), splits


def _fit(model, cfg, n=48, layer="hidden", knn=True, ib=None):
    return OOD.ood_fit(model, _train(cfg, n), layer=layer, knn=knn, internal_batch_size=ib)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("layer", ["hidden", "pooled"])
def test_scores_against_float64_restatement(name, layer):
    cfg, d, model = _setup(name)
    det = _fit(model, cfg, layer=layer)
    k = 5
    res = OOD.ood_scores(model, det, *_args(d), k=k, temperature=1.3)
    f, lg = OOD.features(model, *_args(d), layer=layer)
    assert torch.equal(lg, res.logits)
    ref = OOD.ood_scores_from_features(f, lg, det, k=k, temperature=1.3)
    assert np.abs(res.msp.cpu().numpy() - ref.msp).max() <= 1e-6
    assert np.abs(res.energy.cpu().numpy() - ref.energy).max() <= 1e-6 * max(1.0, np.abs(ref.energy).max())
    per, dref = res.mahalanobis_per_class.double().cpu().numpy(), ref.mahalanobis_per_class
    ok = np.isfinite(dref)
    assert (np.abs(per - dref)[ok] <= 1e-4 * (dref[ok] + 1)).all(), np.max(np.abs(per - dref)[ok] / (dref[ok] + 1))
    assert np.allclose(res.mahalanobis.cpu().numpy(), per.min(1), rtol=0, atol=0)
    assert np.array_equal(res.mahalanobis_class.cpu().numpy(), per.argmin(1))
    _check_knn(res, f, det, k)


def _check_knn(res, f, det, k):
    """knn within 4e-6 of float64, and knn_index equal to the float64 neighbours wherever the float64 gaps on both sides
    of a position exceed 1e-6."""
    q = f.double().cpu().numpy()
    q = q / np.maximum(np.linalg.norm(q, axis=1, keepdims=True), 1e-12)
    sims = q @ det.bank[:det.n_bank, :q.shape[1]].double().cpu().numpy().T
    order = np.lexsort((np.broadcast_to(np.arange(sims.shape[1]), sims.shape), -sims), axis=1)
    srt = np.take_along_axis(sims, order, 1)
    assert np.abs(res.knn.double().cpu().numpy() - (2 - 2 * srt[:, k - 1])).max() <= 4e-6
    got = res.knn_index.cpu().numpy()
    assert got.shape == (sims.shape[0], k)
    gap = np.full(srt.shape, np.inf)
    gap[:, 1:] = srt[:, :-1] - srt[:, 1:]
    clear = np.minimum(gap, np.r_['1', gap[:, 1:], np.full((srt.shape[0], 1), np.inf)])[:, :k] > 1e-6
    assert np.array_equal(got[clear], order[:, :k][clear])


@pytest.mark.gpu
def test_knn_ties_tails_and_exact_match():
    cfg, d, model = _setup("p19_b9")
    t = _train(cfg, 45)
    # duplicate bank rows: samples 3 and 40 identical, and the queries are training samples
    for key in ("src", "times"):
        t[key][:, 40] = t[key][:, 3]
    t["static"][40] = t["static"][3]
    t["lengths"][40] = t["lengths"][3]
    det = OOD.ood_fit(model, t)
    q = {k: (v[:, [3, 7, 40]] if k in ("src", "times") else v[[3, 7, 40]]) for k, v in t.items() if k != "y"}
    args = (q["src"], q["static"], q["times"], q["lengths"])
    f, lg = OOD.features(model, *args)
    for k in (1, 2, 45):
        res = OOD.ood_scores(model, det, *args, k=k)
        ref = OOD.ood_scores_from_features(f, lg, det, k=k)
        assert np.abs(res.knn.double().cpu().numpy() - ref.knn).max() <= 4e-6
        idx = res.knn_index.cpu().numpy()
        if k >= 2:
            assert idx[0, :2].tolist() == [3, 40] and idx[2, :2].tolist() == [3, 40]
        else:
            assert idx[0, 0] == 3 and idx[2, 0] == 3
            assert res.knn.cpu().max() <= 4e-6
        assert sorted(idx[1].tolist()) == sorted(set(idx[1].tolist()))          # distinct neighbours
        if k == 45:
            assert sorted(idx[0].tolist()) == list(range(45))                     # n_bank == k: every row once
    with pytest.raises(ValueError, match="exceeds"):
        OOD.ood_scores(model, det, *args, k=46)


@pytest.mark.gpu
def test_knn_large_k_and_bank_tail():
    cfg, d, model = _setup("tiny_b6")
    det = _fit(model, cfg, n=301)                            # not a multiple of 4 nor of a tile
    for k in (1, 256):
        res = OOD.ood_scores(model, det, *_args(d), k=k)
        f, lg = OOD.features(model, *_args(d))
        _check_knn(res, f, det, k)
        s = f.double().cpu().numpy()
        s = s / np.maximum(np.linalg.norm(s, axis=1, keepdims=True), 1e-12)
        sims = s @ det.bank[:det.n_bank, :s.shape[1]].double().cpu().numpy().T
        got = res.knn_index.cpu().numpy()
        # the returned neighbours' similarities are the k largest, in order, to within the 3xTF32 error
        srt = -np.sort(-sims, axis=1)[:, :k]
        assert np.abs(np.take_along_axis(sims, got, 1) - srt).max() <= 2e-6
    # B = 1
    one = {k: (v[:, :1] if k in ("src", "times") else (None if v is None else v[:1])) for k, v in d.items()}
    r1 = OOD.ood_scores(model, det, one["src"], one["static"], one["times"], one["lengths"], k=3)
    rb = OOD.ood_scores(model, det, *_args(d), k=3, internal_batch_size=1)
    assert torch.equal(r1.knn, rb.knn[:1]) and torch.equal(r1.mahalanobis, rb.mahalanobis[:1])


def _fields(res):
    return [getattr(res, f) for f in ("msp", "energy", "mahalanobis", "mahalanobis_class", "mahalanobis_per_class", "knn",
                                      "knn_index", "logits")]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_chunking_graph_and_no_side_effects(name):
    cfg, d, model = _setup(name, FAST, B=9)
    det = _fit(model, cfg, n=50, ib=7)
    plan = model._prepare(torch.device("cuda"))
    snap = {"rng": plan.rng_state.clone()}
    snap.update({"param." + k: p.detach().clone() for k, p in model.named_parameters()})
    B = d["src"].shape[1]
    res = [OOD.ood_scores(model, det, *_args(d), k=6, internal_batch_size=ib) for ib in (1, 7, B, None)]
    for r in res[1:]:
        for a, b in zip(_fields(r), _fields(res[0])):
            assert torch.equal(a, b)
    det2 = _fit(model, cfg, n=50, ib=1)
    assert torch.equal(det2.bank, det.bank) and np.array_equal(det2.W, det.W)
    kw = dict(k=6, internal_batch_size=4)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        OOD.ood_scores(model, det, *_args(d), **kw)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = OOD.ood_scores(model, det, *_args(d), **kw)
    OOD.ood_scores(model, det, *_args(d), k=2, internal_batch_size=B)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        for a, b in zip(_fields(out), _fields(res[0])):
            assert torch.equal(a, b)
    assert torch.equal(plan.rng_state, snap["rng"])
    for k, p in model.named_parameters():
        assert torch.equal(p.detach(), snap["param." + k]) and p.grad is None, k


@pytest.mark.gpu
@pytest.mark.parametrize("n_bank", [8192, 8190])
def test_full_size_p19_and_bank_slices(n_bank):
    """P19 synthetic weights, B = 3880.  The default chunk (about 1,200 samples) holds the bank in one similarity slice;
    internal_batch_size = 3880 splits it into two (slices of 4,324 columns, the second a partial tail; with 8,190 rows
    also a tail that is not a multiple of 4).  Both must give the float64 neighbours and the same bits."""
    cfg, _, model = _setup("p19_b9", FAST, B=3880)
    d = to_dev(make_batch(cfg, 3880, seed=5))
    det = _fit(model, cfg, n=n_bank)
    lib = L.load()
    dims = model._plan.dims(3880, False)
    one = lib.rd_ood_scores_scratch_bytes(C.byref(dims), det.rank, n_bank, 50, 1000)
    two = lib.rd_ood_scores_scratch_bytes(C.byref(dims), det.rank, n_bank, 50, 3880)
    assert one > 0 and two > 0
    res = OOD.ood_scores(model, det, *_args(d), k=50, internal_batch_size=1000)
    sliced = OOD.ood_scores(model, det, *_args(d), k=50, internal_batch_size=3880)
    for a, b in zip(_fields(sliced), _fields(res)):
        assert torch.equal(a, b)
    f, lg = OOD.features(model, *_args(d))
    ref = OOD.ood_scores_from_features(f, lg, det, k=50)
    for r in (res, sliced):
        _check_knn(r, f, det, 50)
    dref = ref.mahalanobis_per_class
    per = res.mahalanobis_per_class.double().cpu().numpy()
    assert (np.abs(per - dref) <= 1e-4 * (dref + 1)).all(), np.max(np.abs(per - dref) / (dref + 1))
    assert np.abs(res.msp.cpu().numpy() - ref.msp).max() <= 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_features_against_float64_oracle(name):
    """The pooled features and relu(head_pre) of encoder_head_oracle in float64, run on the forward's own encoder input
    (RD_WS_ENC_IN) with the model's weights, at the encoder-head eval tolerance (normwise 1e-5)."""
    from oracle.raindrop_oracle import encoder_head_oracle
    cfg, d, model = _setup(name)
    plan = model._prepare(torch.device("cuda"))
    plan.debug_keep_workspace = True
    model(*_args(d))
    ws, dims = plan.last_workspace, plan.last_dims
    plan.debug_keep_workspace = False
    T, B = d["src"].shape[0], d["src"].shape[1]
    z0 = ws_view(dims, ws, L.WS_ENC_IN).reshape(T, B, -1).double().cpu()
    params = {k: v.detach().double().cpu() for k, v in model.state_dict().items()}
    static = None if d["static"] is None else d["static"].double().cpu()
    lengths = d["lengths"].cpu()
    stages = {}
    encoder_head_oracle(z0, static, lengths, params, cfg["nhead"], 1e-5, stages=stages)
    pad = torch.arange(T)[None, :] >= lengths[:, None]
    pooled = (stages["enc"] * (~pad).T[:, :, None].double()).sum(0) / (lengths[:, None].double() + 1)
    if static is not None:
        pooled = torch.cat([pooled, torch.nn.functional.linear(static, params["emb.weight"], params["emb.bias"])], 1)
    for layer, want in (("pooled", pooled), ("hidden", torch.relu(stages["head_pre"]))):
        f, _ = OOD.features(model, *_args(d), layer=layer)
        assert normwise(f, want) < 1e-5, (layer, normwise(f, want))


@pytest.mark.gpu
def test_non_finite_features():
    """A NaN static makes the pooled features NaN.  ood_fit refuses such a training set; ood_scores returns defined
    outputs for such a query (NaN scores, the lowest bank indices as neighbours), the same bits for any chunking, and
    leaves the other rows as they are."""
    cfg, d, model = _setup("tiny_b6", EXACT)
    bad = _train(cfg, 20)
    bad["static"][4, 0] = float("nan")
    with pytest.raises(ValueError, match="not all finite"):
        OOD.ood_fit(model, bad, layer="pooled")
    det = _fit(model, cfg, n=40, layer="pooled")
    clean = OOD.ood_scores(model, det, *_args(d), k=5)
    d["static"][0, 0] = float("nan")
    res = [OOD.ood_scores(model, det, *_args(d), k=5, internal_batch_size=ib) for ib in (1, 4, None)]
    for r in res[1:]:
        for a, b in zip(_fields(r), _fields(res[0])):
            assert torch.equal(a, b) or (a.is_floating_point() and torch.equal(a.isnan(), b.isnan()) and
                                         torch.equal(a.nan_to_num(), b.nan_to_num()))
    r = res[0]
    assert torch.isnan(r.knn[0]) and torch.isnan(r.mahalanobis[0]) and int(r.mahalanobis_class[0]) == 0
    assert r.knn_index[0].tolist() == list(range(5))
    for a, b in zip(_fields(r), _fields(clean)):
        assert torch.equal(a[1:], b[1:])


@pytest.mark.gpu
def test_bound_flat_adam_untouched():
    """ood_fit and ood_scores leave a bound FlatAdam (flat parameters and gradients, moments, step count) as it was."""
    import torch.nn.functional as F
    from raindrop_b200.optim import FlatAdam
    cfg = model_config("TINY", dropout=0.2)
    model = build_dropin(cfg, 8).train()
    opt = FlatAdam(model, lr=1e-3)
    d = to_dev(make_batch(cfg, 6, seed=60))
    for _ in range(2):
        logits, _, _ = model.forward(*_args(d))
        F.cross_entropy(logits, d["y"]).backward()
        opt.step()
    model.eval()
    model._plan.obprop_mode = EXACT
    snap = {"flat_p": opt.flat_p.detach(), "flat_g": opt.flat_g, "exp_avg": opt.exp_avg, "exp_avg_sq": opt.exp_avg_sq,
            "step": opt.step_count, "rng": model._plan.rng_state}
    snap.update({"param." + k: p.detach() for k, p in model.named_parameters()})
    before = {k: v.clone() for k, v in snap.items()}
    det = _fit(model, cfg, n=30)
    OOD.ood_scores(model, det, *_args(d), k=3)
    torch.cuda.synchronize()
    for k, v in snap.items():
        assert torch.equal(v, before[k]), k
