"""Faithfulness of attributions by removal (raindrop_b200.faithfulness; rd_raindrop_v2_removal_curves,
rd_raindrop_v2_removal_infidelity, rd_debug_removal_inputs): the ranking against a numpy lexsort, the keep tables and
expanded rows against torch-built removed copies, the curve logits against the module's forward, the infidelity
moments against a float64 restatement, the host formulas against hand cases, determinism and side effects."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest
import torch

from helpers import build_dropin, to_dev
from oracle.dropout_masks import dropout_words_at
from raindrop_b200 import attribution as A
from raindrop_b200 import faithfulness as F
from raindrop_b200 import lib as L
from raindrop_b200.synth import make_batch, model_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SITE = 107


# ---- numpy restatements ---------------------------------------------------------------------------------------------
def _np_rank(phi, order):
    """rank [B, P]: lexsort by (order key, index); NaN after every number, -0 == +0 (numpy compares them equal)."""
    phi = np.asarray(phi, dtype=np.float32)
    key = {"descending": -phi, "ascending": phi, "absolute": -np.abs(phi)}[order]
    rank = np.empty(phi.shape, dtype=np.int32)
    for b in range(phi.shape[0]):
        k = key[b].astype(np.float64)
        pos = np.lexsort((np.arange(phi.shape[1]), np.where(np.isnan(k), 0.0, k), np.isnan(k)))
        rank[b, pos] = np.arange(phi.shape[1])
    return rank


def _np_sample_keep(seed, step, m0, nc, B, P, p_remove):
    """keep [nc*B, P] of replicates m0 .. m0+nc-1: removed iff the site-107 word b*P + g at (seed, step + m) is below
    floor(p_remove 2^32)."""
    below = int(np.floor(p_remove * 2.0 ** 32))
    idx = np.arange(B * P, dtype=np.uint64)
    rows = [(dropout_words_at(seed, step + m, SITE, idx).astype(np.int64) >= below).reshape(B, P)
            for m in range(m0, m0 + nc)]
    return np.concatenate(rows).astype(np.uint8)


def _np_curve_keep(rank, counts, q0, nc):
    K = len(counts)
    rows = []
    for q in range(q0, q0 + nc):
        top = rank < counts[q % K]
        rows.append(top if q >= K else ~top)
    return np.concatenate(rows).astype(np.uint8)


def _removed_rows(d, cells, keep, x0=None, st0=None):
    """Torch-built inputs of keep [R*B, P] rows (row j = r*B + b): cells [T, B, N] player ids (-1 / >= G: no player)."""
    src, st = d["src"], d["static"]
    T, B, N2 = src.shape
    N, P = N2 // 2, keep.shape[1]
    G = P - (1 if st is not None else 0)
    R = keep.shape[0] // B
    cells = torch.as_tensor(cells, device=src.device).long().expand(T, B, N)
    ids = torch.where((cells < 0) | (cells >= G), G, cells)                       # G: the always-kept column
    kk = torch.as_tensor(keep, device=src.device).bool().view(R, B, P)
    k = torch.cat([kk[:, :, :G], torch.ones(R, B, 1, dtype=torch.bool, device=src.device)], dim=2)
    kept = torch.gather(k.unsqueeze(1).expand(R, T, B, G + 1), 3, ids.unsqueeze(0).expand(R, T, B, N))
    base = torch.zeros_like(src) if x0 is None else x0
    val = torch.where(kept, src[None, :, :, :N], base[None, :, :, :N])              # [R, T, B, N]
    rows = torch.cat([val, src[None, :, :, N:].expand(R, T, B, N)], dim=3).permute(1, 0, 2, 3).reshape(T, R * B, N2)
    sts = None
    if st is not None:
        b0 = torch.zeros_like(st) if st0 is None else st0
        sts = torch.where(kk[:, :, P - 1:], st[None], b0[None]).reshape(R * B, -1)
    return rows.contiguous(), sts, d["times"].repeat(1, R), d["lengths"].repeat(R)


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_symbols_exported():
    lib_path = os.path.join(ROOT, "raindrop_b200", "csrc", "librd_b200.so")
    out = subprocess.run(["nm", "-D", "--defined-only", lib_path], capture_output=True, text=True, check=True).stdout
    names = {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert {"rd_removal_curves_scratch_bytes", "rd_raindrop_v2_removal_curves", "rd_removal_infidelity_scratch_bytes",
            "rd_raindrop_v2_removal_infidelity", "rd_debug_removal_inputs"} <= names


def test_scratch_queries():
    model = build_dropin(model_config("P19", dropout=0.2), 1, device="cpu")
    lib = L.load()
    dims = model._plan.dims(128, False)
    for q in (lib.rd_removal_curves_scratch_bytes, lib.rd_removal_infidelity_scratch_bytes):
        sizes = [q(C.byref(dims), 35, c) for c in (1, 2, 5, 12)]
        assert 0 < sizes[0] and all(a < b for a, b in zip(sizes, sizes[1:]))
        assert q(C.byref(dims), 36, 2) > q(C.byref(dims), 35, 2)
        assert q(C.byref(dims), 35, 0) == 0 and q(C.byref(dims), 0, 2) == 0
        assert q(C.byref(dims), F.MAX_PLAYERS, 1) > 0 and q(C.byref(dims), F.MAX_PLAYERS + 1, 1) == 0


def _cpu_model(name="TINY", train=False):
    cfg = model_config(name, dropout=0.2)
    return build_dropin(cfg, 3, device="cpu").train(train), make_batch(cfg, 3, seed=1)


def test_argument_validation():
    model, b = _cpu_model()
    args = (b["src"], b["static"], b["times"], b["lengths"])
    T, N = b["src"].shape[0], b["src"].shape[2] // 2
    P = N + 1
    phi = torch.randn(3, P)
    for fn, extra in ((F.deletion_curves, [dict(order="sideways"), dict(steps=[0, 2, 2]), dict(steps=[0, P + 1]),
                                           dict(steps=[-1, 2]), dict(steps=1), dict(steps=P + 2),
                                           dict(steps=np.array([0.5, 1.0]))]),
                      (F.infidelity, [dict(p_remove=0.0), dict(p_remove=1.5), dict(p_remove=-0.1), dict(n_samples=0),
                                      dict(seed=-1)])):
        with pytest.raises(TypeError):
            fn(torch.nn.Linear(2, 2), *args, phi)
        with pytest.raises(ValueError, match="eval"):
            fn(model.train(), *args, phi)
        model.eval()
        bad = extra + [dict(attributions=torch.randn(3, P - 1)), dict(attributions=torch.randn(2, P)),
                       dict(attributions=torch.randn(P + 1)), dict(attributions=(torch.randn(3, N), None)),
                       dict(attributions=(torch.randn(3, N), torch.randn(3, 2))), dict(target=7),
                       dict(sensor_groups=[0, 0, 2] + list(range(3, N))),
                       dict(feature_mask=np.zeros((T, N), dtype=np.float32)), dict(internal_batch_size=0),
                       dict(feature_mask=np.full((T, N), F.MAX_PLAYERS, dtype=np.int64))]
        for kw in bad:
            kw = dict(kw)
            a = kw.pop("attributions", phi)
            with pytest.raises(ValueError):
                fn(model, *args, a, **kw)
    mask = np.full((T, N), -1, dtype=np.int64)
    mask[0, 0] = F.MAX_PLAYERS - 1
    with pytest.raises(ValueError, match="at most"):
        F.deletion_curves(model, *args, torch.zeros(F.MAX_PLAYERS + 1), feature_mask=mask, steps=2)


def test_no_cuda_raises(monkeypatch):
    model, b = _cpu_model()
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    args = (model.eval(), b["src"], b["static"], b["times"], b["lengths"], torch.randn(3, b["src"].shape[2] // 2 + 1))
    with pytest.raises(L.RaindropB200Error):
        F.deletion_curves(*args)
    with pytest.raises(L.RaindropB200Error):
        F.infidelity(*args, n_samples=4)
    # P = 16384 passes the host checks and fails only for want of CUDA
    T, N = b["src"].shape[0], b["src"].shape[2] // 2
    mask = np.full((T, N), -1, dtype=np.int64)
    mask[0, 0] = F.MAX_PLAYERS - 2
    with pytest.raises(L.RaindropB200Error):
        F.deletion_curves(*args[:5], torch.zeros(F.MAX_PLAYERS), feature_mask=mask, steps=2)


def test_removal_counts():
    np.testing.assert_array_equal(F.removal_counts(5), np.arange(6))
    np.testing.assert_array_equal(F.removal_counts(64), np.arange(65))
    np.testing.assert_array_equal(F.removal_counts(100), np.arange(0, 101, 5))
    np.testing.assert_array_equal(F.removal_counts(10201), np.floor(np.linspace(0, 1, 21) * 10201 + 0.5))
    np.testing.assert_array_equal(F.removal_counts(10, 3), [0, 5, 10])
    np.testing.assert_array_equal(F.removal_counts(10, 11), np.arange(11))
    np.testing.assert_array_equal(F.removal_counts(10, [0, 3, 10]), [0, 3, 10])
    assert F.removal_counts(10).dtype == np.int32


def test_site_107_words_pinned_and_removal_rate():
    """The words are Philox site 107 (numpy restatement, pinned values), and the removal rate is p_remove."""
    w = dropout_words_at(3, 5, SITE, np.arange(8, dtype=np.uint64))
    np.testing.assert_array_equal(w, [599038556, 671472771, 2053314942, 2368868727, 1111865903, 781441816, 256507104,
                                      1300309792])
    np.testing.assert_array_equal(dropout_words_at(0, 0, SITE, np.array([0, 5, 1000003], dtype=np.uint64)),
                                  [2993549102, 4112477014, 730556050])
    assert not np.array_equal(w, dropout_words_at(3, 5, 106, np.arange(8, dtype=np.uint64)))
    assert not np.array_equal(w, dropout_words_at(3, 6, SITE, np.arange(8, dtype=np.uint64)))
    B, P, M = 16, 37, 50
    for p in (0.1, 0.5, 0.9):
        keep = _np_sample_keep(11, 7, 0, M, B, P, p)
        n, k = keep.size, int((keep == 0).sum())
        assert abs(k - n * p) < 4.5 * np.sqrt(n * p * (1 - p)), (p, k, n)
    assert (_np_sample_keep(11, 7, 0, 2, B, P, 1.0) == 0).all()
    # replicate m0 + m of a later chunk draws at step + m0 + m
    np.testing.assert_array_equal(_np_sample_keep(1, 2, 3, 2, B, P, 0.5), _np_sample_keep(1, 2, 0, 5, B, P, 0.5)[3 * B:])


def _host_summaries(counts, P, dele, ins, clean):
    """(deletion AUC, insertion AUC, AOPC) restated on the host: trapezoids over counts / P, mean of clean - dele."""
    x = np.asarray(counts, dtype=np.float64) / P
    auc = lambda y: float(np.sum(np.diff(x) * (y[1:] + y[:-1]) / 2))
    return auc(np.asarray(dele, float)), auc(np.asarray(ins, float)), float(np.mean(clean - np.asarray(dele, float)))


def test_auc_aopc_hand_cases():
    # a linear drop from 1 to 0 over 4 players: deletion AUC 1/2, insertion 1/2; AOPC over 5 points = mean(0..1)
    d, i, a = _host_summaries([0, 1, 2, 3, 4], 4, [1, .75, .5, .25, 0], [0, .25, .5, .75, 1], 1.0)
    assert (d, i, a) == (0.5, 0.5, 0.5)
    # uneven counts: trapezoids of widths 0.1, 0.9
    d, _, a = _host_summaries([0, 1, 10], 10, [2, 0, 0], [0, 0, 2], 2.0)
    assert abs(d - 0.1) < 1e-15 and abs(a - (0 + 2 + 2) / 3) < 1e-15


def test_infidelity_from_moments_hand_cases():
    a = np.array([1.0, -2.0, 0.5, 3.0])
    d = np.array([0.8, -1.5, 1.0, 2.0])
    mom = np.array([[len(a), a.sum(), d.sum(), (a * a).sum(), (a * d).sum(), (d * d).sum()]])
    np.testing.assert_allclose(F.infidelity_from_moments(mom).numpy(), [np.mean((a - d) ** 2)], rtol=1e-14)
    beta = (a * d).sum() / (a * a).sum()
    np.testing.assert_allclose(F.infidelity_from_moments(mom, True).numpy(), [np.mean((beta * a - d) ** 2)], rtol=1e-13)
    np.testing.assert_allclose(F.infidelity_beta(mom).numpy(), [beta], rtol=1e-15)
    # beta scale invariance: scaling the attributions leaves the normalised infidelity unchanged
    for c in (1e-3, 7.0, -2.0):
        ms = np.array([[len(a), (c * a).sum(), d.sum(), (c * a * c * a).sum(), (c * a * d).sum(), (d * d).sum()]])
        np.testing.assert_allclose(F.infidelity_from_moments(ms, True).numpy(),
                                   F.infidelity_from_moments(mom, True).numpy(), rtol=1e-12)
    # sum a^2 = 0: beta = 0, the normalised infidelity is mean d^2
    z = np.array([[4.0, 0.0, d.sum(), 0.0, 0.0, (d * d).sum()]])
    assert float(F.infidelity_beta(z)[0]) == 0.0
    np.testing.assert_allclose(F.infidelity_from_moments(z, True).numpy(), [np.mean(d * d)], rtol=1e-15)


def test_player_attributions_against_numpy_loop():
    rng = np.random.default_rng(0)
    T, B, N = 7, 3, 5
    a = torch.from_numpy(rng.normal(size=(T, B, 2 * N)).astype(np.float32))
    st = torch.from_numpy(rng.normal(size=(B, 4)).astype(np.float32))
    groups = np.array([1, 0, 1, 2, 0])
    masks = [rng.integers(-1, 6, size=(T, N)), rng.integers(-1, 9, size=(T, B, N))]
    cases = [(dict(sensor_groups=groups), lambda t, b, n: groups[n], 3),
             (dict(), lambda t, b, n: n, N),
             (dict(feature_mask=masks[0]), lambda t, b, n: masks[0][t, n], masks[0].max() + 1),
             (dict(feature_mask=masks[1]), lambda t, b, n: masks[1][t, b, n], masks[1].max() + 1)]
    for kw, pid, G in cases:
        ref = np.zeros((B, G + 1))
        for t, b, n in itertools.product(range(T), range(B), range(N)):
            if pid(t, b, n) >= 0:
                ref[b, pid(t, b, n)] += float(a[t, b, n])
        ref[:, G] = st.double().sum(dim=1).numpy()
        got = F.player_attributions(a, st, **kw)
        assert got.dtype == torch.float64 and got.shape == (B, G + 1)
        np.testing.assert_allclose(got.numpy(), ref, rtol=1e-13, atol=1e-13)
    assert F.player_attributions(a).shape == (B, N)
    torch.use_deterministic_algorithms(True)
    try:
        F.player_attributions(a, st, feature_mask=masks[1])
    finally:
        torch.use_deterministic_algorithms(False)


# ---- GPU ------------------------------------------------------------------------------------------------------------
EXACT = 2
CONFIGS = [("TINY", 4), ("TINY8", 3), ("P19", 4), ("P12", 3), ("PAM", 2)]


def _setup(name, B, seed=1, mode=EXACT):
    cfg = model_config(name, dropout=0.2)
    model = build_dropin(cfg, 5).eval()
    model._plan.obprop_mode = mode
    d = to_dev(make_batch(cfg, B, seed=seed))
    return cfg, model, d


def _args(model, d):
    return (model, d["src"], d["static"], d["times"], d["lengths"])


def _phi(B, P, seed=0, special=False):
    g = torch.Generator().manual_seed(seed)
    phi = torch.randn(B, P, generator=g)
    if special:
        phi = torch.round(phi * 2) / 2                       # ties
        phi[:, ::7] = 0.0
        phi[:, 1::7] = -0.0
        phi[:, 3::11] = float("nan")
        phi[:, 5::13] = float("inf")
        phi[:, 6::13] = -float("inf")
    return phi.cuda()


def _masks(cfg, d):
    T, B, N = d["src"].shape[0], d["src"].shape[1], cfg["d_inp"]
    g = torch.Generator().manual_seed(3)
    shared = torch.randint(-1, 2 * N, (T, N), generator=g)
    per_sample = torch.randint(-1, N + 3, (T, B, N), generator=g)
    shared[0, 0], per_sample[0, 0, 0] = 2 * N - 1, N + 2
    return shared, per_sample


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 37, 341, 10201, 16384])
def test_rank_matches_lexsort(P):
    cfg, model, d = _setup("TINY", 3)
    T, N = d["src"].shape[0], cfg["d_inp"]
    G = P - 1
    if G >= 1:
        mask = torch.full((T, N), -1, dtype=torch.int64)
        mask.view(-1)[: min(G, T * N)] = torch.arange(min(G, T * N))
        mask[0, 0] = G - 1
        phi = _phi(3, P, seed=P, special=True)
        for order in F.ORDERS:
            got = F.deletion_curves(*_args(model, d), phi, feature_mask=mask, steps=2, order=order)
            np.testing.assert_array_equal(got.rank.cpu().numpy(), _np_rank(phi.cpu().numpy(), order), err_msg=order)
    else:   # one player: the static vector alone is not a model with value-cell players; use TINY8 without statics
        cfg, model, d = _setup("TINY8", 3)
        mask = torch.full((d["src"].shape[0], cfg["d_inp"]), -1, dtype=torch.int64)
        mask[0, 0] = 0
        got = F.deletion_curves(*_args(model, d), torch.zeros(1), feature_mask=mask)
        assert got.rank.cpu().numpy().tolist() == [[0]] * 3


def _debug_rows(model, d, r, rank=None, counts=None, seed=0, step=0, p_remove=0.5, q0=0, nc=1):
    """rd_debug_removal_inputs of one chunk: (keep [nc*B, P], src_e, statics_e, times_e, lengths_e)."""
    cl, lib, B, P = r.cl, r.cl.lib, d["src"].shape[1], r.P
    T, N2 = d["src"].shape[0], d["src"].shape[2]
    dev = d["src"].device
    keep = torch.empty(nc * B, P, dtype=torch.uint8, device=dev)
    src_e = torch.empty(T, nc * B, N2, device=dev)
    st_e = torch.empty(nc * B, cl.st.shape[1], device=dev) if cl.st is not None else None
    tm_e = torch.empty(T, nc * B, device=dev)
    ln_e = torch.empty(nc * B, dtype=torch.int64, device=dev)
    key = torch.tensor(np.array([seed, step], dtype=np.uint64).view(np.int64), device=dev)
    counts_d = torch.as_tensor(counts, dtype=torch.int32, device=dev) if counts is not None else None
    dims = cl.plan.dims(B, False)
    L.check(lib.rd_debug_removal_inputs(C.byref(dims), cl.x.data_ptr(), L.ptr(cl.st), cl.tm.data_ptr(), cl.ln.data_ptr(),
                                        cl.x0.data_ptr(), L.ptr(cl.st0), r.player.data_ptr(), r.stride_t, r.stride_b, P,
                                        L.ptr(rank), L.ptr(counts_d), 0 if counts is None else len(counts), key.data_ptr(),
                                        p_remove, q0, nc, keep.data_ptr(), src_e.data_ptr(), L.ptr(st_e),
                                        tm_e.data_ptr(), ln_e.data_ptr(), L.stream_ptr(dev)), "rd_debug_removal_inputs")
    return keep, src_e, st_e, tm_e, ln_e


def _removal(model, d, phi, baselines=None, **players):
    r = F._Removal("t", model, d["src"], d["static"], baselines, phi, players.get("sensor_groups"),
                   players.get("feature_mask"), None)
    r.load(model, d["src"], d["static"], d["times"], d["lengths"], None, baselines)
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["TINY", "TINY8"])
def test_expanded_rows_bitwise(name):
    """Keep tables and rows of curve pairs and infidelity replicates equal torch-built removed copies bit for bit:
    sensor groups, [T, N] and [T, B, N] masks, with and without statics, zero and nonzero baselines."""
    B = 4
    cfg, model, d = _setup(name, B)
    T, N = d["src"].shape[0], cfg["d_inp"]
    shared, per_sample = _masks(cfg, d)
    groups = [n % 3 for n in range(N)]
    g = torch.Generator().manual_seed(9)
    x0 = torch.randn(d["src"].shape, generator=g).cuda()
    st0 = torch.randn(d["static"].shape, generator=g).cuda() if d["static"] is not None else None
    cases = [(dict(sensor_groups=groups), torch.tensor(groups).view(1, 1, N).expand(T, B, N)),
             (dict(feature_mask=shared), shared[:, None, :].expand(T, B, N)),
             (dict(feature_mask=per_sample), per_sample)]
    for (players, cells), base in itertools.product(cases, (None, (x0, st0))):
        G = int(cells.max()) + 1
        P = G + (1 if d["static"] is not None else 0)
        phi = _phi(B, P, seed=P)
        r = _removal(model, d, phi, base, **players)
        xb, sb = (None, None) if base is None else base
        curves = F.deletion_curves(*_args(model, d), phi, baselines=base, steps=min(P + 1, 6), **players)
        counts = curves.counts
        K = len(counts)
        keep, *rows = _debug_rows(model, d, r, rank=curves.rank, counts=counts, q0=1, nc=2 * K - 1)
        np.testing.assert_array_equal(keep.cpu().numpy(), _np_curve_keep(curves.rank.cpu().numpy(), counts, 1, 2 * K - 1))
        want = _removed_rows(d, cells, keep, xb, sb)
        for got, ref in zip(rows, want):
            assert (got is None) == (ref is None) and (got is None or torch.equal(got, ref))
        keep, *rows = _debug_rows(model, d, r, seed=5, step=3, p_remove=0.3, q0=2, nc=3)
        np.testing.assert_array_equal(keep.cpu().numpy(), _np_sample_keep(5, 3, 2, 3, B, P, 0.3))
        want = _removed_rows(d, cells, keep, xb, sb)
        for got, ref in zip(rows, want):
            assert (got is None) == (ref is None) and (got is None or torch.equal(got, ref))


@pytest.mark.gpu
@pytest.mark.parametrize("name,B", CONFIGS)
def test_curve_logits_against_module_forward(name, B):
    """One chunk: the curve logits are bitwise the module's eval forward on the same concatenated rows; the curves
    start and end at F(x) and F(x'); deletion at count 1 is F(x) - feature_ablation of the top-ranked player."""
    cfg, model, d = _setup(name, B)
    args = _args(model, d)
    N = cfg["d_inp"]
    groups = [n // 2 for n in range(N)]
    phi_p, phi_s = A.feature_ablation(*args, sensor_groups=groups)
    phi = phi_p if phi_s is None else torch.cat([phi_p, phi_s[:, None]], dim=1)
    P = phi.shape[1]
    K = P + 1
    cur = F.deletion_curves(*args, (phi_p, phi_s), sensor_groups=groups, internal_batch_size=2 * K * B)
    assert len(cur.counts) == K
    r = _removal(model, d, phi, sensor_groups=groups)
    keep, src_e, st_e, tm_e, ln_e = _debug_rows(model, d, r, rank=cur.rank, counts=cur.counts, nc=2 * K)
    with torch.no_grad():
        ref = model.forward(src_e, st_e, tm_e, ln_e)[0].view(2, K, B, -1)
    assert torch.equal(cur.deletion_logits, ref[0].transpose(0, 1))
    assert torch.equal(cur.insertion_logits, ref[1].transpose(0, 1))
    tgt = cur.target
    fx = cur.clean.double()
    x0 = d["src"].clone()
    x0[:, :, :N] = 0.0
    st0 = None if d["static"] is None else torch.zeros_like(d["static"])
    with torch.no_grad():
        lx = model.forward(*args[1:])[0]
        fx0 = model.forward(x0, st0, d["times"], d["lengths"])[0].gather(1, tgt[:, None])[:, 0].double()
    assert torch.equal(tgt, lx.argmax(dim=1))
    scale = float(fx.abs().max()) + 1.0
    for got in (cur.deletion[:, 0], cur.insertion[:, -1]):
        assert float((got.double() - fx).abs().max()) < 1e-5 * scale
    for got in (cur.deletion[:, -1], cur.insertion[:, 0]):
        assert float((got.double() - fx0).abs().max()) < 1e-4 * scale
    top = cur.rank.long().argmin(dim=1)
    want = fx - phi.double().gather(1, top[:, None])[:, 0]
    assert float((cur.deletion[:, 1].double() - want).abs().max()) < 2e-6 * scale
    # the device summaries against the host restatement of the returned values
    x = torch.as_tensor(cur.counts, dtype=torch.float64, device=fx.device) / P
    auc = lambda y: ((x[1:] - x[:-1]) * (y[:, 1:] + y[:, :-1]) / 2).sum(1)
    torch.testing.assert_close(cur.deletion_auc(), auc(cur.deletion.double()), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(cur.insertion_auc(), auc(cur.insertion.double()), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(cur.aopc(), (fx[:, None] - cur.deletion.double()).mean(1), rtol=1e-12, atol=1e-12)
    prob = lambda lg: torch.softmax(lg.double(), -1).gather(-1, tgt.view(B, 1, 1).expand(B, K, 1))[..., 0]
    torch.testing.assert_close(cur.deletion_auc("probability"), auc(prob(cur.deletion_logits)), rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(cur.insertion_auc("probability"), auc(prob(cur.insertion_logits)), rtol=1e-12,
                               atol=1e-14)
    px = torch.softmax(lx.double(), -1).gather(1, tgt[:, None])[:, 0]
    torch.testing.assert_close(cur.aopc("probability"), (px[:, None] - prob(cur.deletion_logits)).mean(1), rtol=1e-12,
                               atol=1e-14)


def _restated_moments(model, d, phi, cells, seed, step, M, p_remove):
    """[B, 6] fp64 from module forwards on the restated keep tables, summed in replicate order."""
    B, P = phi.shape
    keep = _np_sample_keep(seed, step, 0, M, B, P, p_remove)
    rows = _removed_rows(d, cells, keep)
    with torch.no_grad():
        lx = model.forward(d["src"], d["static"], d["times"], d["lengths"])[0]
        lr = model.forward(*rows)[0]
    tgt = lx.argmax(1)
    fx = lx.gather(1, tgt[:, None])[:, 0].double().cpu().numpy()
    fr = lr.view(M, B, -1).gather(2, tgt.view(1, B, 1).expand(M, B, 1))[..., 0].double().cpu().numpy()
    ph = phi.double().cpu().numpy()
    mom = np.zeros((B, 6))
    for m in range(M):
        a = ((1 - keep[m * B:(m + 1) * B]) * ph).sum(axis=1)
        dd = fx - fr[m]
        mom += np.stack([np.ones(B), a, dd, a * a, a * dd, dd * dd], 1)
    return mom


@pytest.mark.gpu
@pytest.mark.parametrize("name,B", CONFIGS)
def test_infidelity_moments_against_restatement(name, B):
    cfg, model, d = _setup(name, B)
    N = cfg["d_inp"]
    P = N + (1 if d["static"] is not None else 0)
    phi = _phi(B, P, seed=4)
    M = 12
    got = F.infidelity(*_args(model, d), phi, n_samples=M, p_remove=0.4, seed=7, step=2)
    ref = _restated_moments(model, d, phi, torch.arange(N).view(1, 1, N), 7, 2, M, 0.4)
    m = got.moments.cpu().numpy()
    np.testing.assert_array_equal(m[:, 0], ref[:, 0])
    np.testing.assert_array_equal(m[:, [2, 5]], ref[:, [2, 5]])      # d summed in replicate order by both
    np.testing.assert_allclose(m, ref, rtol=1e-12, atol=1e-12 * np.abs(ref).max())
    torch.testing.assert_close(got.infidelity, F.infidelity_from_moments(got.moments))


@pytest.mark.gpu
def test_infidelity_at_p1_is_the_squared_shapley_delta():
    """p_remove = 1 removes every player: a - d is the efficiency gap of the attributions, so the infidelity is the
    squared convergence delta; exact Shapley values (all permutations on TINY) give ~0."""
    cfg, model, d = _setup("TINY", 4)
    args = _args(model, d)
    P = cfg["d_inp"] + 1
    perms = np.array(list(itertools.permutations(range(P))))
    phi_p, phi_s, delta = A.shapley_value_sampling(*args, permutations=perms, return_convergence_delta=True)
    inf = F.infidelity(*args, (phi_p, phi_s), n_samples=3, p_remove=1.0)
    scale = float(inf.clean_logits.abs().max()) ** 2
    torch.testing.assert_close(inf.infidelity, delta.double() ** 2, rtol=1e-3, atol=1e-10 * scale)
    assert float(inf.infidelity.max()) < 1e-9 * scale
    phi_p, phi_s, delta = A.shapley_value_sampling(*args, n_samples=2, return_convergence_delta=True)
    phi_p = phi_p * 1.5
    inf = F.infidelity(*args, (phi_p, phi_s), n_samples=2, p_remove=1.0)
    gap = phi_p.double().sum(1) + phi_s.double() - (inf.clean_logits.double().gather(1, inf.target[:, None])[:, 0] -
                                                    F.deletion_curves(*args, (phi_p, phi_s), steps=[P]).deletion[:, 0])
    torch.testing.assert_close(inf.infidelity, gap ** 2, rtol=1e-6, atol=1e-9 * scale)


@pytest.mark.gpu
def test_determinism_chunking_and_split_calls():
    cfg, model, d = _setup("P19", 6)
    args = _args(model, d)
    mask, _ = A.time_window_mask(d["times"], 6.0, sensor_groups=cfg["d_inp"])
    B = 6
    P = int(mask.max()) + 2
    phi = _phi(B, P, seed=2)
    kw = dict(feature_mask=mask.cpu(), steps=7)
    ref = F.deletion_curves(*args, phi, **kw)
    for ibs in (B, 3 * B, 1, 5 * B, None):             # one pair, a chunk that does not divide 14 pairs, everything
        got = F.deletion_curves(*args, phi, internal_batch_size=ibs, **kw)
        for f in ("rank", "deletion_logits", "insertion_logits", "summaries", "target"):
            assert torch.equal(getattr(got, f), getattr(ref, f)), (ibs, f)
    ikw = dict(feature_mask=mask.cpu(), n_samples=10, seed=4, step=1)
    iref = F.infidelity(*args, phi, **ikw)
    for ibs in (B, 3 * B, 1, 7 * B):
        got = F.infidelity(*args, phi, internal_batch_size=ibs, **ikw)
        assert torch.equal(got.moments, iref.moments), ibs
    assert torch.equal(F.infidelity(*args, phi, **ikw).moments, iref.moments)
    a = F.infidelity(*args, phi, feature_mask=mask.cpu(), n_samples=4, seed=4, step=1)
    b = F.infidelity(*args, phi, feature_mask=mask.cpu(), n_samples=6, seed=4, step=5)
    torch.testing.assert_close(a.moments + b.moments, iref.moments, rtol=1e-13, atol=1e-12)
    assert not torch.equal(F.infidelity(*args, phi, feature_mask=mask.cpu(), n_samples=10, seed=5, step=1).moments,
                           iref.moments)


@pytest.mark.gpu
def test_cuda_graph_capture_and_no_side_effects():
    from raindrop_b200.optim import FlatAdam
    import torch.nn.functional as TF
    cfg = model_config("P19", dropout=0.2)
    B = 8
    model = build_dropin(cfg, 8).train()
    opt = FlatAdam(model, lr=1e-3)
    for it in range(3):
        d = to_dev(make_batch(cfg, B, seed=60 + it))
        logits, _, _ = model.forward(d["src"], d["static"], d["times"], d["lengths"])
        TF.cross_entropy(logits, d["y"]).backward()
        opt.step()
    P = cfg["d_inp"] + 1
    phi = _phi(B, P, seed=1)
    args = (model, d["src"], d["static"], d["times"], d["lengths"], phi)
    with pytest.raises(ValueError):
        F.deletion_curves(*args)
    plan = model._plan
    slot = next(iter(plan._slots.values()))
    snap = {"flat_p": opt.flat_p.detach(), "flat_g": opt.flat_g, "exp_avg": opt.exp_avg, "exp_avg_sq": opt.exp_avg_sq,
            "step": opt.step_count, "rng": plan.rng_state, "slot.src": slot.src, "slot.logits": slot.logits}
    snap.update({"param." + k: p.detach() for k, p in model.named_parameters()})
    snap.update({"grad." + k: p.grad for k, p in model.named_parameters() if p.grad is not None})
    before = {k: v.clone() for k, v in snap.items()}
    model.eval()
    plan.obprop_mode = EXACT
    calls = (lambda: F.deletion_curves(*args, steps=9, internal_batch_size=4 * B),
             lambda: F.infidelity(*args, n_samples=20, seed=3, internal_batch_size=6 * B, normalize=True))
    for call in calls:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            eager = call()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = call()
        outs = [v for v in vars(out).values() if torch.is_tensor(v)]
        for t in outs:
            t.zero_()
        g.replay()
        torch.cuda.synchronize()
        for k, v in vars(eager).items():
            if torch.is_tensor(v):
                assert torch.equal(getattr(out, k), v), k
    torch.cuda.synchronize()
    for k, v in snap.items():
        assert torch.equal(v, before[k]), k
    model.train()
    logits, _, _ = model.forward(d["src"], d["static"], d["times"], d["lengths"])
    TF.cross_entropy(logits, d["y"]).backward()
    opt.step()


@pytest.mark.gpu
def test_full_size_p19_windows_and_pam_cells():
    cfg, model, d = _setup("P19", 128, mode=0)
    mask, n_win = A.time_window_mask(d["times"], 6.0, sensor_groups=cfg["d_inp"])
    P = int(mask.max()) + 2
    phi = _phi(128, P, seed=3)
    cur = F.deletion_curves(*_args(model, d), phi, feature_mask=mask)
    assert cur.deletion.shape == (128, 21) and torch.isfinite(cur.summaries).all()
    inf = F.infidelity(*_args(model, d), phi, feature_mask=mask, n_samples=64)
    assert torch.isfinite(inf.infidelity).all() and float(inf.moments[0, 0]) == 64
    cfg, model, d = _setup("PAM", 2, mode=0)
    T, N = d["src"].shape[0], cfg["d_inp"]
    cells = torch.arange(T * N).view(T, N)             # a player per value cell: P = 10,200 (PAM has no statics)
    P = T * N + (1 if d["static"] is not None else 0)
    phi = _phi(2, P, seed=4)
    cur = F.deletion_curves(*_args(model, d), phi, feature_mask=cells, steps=5)
    assert torch.isfinite(cur.summaries).all()
    np.testing.assert_array_equal(cur.rank.cpu().numpy(), _np_rank(phi.cpu().numpy(), "descending"))
    inf = F.infidelity(*_args(model, d), phi, feature_mask=cells, n_samples=8)
    assert torch.isfinite(inf.infidelity).all()
