"""KernelSHAP of Raindrop_v2 (raindrop_b200.attribution.kernel_shap, rd_raindrop_v2_kernel_shap).  Reference values:
tests/golden/kernel_shap.npz, the value of every coalition of the TINY cases from the reference's own files
(tools/make_kernel_shap_golden.py), and the exact Shapley values of sensor_attribution.npz and cell_attribution.npz.
Tolerances follow test_sensor_attribution.py."""
import itertools
import json
import math

import numpy as np
import pytest
import torch

from helpers import build_dropin, case_setup, load_golden, normwise, to_dev
from raindrop_b200 import attribution as A
from raindrop_b200.synth import make_batch, model_config

EXACT, FAST = 2, 1
TOL_EXACT, TOL_EXACT_WIDE, TOL_FAST = 2e-3, 1e-2, 2e-2
CASES = ["tiny_dense", "tiny_t0", "tiny_sparse", "tiny8_nostatic"]


def _exact_tol(cfg):
    return TOL_EXACT_WIDE if cfg["max_len"] * cfg["d_ob"] >= 1024 else TOL_EXACT


def _fixture(golden_dir, name="kernel_shap"):
    z = np.load(golden_dir + "/%s.npz" % name)
    return z, json.loads(bytes(z["meta"]).decode())


def _rows(Z):
    """Row of each coalition of Z in the fixture's index (itertools.product order: player 0 is the top bit)."""
    P = Z.shape[1]
    return (Z.astype(np.int64) << np.arange(P - 1, -1, -1)).sum(axis=1)


def _restate(values, Z, w):
    """kernel_shap_from_values on a fixture table values [2^P, B] (v(empty) is row 0, v(all) the last row)."""
    return A.kernel_shap_from_values(values[_rows(Z)], values[0], values[-1], Z, w)


def _exact_shapley(v, P):
    """Brute-force Shapley values of a host game v(keep [P] bool) -> float."""
    phi = np.zeros(P)
    for bits in itertools.product([False, True], repeat=P):
        S = np.array(bits)
        s = int(S.sum())
        for g in np.nonzero(~S)[0]:
            T = S.copy()
            T[g] = True
            phi[g] += math.factorial(s) * math.factorial(P - s - 1) / math.factorial(P) * (v(T) - v(S))
    return phi


def _game(P, seed):
    rng = np.random.default_rng(seed)
    a, W = rng.normal(size=P), rng.normal(size=(P, P))
    return lambda S: float(np.tanh(a @ S + S @ W @ S / P))


def _estimate(v, Z, w):
    P = Z.shape[1]
    vals = np.array([v(z.astype(bool)) for z in Z]).reshape(-1, 1)
    return A.kernel_shap_from_values(vals, [v(np.zeros(P, bool))], [v(np.ones(P, bool))], Z, w)[0]


# ---- CPU: host math -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [2, 3, 5, 8])
def test_exhaustive_coalitions_give_exact_shapley_values(P):
    v = _game(P, P)
    Z, w = A.all_coalitions(P)
    assert Z.shape == (2 ** P - 2, P) and Z.dtype == np.uint8
    np.testing.assert_allclose(_estimate(v, Z, w), _exact_shapley(v, P), rtol=0, atol=1e-13)


def test_additive_game_is_recovered_from_a_sampled_set():
    """v(S) = sum_{i in S} a_i: any coalition set whose A has full rank gives back a (fp64 rounding)."""
    P = 12
    a = np.random.default_rng(1).normal(size=P)
    for M, seed in ((60, 0), (200, 1), (2048, 2)):
        Z, w = A.sample_coalitions(P, M, seed)
        assert np.linalg.matrix_rank((Z.T * w) @ Z.astype(np.float64)) == P
        phi = A.kernel_shap_from_values((Z @ a)[:, None], [0.0], [a.sum()], Z, w)[0]
        np.testing.assert_allclose(phi, a, rtol=0, atol=1e-12)


@pytest.mark.parametrize("M", [2, 4, 6, 10])
def test_efficiency_holds_below_P_coalitions(M):
    P = 12
    v = _game(P, 7)
    Z, w = A.sample_coalitions(P, M, seed=M)
    phi = _estimate(v, Z, w)
    assert np.all(np.isfinite(phi))
    assert abs(phi.sum() - (v(np.ones(P, bool)) - v(np.zeros(P, bool)))) < 1e-13


def test_weight_scaling_does_not_change_the_result():
    P = 9
    v = _game(P, 3)
    for Z, w in (A.sample_coalitions(P, 300, seed=5), A.all_coalitions(P)):
        ref = _estimate(v, Z, w)
        for c in (1e-3, 37.5):
            np.testing.assert_allclose(_estimate(v, Z, c * w), ref, rtol=0, atol=1e-10)


def test_one_and_two_players():
    """P = 1 has no proper coalition: phi = v(all) - v(empty); P = 2 gives the exact values from any paired sample."""
    Z, w = A.sample_coalitions(1, 10)
    assert Z.shape == (0, 1) and w.shape == (0,)
    Ze, _ = A.all_coalitions(1)
    assert Ze.shape == (0, 1)
    phi = A.kernel_shap_from_values(np.zeros((0, 3)), [1.0, 2.0, -1.0], [4.0, 2.5, 3.0], Z, w)
    np.testing.assert_allclose(phi[:, 0], [3.0, 0.5, 4.0], rtol=0, atol=1e-15)
    v = _game(2, 11)
    for Z, w in (A.sample_coalitions(2, 7, seed=3), A.all_coalitions(2)):
        np.testing.assert_allclose(_estimate(v, Z, w), _exact_shapley(v, 2), rtol=0, atol=1e-14)


def test_sample_coalitions_follow_the_seed_and_pair():
    Z, w = A.sample_coalitions(35, 25, seed=3)
    assert Z.shape == (26, 35) and Z.dtype == np.uint8 and w.dtype == np.float64
    np.testing.assert_array_equal(w, np.full(26, 1 / 26))
    Z2, _ = A.sample_coalitions(35, 25, seed=3)
    np.testing.assert_array_equal(Z, Z2)
    assert not np.array_equal(Z, A.sample_coalitions(35, 25, seed=4)[0])
    np.testing.assert_array_equal(Z[0::2] + Z[1::2], np.ones((13, 35)))
    s = Z.sum(axis=1)
    assert s.min() >= 1 and s.max() <= 34


def test_sample_coalition_sizes_follow_the_kernel():
    """Size histogram of 40000 pairs at P = 10, seed 0, against p(s) ~ (P-1) / (s (P-s)): every bin within 4.5 sigma."""
    P, pairs = 10, 40000
    Z, _ = A.sample_coalitions(P, 2 * pairs, seed=0)
    sizes = np.arange(1, P)
    p = (P - 1) / (sizes * (P - sizes))
    p /= p.sum()
    counts = np.bincount(Z[0::2].sum(axis=1), minlength=P)[1:]
    sigma = np.sqrt(pairs * p * (1 - p))
    assert np.all(np.abs(counts - pairs * p) < 4.5 * sigma), (counts, pairs * p)
    # within a size, every player is equally likely
    per_player = Z[0::2][Z[0::2].sum(axis=1) == 3].mean(axis=0)
    assert np.all(np.abs(per_player - 0.3) < 0.03), per_player


def test_all_coalitions_weights_and_range():
    Z, w = A.all_coalitions(6)
    s = Z.sum(axis=1)
    assert len({tuple(r) for r in Z}) == 62 and s.min() == 1 and s.max() == 5
    np.testing.assert_allclose(w, 5 / (np.array([math.comb(6, int(k)) for k in s]) * s * (6 - s)))
    for bad in (0, 21):
        with pytest.raises(ValueError):
            A.all_coalitions(bad)
    with pytest.raises(ValueError):
        A.sample_coalitions(0, 4)
    with pytest.raises(ValueError):
        A.sample_coalitions(4, 0)


@pytest.mark.parametrize("name", CASES)
def test_restatement_reproduces_exact_shapley_fixture(golden_dir, name):
    """The fp64 restatement applied to the reference's coalition values through all_coalitions reproduces the exact
    Shapley values of sensor_attribution.npz (sensors, and sensor groups) and cell_attribution.npz (the cell map)."""
    z, meta = _fixture(golden_dir)
    zs, _ = _fixture(golden_dir, "sensor_attribution")
    vals = z[name + ".values"]
    P = vals.shape[0].bit_length() - 1
    np.testing.assert_array_equal(z["coalitions_%d" % P][_rows(A.all_coalitions(P)[0])], A.all_coalitions(P)[0])
    assert normwise(_restate(vals, *A.all_coalitions(P)), zs[name + ".shapley"]) < 1e-6
    ends, tgt = z[name + ".endpoint_logits"], z[name + ".target"]
    f = np.take_along_axis(ends, np.broadcast_to(tgt[None, :, None], (2, len(tgt), 1)), axis=2)[:, :, 0]
    assert np.abs(vals[-1] - f[1]).max() < 1e-5 * np.abs(f).max()
    assert np.abs(vals[0] - f[0]).max() < 1e-5 * np.abs(f).max()
    if name in meta["groups"]:
        vg = z[name + ".values_grouped"]
        Pg = vg.shape[0].bit_length() - 1
        assert normwise(_restate(vg, *A.all_coalitions(Pg)), zs[name + ".shapley_grouped"]) < 1e-6
    if name == meta["cell_case"]:
        zc, _ = _fixture(golden_dir, "cell_attribution")
        np.testing.assert_array_equal(z[name + ".cells"], zc[name + ".cells"])
        vc = z[name + ".values_cells"]
        Pc = vc.shape[0].bit_length() - 1
        assert normwise(_restate(vc, *A.all_coalitions(Pc)), zc[name + ".shapley"]) < 1e-6


def test_operands_are_cached_in_one_entry():
    """One pinv and one copy per coalition set; another set replaces the entry; seed None never hits."""
    class Plan:
        pass
    plan, dev, calls = Plan(), torch.device("cpu"), []

    def make(seed):
        def f():
            calls.append(seed)
            return A.sample_coalitions(5, 8, seed)
        return f
    a = A._kernel_shap_operands(plan, ("sampled", 5, 8, 0), make(0), dev)
    assert A._kernel_shap_operands(plan, ("sampled", 5, 8, 0), make(0), dev) is a
    b = A._kernel_shap_operands(plan, ("sampled", 5, 8, 1), make(1), dev)
    assert b is not a and calls == [0, 1]
    assert a[2].shape == (5, 6) and a[2].dtype == torch.float64 and a[0].dtype == torch.uint8
    A._kernel_shap_operands(plan, None, make(2), dev)
    A._kernel_shap_operands(plan, None, make(2), dev)
    assert calls == [0, 1, 2, 2]
    assert A._sampled_key(5, 8, 3) == A._sampled_key(5, 8, np.int64(3)) == ("sampled", 5, 8, 3)
    for seed in (None, np.random.default_rng(0), np.random.SeedSequence(0), True):
        assert A._sampled_key(5, 8, seed) is None


def _cpu_model(train=False):
    cfg = model_config("TINY", dropout=0.2)
    return build_dropin(cfg, 3, device="cpu").train(train), make_batch(cfg, 3, seed=1)


def test_argument_validation():
    model, b = _cpu_model()
    args = (b["src"], b["static"], b["times"], b["lengths"])
    fn = A.kernel_shap
    with pytest.raises(TypeError):
        fn(torch.nn.Linear(2, 2), *args)
    with pytest.raises(ValueError, match="eval"):
        fn(model.train(), *args)
    model.eval()
    T, N = b["src"].shape[0], b["src"].shape[2] // 2
    Z, w = A.sample_coalitions(6, 8)
    bad = [dict(target=2), dict(target=torch.tensor([0, 1, -1])), dict(baselines=torch.zeros(1)),
           dict(sensor_groups=[0, 1, 2]), dict(sensor_groups=[0, 0, 2, 2, 2]),
           dict(sensor_groups=np.arange(N), feature_mask=np.zeros((T, N), dtype=np.int64)),
           dict(feature_mask=np.zeros((T, N), dtype=np.float32)), dict(internal_batch_size=0), dict(n_samples=0),
           dict(feature_mask=np.full((T, N), 5000, dtype=np.int64)),
           dict(coalitions=Z), dict(coalitions=(Z[:, :5], w)), dict(coalitions=(Z.astype(np.float64), w)),
           dict(coalitions=(2 * Z, w)), dict(coalitions=(Z, w[:-1])), dict(coalitions=(Z, -w)),
           dict(coalitions=(Z, np.full(8, np.nan)))]
    for kw in bad:
        with pytest.raises(ValueError):
            fn(model, *args, **kw)
    with pytest.raises(ValueError):
        fn(model, b["src"][:, :, :3], b["static"], b["times"], b["lengths"])


def test_no_cuda_raises(monkeypatch):
    from raindrop_b200.lib import RaindropB200Error
    model, b = _cpu_model()
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RaindropB200Error):
        A.kernel_shap(model.eval(), b["src"], b["static"], b["times"], b["lengths"], target=1, n_samples=8)


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _model(cfg, wseed, mode):
    m = build_dropin(cfg, wseed).eval()
    m._plan.obprop_mode = mode
    return m


def _cat(a_players, a_static):
    return a_players if a_static is None else torch.cat([a_players, a_static[:, None]], dim=1)


def _loop_values(model, d, cells, Z, target, x0=None, st0=None):
    """[M, B] fp64 v_b(z_j) from a loop of B-row module forwards; cells [T, B, N] (id -1 / >= G: no player), the
    static player last."""
    src, static = d["src"], d["static"]
    N = src.shape[2] // 2
    G = Z.shape[1] - (1 if static is not None else 0)
    cells = torch.as_tensor(cells, device=src.device).long()
    cells = torch.where((cells < 0) | (cells >= G), G, cells)
    base = torch.zeros_like(src[:, :, :N]) if x0 is None else x0[:, :, :N]
    out = []
    for z in Z:
        keep = torch.as_tensor(np.append(z[:G], 1).astype(bool), device=src.device)[cells]
        x = src.clone()
        x[:, :, :N] = torch.where(keep, src[:, :, :N], base)
        st = None
        if static is not None:
            st = static if z[-1] else (torch.zeros_like(static) if st0 is None else st0)
        with torch.no_grad():
            logits = model.forward(x, st, d["times"], d["lengths"])[0]
        out.append(logits.gather(1, target[:, None])[:, 0].double().cpu())
    return torch.stack(out).numpy()


def _loop_kernel_shap(model, d, cells, Z, w, target, x0=None, st0=None):
    P = Z.shape[1]
    v = _loop_values(model, d, cells, np.concatenate([np.zeros((1, P), np.uint8), np.ones((1, P), np.uint8), Z]),
                     target, x0, st0)
    return A.kernel_shap_from_values(v[2:], v[0], v[1], Z, w)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
@pytest.mark.parametrize("name", CASES)
def test_golden_exhaustive_and_sampled(golden_dir, name, mode):
    """all_coalitions(P) gives the reference's exact Shapley values (sensors; on tiny_dense also sensor groups and the
    cell map); a fixed-seed sampled set matches the fp64 restatement on the reference's coalition values."""
    z, meta = _fixture(golden_dir)
    zs, _ = _fixture(golden_dir, "sensor_attribution")
    zc, _ = _fixture(golden_dir, "cell_attribution")
    _, gm = load_golden(golden_dir, name)
    cfg, batch = case_setup(gm)
    d = to_dev(batch)
    model = _model(cfg, gm["weight_seed"], mode)
    target = None if gm["case"] == "tiny_t0" else torch.from_numpy(z[name + ".target"]).cuda()
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    tol = _exact_tol(cfg) if mode == EXACT else TOL_FAST
    vals = z[name + ".values"]
    P = vals.shape[0].bit_length() - 1
    phi, phi_st, delta = A.kernel_shap(*args, target=target, coalitions=A.all_coalitions(P), return_convergence_delta=True)
    errs = {"exhaustive": normwise(_cat(phi, phi_st), zs[name + ".shapley"]),
            "delta": float(delta.abs().max()) / float(np.abs(z[name + ".endpoint_logits"]).max())}
    Z, w = A.sample_coalitions(P, 40, seed=3)
    errs["sampled"] = normwise(_cat(*A.kernel_shap(*args, target=target, n_samples=40, seed=3)), _restate(vals, Z, w))
    if name in meta["groups"]:
        groups = meta["groups"][name]
        Pg = max(groups) + 2
        got = _cat(*A.kernel_shap(*args, target=target, sensor_groups=groups, coalitions=A.all_coalitions(Pg)))
        errs["grouped"] = normwise(got, zs[name + ".shapley_grouped"])
    if name == meta["cell_case"]:
        cells = torch.from_numpy(z[name + ".cells"][:, 0, :].copy())
        Pc = int(cells.max()) + 2
        got = _cat(*A.kernel_shap(*args, target=target, feature_mask=cells, coalitions=A.all_coalitions(Pc)))
        errs["cells"] = normwise(got, zc[name + ".shapley"])
        Zc, wc = A.sample_coalitions(Pc, 30, seed=5)
        got = _cat(*A.kernel_shap(*args, target=target, feature_mask=cells, coalitions=(Zc, wc)))
        errs["cells_sampled"] = normwise(got, _restate(z[name + ".values_cells"], Zc, wc))
    print(name, mode, errs)
    assert max(errs.values()) < tol, errs


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name,B,opts,window,M", [("P19", 6, {"zero_sensors": 10}, None, 96), ("P19", 1, {}, None, 64),
                                                      ("TINY8", 5, {}, None, 40), ("P19", 4, {}, 6.0, 48),
                                                      ("PAM", 2, {}, None, 24)])
def test_equals_module_loop(cfg_name, B, opts, window, M):
    """Exact mode: the device call equals the loop of B-row module forwards over the same coalitions followed by the
    numpy solve (sensor players, no statics, B = 1, the PAM shape and time-window players, P = 205 at P19), with a
    nonzero baseline."""
    cfg = model_config(cfg_name, dropout=0.2)
    d = to_dev(make_batch(cfg, B, seed=40 + B, **opts))
    model = _model(cfg, 9, EXACT)
    T, N = cfg["max_len"], cfg["d_inp"]
    gen = torch.Generator(device="cuda").manual_seed(3)
    x0 = 0.3 * torch.randn(d["src"].shape, device="cuda", generator=gen)
    st0 = None if d["static"] is None else 0.3 * torch.randn(d["static"].shape, device="cuda", generator=gen)
    kw = dict(target=d["y"], baselines=(x0, st0), n_samples=M, seed=B, internal_batch_size=7 * B)
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    if window is None:
        cells = torch.arange(N, device="cuda").view(1, 1, N).expand(T, B, N)
        got = _cat(*A.kernel_shap(*args, **kw))
    else:
        cells, _ = A.time_window_mask(d["times"], window, n_windows=6, sensor_groups=N)
        got = _cat(*A.kernel_shap(*args, feature_mask=cells, **kw))
    P = got.shape[1]
    if window is not None:
        assert P == 205, P
    Z, w = A.sample_coalitions(P, M, seed=B)
    ref = _loop_kernel_shap(model, d, cells, Z, w, d["y"], x0, st0)
    e = normwise(got, ref)
    print(cfg_name, B, P, M, e)
    assert e < 1e-6, e
    assert torch.count_nonzero(got) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
def test_efficiency(mode):
    """The default budget (2P + 2048 coalitions): sum_g phi + phi_static = F(x) - F(x') to 1e-6 of max|F|."""
    cfg = model_config("P19", dropout=0.2)
    d = to_dev(make_batch(cfg, 16, seed=21))
    model = _model(cfg, 6, mode)
    phi, phi_st, delta = A.kernel_shap(model, d["src"], d["static"], d["times"], d["lengths"],
                                       return_convergence_delta=True)
    P = cfg["d_inp"] + 1
    assert model._plan._kshap[1][0].shape == (2 * P + 2048, P)
    with torch.no_grad():
        fmax = float(model.forward(d["src"], d["static"], d["times"], d["lengths"])[0].abs().max())
    print("efficiency residual / max|F|:", float(delta.abs().max()) / fmax)
    assert float(delta.abs().max()) < 1e-6 * fmax
    assert torch.count_nonzero(phi) > 0 and torch.count_nonzero(phi_st) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
def test_players_without_cells_get_zero(mode):
    """Exhaustive coalitions: a player with no cell (an unused id of the map) and a sensor whose values equal their
    baseline get 0 up to the rounding of the fp64 solve (1e-9 of the largest attribution); the others do not."""
    cfg = model_config("TINY", dropout=0.2)
    B = 4
    d = to_dev(make_batch(cfg, B, seed=5, zero_sensors=1))
    model = _model(cfg, 3, mode)
    T, N = cfg["max_len"], cfg["d_inp"]
    cells = torch.as_tensor(np.broadcast_to(np.array([0, 1, 2, 4, 5])[:N], (T, N)).copy())   # id 3 names no cell
    G = int(cells.max()) + 1
    dummy_sensor = (d["src"][:, :, :N] == 0).all(dim=0)                                       # [B, N]
    assert dummy_sensor.any()
    phi, phi_st = A.kernel_shap(model, d["src"], d["static"], d["times"], d["lengths"], feature_mask=cells,
                                coalitions=A.all_coalitions(G + 1))
    scale = float(_cat(phi, phi_st).abs().max())
    assert float(phi[:, 3].abs().max()) < 1e-9 * scale
    ids = cells[0].cuda()
    for b in range(B):
        for n in torch.nonzero(dummy_sensor[b])[:, 0].tolist():
            assert float(phi[b, ids[n]].abs()) < 1e-9 * scale
    live = [g for g in range(G) if g != 3]
    assert torch.count_nonzero(phi[:, live]) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
def test_chunking_invariance(mode):
    """With the arithmetic mode pinned, one coalition per chunk, 7 per chunk (a ragged tail) and all in one chunk give
    bitwise-equal results, for sensor and time-window players."""
    cfg = model_config("P19", dropout=0.2)
    B, M = 8, 50
    d = to_dev(make_batch(cfg, B, seed=3))
    model = _model(cfg, 4, mode)
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    mask, _ = A.time_window_mask(d["times"], 12.0, sensor_groups=cfg["d_inp"])
    for kw in (dict(), dict(feature_mask=mask)):
        res = [_cat(*A.kernel_shap(*args, n_samples=M, internal_batch_size=ib, **kw)) for ib in (B, 7 * B, M * B)]
        for r in res[1:]:
            assert torch.equal(r, res[0]), normwise(r, res[0])


@pytest.mark.gpu
def test_targets_and_baselines():
    """target as an int, a tensor and None (argmax at x) agree; an explicit zero baseline pair equals the default; a
    nonzero baseline keeps efficiency."""
    cfg = model_config("P19", dropout=0.2)
    B = 5
    d = to_dev(make_batch(cfg, B, seed=8))
    model = _model(cfg, 2, EXACT)
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    fn = A.kernel_shap
    kw = dict(n_samples=200)
    a_int = fn(*args, target=1, **kw)
    a_vec = fn(*args, target=torch.ones(B, dtype=torch.int64, device="cuda"), **kw)
    assert torch.equal(a_int[0], a_vec[0]) and torch.equal(a_int[1], a_vec[1])
    with torch.no_grad():
        top = model.forward(d["src"], d["static"], d["times"], d["lengths"])[0].argmax(dim=1)
    a_none, a_top = fn(*args, target=None, **kw), fn(*args, target=top, **kw)
    assert torch.equal(a_none[0], a_top[0]) and torch.equal(a_none[1], a_top[1])
    a_zero = fn(*args, target=top, baselines=(0.0, torch.zeros(1, cfg["d_static"])), **kw)
    assert torch.equal(a_zero[0], a_top[0]) and torch.equal(a_zero[1], a_top[1])
    N = cfg["d_inp"]
    base = torch.full((1, 1, 2 * N), 0.3, device="cuda")
    _, _, delta = fn(*args, baselines=(base, None), return_convergence_delta=True, **kw)
    assert float(delta.abs().max()) < 1e-5
    one = fn(*args, sensor_groups=np.zeros(N, dtype=np.int64), target=top, baselines=(None, d["static"]), **kw)
    with torch.no_grad():     # the static player held fixed gets 0 up to rounding; P = 2 leaves the group F(x) - F(x')
        f1 = model.forward(d["src"], d["static"], d["times"], d["lengths"])[0]
        x = d["src"].clone()
        x[:, :, :N] = 0
        f0 = model.forward(x, d["static"], d["times"], d["lengths"])[0]
    df = (f1 - f0).gather(1, top[:, None])[:, 0]
    assert normwise(one[0][:, 0], df) < 1e-6 and float(one[1].abs().max()) < 1e-6 * float(df.abs().max())


@pytest.mark.gpu
def test_no_side_effects():
    """Parameters, their .grad, the dropout rng state and a bound FlatAdam (moments, step count, captured slots) are
    untouched; a model in training mode raises."""
    from raindrop_b200.optim import FlatAdam
    import torch.nn.functional as F
    cfg = model_config("P19", dropout=0.2)
    B = 16
    model = build_dropin(cfg, 8).train()
    opt = FlatAdam(model, lr=1e-3)
    for it in range(3):            # eager step, then CUDA-graph capture and replay
        d = to_dev(make_batch(cfg, B, seed=60 + it))
        logits, _, _ = model.forward(d["src"], d["static"], d["times"], d["lengths"])
        F.cross_entropy(logits, d["y"]).backward()
        opt.step()
    with pytest.raises(ValueError):
        A.kernel_shap(model, d["src"], d["static"], d["times"], d["lengths"])
    plan = model._plan
    slot = next(iter(plan._slots.values()))
    snap = {"flat_p": opt.flat_p.detach(), "flat_g": opt.flat_g, "exp_avg": opt.exp_avg, "exp_avg_sq": opt.exp_avg_sq,
            "step": opt.step_count, "rng": plan.rng_state, "slot.src": slot.src, "slot.logits": slot.logits}
    snap.update({"param." + k: p.detach() for k, p in model.named_parameters()})
    snap.update({"grad." + k: p.grad for k, p in model.named_parameters() if p.grad is not None})
    before = {k: v.clone() for k, v in snap.items()}
    model.eval()
    A.kernel_shap(model, d["src"], d["static"], d["times"], d["lengths"], n_samples=64)
    torch.cuda.synchronize()
    for k, v in snap.items():
        assert torch.equal(v, before[k]), k
    assert slot.fwd_graph is not None and slot.bwd_graph is not None
    model.train()
    logits, _, _ = model.forward(d["src"], d["static"], d["times"], d["lengths"])      # the captured step still runs
    F.cross_entropy(logits, d["y"]).backward()
    opt.step()


@pytest.mark.gpu
def test_cuda_graph_capture():
    """A CUDA-graph capture after an eager call with the same coalition set copies nothing and replays to the eager
    result, also after a later call has replaced both the cached coalition set and the scratch (more players and larger
    chunks): the buffers the graph reads stay held by the plan, so memory allocated after the replacement is not
    written by the replay."""
    cfg = model_config("P19", dropout=0.2)
    B = 8
    d = to_dev(make_batch(cfg, B, seed=11))
    model = _model(cfg, 5, 0)
    plan = model._plan
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    mask, _ = A.time_window_mask(d["times"], 12.0, sensor_groups=cfg["d_inp"])
    for i, kw in enumerate((dict(n_samples=60, sensor_groups=[i // 2 for i in range(cfg["d_inp"])],
                                 return_convergence_delta=True),
                            dict(n_samples=40, seed=2, feature_mask=mask.cpu()))):
        kw["internal_batch_size"] = 4 * B
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            eager = A.kernel_shap(*args, **kw)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        entry = plan._kshap
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = A.kernel_shap(*args, **kw)
        assert plan._kshap is entry
        scratch = plan._coal_attr_scratch[1]
        assert any(t is scratch for t in plan._scratch_captured)
        # a new coalition set, and chunks of 16 << i coalitions: a larger scratch replaces the captured one
        A.kernel_shap(*args, n_samples=40, seed=9, internal_batch_size=(16 << i) * B)
        assert plan._kshap is not entry and plan._coal_attr_scratch[1] is not scratch
        filler = torch.full_like(scratch, 7.0)
        for t in out:
            t.zero_()
        g.replay()
        torch.cuda.synchronize()
        for x, y in zip(out, eager):
            assert torch.equal(x, y)
        assert bool((filler == 7.0).all())
