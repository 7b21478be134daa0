"""Sensor-level Shapley-value sampling and leave-one-out ablation of Raindrop_v2 (raindrop_b200.attribution,
rd_raindrop_v2_coalition_attribution).  Reference values: tests/golden/sensor_attribution.npz, produced by the
reference's own files in eval mode with zero baselines (tools/make_sensor_attribution_golden.py): exact Shapley values by
subset enumeration for the TINY cases, ablation values for every case.  Tolerances follow test_integrated_gradients.py."""
import itertools
import json

import numpy as np
import pytest
import torch

from helpers import build_dropin, case_setup, load_golden, normwise, to_dev
from raindrop_b200 import attribution as A
from raindrop_b200.synth import make_batch, model_config, synth_weights

EXACT, FAST = 2, 1
TOL_EXACT, TOL_EXACT_WIDE, TOL_FAST = 2e-3, 1e-2, 2e-2
SHAPLEY = ["tiny_dense", "tiny_t0", "tiny_sparse", "tiny8_nostatic"]
ABLATION_ONLY = ["p19_b5_leave10", "p12_b2", "pam_b2"]


def _exact_tol(cfg):
    return TOL_EXACT_WIDE if cfg["max_len"] * cfg["d_ob"] >= 1024 else TOL_EXACT


def _fixture(golden_dir):
    z = np.load(golden_dir + "/sensor_attribution.npz")
    return z, json.loads(bytes(z["meta"]).decode())


def _all_orders(P):
    return np.array(list(itertools.permutations(range(P))), dtype=np.int64)


def _removed(src, static, groups, keep, x0=None, st0=None):
    """The input whose players outside `keep` ([P] bool; sensor groups `groups` [N], then the static player) are
    replaced by the baselines (default zeros); the mask half is untouched."""
    N = src.shape[2] // 2
    k = torch.as_tensor(np.asarray(keep)[np.asarray(groups)], device=src.device)
    x = src.clone()
    base = torch.zeros_like(src[:, :, :N]) if x0 is None else x0[:, :, :N]
    x[:, :, :N] = torch.where(k, src[:, :, :N], base)
    st = None
    if static is not None:
        st = static if keep[-1] else (torch.zeros_like(static) if st0 is None else st0)
    return x, st


class Game:
    """v(S) for one batch through a forward (module or oracle), each coalition evaluated once, in fp64 [B]."""

    def __init__(self, forward, d, groups, target, x0=None, st0=None):
        self.forward, self.d, self.groups, self.target, self.x0, self.st0 = forward, d, groups, target, x0, st0
        self.memo = {}

    def __call__(self, keep):
        key = tuple(bool(k) for k in keep)
        if key not in self.memo:
            x, st = _removed(self.d["src"], self.d["static"], self.groups, key, self.x0, self.st0)
            with torch.no_grad():
                logits = self.forward(x, st, self.d["times"], self.d["lengths"])
            self.memo[key] = logits.gather(1, self.target[:, None])[:, 0].double().cpu()
        return self.memo[key]


def shapley_by_permutations(game, P, orders):
    """(1/m) sum_p [v(S_pg + g) - v(S_pg)], host fp64: [B, P]."""
    phi = None
    for p in orders:
        keep = np.zeros(P, dtype=bool)
        prev = game(keep)
        for g in p:
            keep[g] = True
            cur = game(keep)
            phi = torch.zeros(cur.shape[0], P, dtype=torch.float64) if phi is None else phi
            phi[:, g] += cur - prev
            prev = cur
    return phi / len(orders)


def ablation_by_loop(game, P):
    full = game(np.ones(P, dtype=bool))
    return torch.stack([full - game(np.arange(P) != g) for g in range(P)], dim=1)


# ---- CPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SHAPLEY)
def test_oracle_reproduces_sensor_attribution_fixture(golden_dir, name):
    """The CPU oracle, averaging over all P! permutations, reproduces the reference's subset-enumeration Shapley values;
    its leave-one-out values reproduce the ablation fixture (TINY shapes)."""
    from oracle.raindrop_oracle import build_oracle_model
    z, meta = _fixture(golden_dir)
    _, gm = load_golden(golden_dir, name)
    cfg, batch = case_setup(gm)
    oracle = build_oracle_model(cfg).eval()
    synth_weights(oracle, cfg, seed=gm["weight_seed"])

    def fwd(s, st, t, ln):
        return oracle.forward_dense(s, st, t, ln)[0]
    target = torch.from_numpy(z[name + ".target"])
    N = cfg["d_inp"]
    P = N + (1 if cfg["static"] else 0)
    game = Game(fwd, batch, np.arange(N), target)
    phi = shapley_by_permutations(game, P, _all_orders(P))
    assert normwise(phi, z[name + ".shapley"]) < 1e-4, normwise(phi, z[name + ".shapley"])
    assert normwise(ablation_by_loop(game, P), z[name + ".ablation"]) < 1e-4
    ends = torch.from_numpy(z[name + ".endpoint_logits"])
    f = ends.gather(2, target.view(1, -1, 1).expand(2, -1, 1))[:, :, 0].double()
    assert float((phi.sum(dim=1) - (f[1] - f[0])).abs().max()) < 1e-5 * float(ends.abs().max())
    if name == "tiny_t0":                          # target None: the argmax class at x
        assert torch.equal(target, ends[1].argmax(dim=1))
    if name in meta["groups"]:
        groups = np.asarray(meta["groups"][name])
        Pg = int(groups.max()) + 2
        phi_g = shapley_by_permutations(Game(fwd, batch, groups, target), Pg, _all_orders(Pg))
        assert normwise(phi_g, z[name + ".shapley_grouped"]) < 1e-4


def test_sample_permutations_follow_the_seed():
    a = A.sample_permutations(35, 25, seed=3)
    assert a.shape == (25, 35) and a.dtype == np.int64
    np.testing.assert_array_equal(a, A.sample_permutations(35, 25, seed=3))
    assert not np.array_equal(a, A.sample_permutations(35, 25, seed=4))
    np.testing.assert_array_equal(np.sort(a, axis=1), np.broadcast_to(np.arange(35), a.shape))
    rng = np.random.default_rng(3)
    np.testing.assert_array_equal(a[0], rng.permutation(35))


def test_shapley_and_ablation_rankings_feed_removal_indices():
    from raindrop_b200.data import removal_indices
    B, N = 4, 6
    g = torch.Generator().manual_seed(0)
    phi = torch.randn(B, N, generator=g)
    phi[:, 3] = 0                                  # a dummy sensor ranks last
    imp = phi.abs().mean(dim=0)
    r = A.sensor_ranking(imp)
    idx = r[:, 0].astype(int)
    assert idx[-1] == 3 and sorted(idx.tolist()) == list(range(N))
    assert np.all(np.diff(imp.numpy()[idx]) <= 0)
    np.testing.assert_array_equal(removal_indices(B, N, 0.5, level="set", density_scores=r[:, 0]), idx[:3])


def _cpu_model(train=False):
    cfg = model_config("TINY", dropout=0.2)
    return build_dropin(cfg, 3, device="cpu").train(train), make_batch(cfg, 3, seed=1)


@pytest.mark.parametrize("fn", [A.feature_ablation, A.shapley_value_sampling])
def test_argument_validation(fn):
    model, b = _cpu_model()
    args = (b["src"], b["static"], b["times"], b["lengths"])
    with pytest.raises(TypeError):
        fn(torch.nn.Linear(2, 2), *args)
    with pytest.raises(ValueError, match="eval"):
        fn(model.train(), *args)
    model.eval()
    bad = [dict(target=2), dict(target=torch.tensor([0, 1, -1])), dict(target=torch.tensor([0, 1])),
           dict(target=torch.zeros(3)), dict(baselines=torch.zeros(1)),
           dict(sensor_groups=[0, 1, 2]), dict(sensor_groups=[0, 0, 2, 2, 1, 1]), dict(sensor_groups=[0, 0, 2, 2, 2]),
           dict(sensor_groups=[0, -1, 1, 1, 1]), dict(sensor_groups=np.zeros(5, dtype=np.float32)),
           dict(internal_batch_size=0)]
    if fn is A.shapley_value_sampling:
        bad += [dict(n_samples=0), dict(permutations=np.arange(5)[None]), dict(permutations=np.zeros((2, 6))),
                dict(permutations=np.array([[0, 1, 2, 3, 4, 5], [0, 1, 2, 3, 5, 5]])), dict(permutations=np.zeros((0, 6)))]
    for kw in bad:
        with pytest.raises(ValueError):
            fn(model, *args, **kw)
    with pytest.raises(ValueError):
        fn(model, b["src"][:, :, :3], b["static"], b["times"], b["lengths"])


@pytest.mark.parametrize("fn", [A.feature_ablation, A.shapley_value_sampling])
def test_no_cuda_raises(monkeypatch, fn):
    from raindrop_b200.lib import RaindropB200Error
    model, b = _cpu_model()
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RaindropB200Error):
        fn(model, b["src"], b["static"], b["times"], b["lengths"], target=1)


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _model(cfg, wseed, mode):
    m = build_dropin(cfg, wseed).eval()
    m._plan.obprop_mode = mode
    return m


def _module_forward(model):
    def fwd(s, st, t, ln):
        return model.forward(s, st, t, ln)[0]
    return fwd


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
@pytest.mark.parametrize("name", SHAPLEY + ABLATION_ONLY)
def test_golden_sensor_attribution(golden_dir, name, mode):
    """Exact Shapley values on the device from all P! permutations (TINY: 6! = 720; tiny_dense also over sensor groups)
    and ablation values for every case, against the reference's fixture."""
    z, meta = _fixture(golden_dir)
    _, gm = load_golden(golden_dir, name)
    cfg, batch = case_setup(gm)
    d = to_dev(batch)
    model = _model(cfg, gm["weight_seed"], mode)
    tgt = torch.from_numpy(z[name + ".target"]).cuda()
    target = None if gm["case"] == "tiny_t0" else tgt
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    tol = _exact_tol(cfg) if mode == EXACT else TOL_FAST
    ref = z[name + ".ablation"]
    a_s, a_st = A.feature_ablation(*args, target=target)
    errs = {"ablation": normwise(_cat(a_s, a_st), ref)}
    if name in SHAPLEY:
        P = ref.shape[1]
        phi, phi_st, delta = A.shapley_value_sampling(*args, target=target, permutations=_all_orders(P),
                                                      return_convergence_delta=True)
        errs["shapley"] = normwise(_cat(phi, phi_st), z[name + ".shapley"])
        errs["delta"] = float(delta.abs().max()) / float(np.abs(z[name + ".endpoint_logits"]).max())
        if name in meta["groups"]:
            groups = meta["groups"][name]
            Pg = max(groups) + 2
            phi, phi_st = A.shapley_value_sampling(*args, target=target, sensor_groups=groups,
                                                   permutations=_all_orders(Pg))
            errs["shapley_grouped"] = normwise(_cat(phi, phi_st), z[name + ".shapley_grouped"])
    print(name, mode, errs)
    assert max(errs.values()) < tol, errs


def _cat(a_sensors, a_static):
    return a_sensors if a_static is None else torch.cat([a_sensors, a_static[:, None]], dim=1)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name,B,opts", [("P19", 6, {"zero_sensors": 10}), ("P19", 1, {}), ("P19", 7, {"first_time_zero": True}),
                                             ("TINY8", 5, {}), ("P12", 3, {}), ("PAM", 2, {})])
def test_equals_module_loop(cfg_name, B, opts):
    """Exact mode: the device call equals the hand-written loop of B-row module forwards over the same coalition inputs
    with host-side fp64 sums (shapes: B = 1, odd B, no statics, the P12 and PAM (T > 64 attention) shapes)."""
    cfg = model_config(cfg_name, dropout=0.2)
    d = to_dev(make_batch(cfg, B, seed=70 + B, **opts))
    model = _model(cfg, 9, EXACT)
    N = cfg["d_inp"]
    P = N + (1 if cfg["static"] else 0)
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    game = Game(_module_forward(model), d, np.arange(N), d["y"])
    orders = A.sample_permutations(P, 2, seed=B)
    phi = _cat(*A.shapley_value_sampling(*args, target=d["y"], n_samples=2, seed=B, internal_batch_size=5 * B))
    abl = _cat(*A.feature_ablation(*args, target=d["y"], internal_batch_size=4 * B))
    e = {"shapley": normwise(phi, shapley_by_permutations(game, P, orders)), "ablation": normwise(abl, ablation_by_loop(game, P))}
    print(cfg_name, B, e)
    assert max(e.values()) < 1e-6, e
    assert torch.count_nonzero(phi) > 0 and torch.count_nonzero(abl) > 0


@pytest.mark.gpu
def test_efficiency():
    """Sampled permutations: sum_g phi + phi_static = F(x) - F(x') to 1e-6 of max|F| for every sample."""
    cfg = model_config("P19", dropout=0.2)
    d = to_dev(make_batch(cfg, 16, seed=21))
    model = _model(cfg, 6, 0)
    phi, phi_st, delta = A.shapley_value_sampling(model, d["src"], d["static"], d["times"], d["lengths"], n_samples=5,
                                                  seed=1, return_convergence_delta=True)
    with torch.no_grad():
        fmax = float(model.forward(d["src"], d["static"], d["times"], d["lengths"])[0].abs().max())
    total = phi.double().sum(dim=1) + phi_st.double()
    print("efficiency residual / max|F|:", float(delta.abs().max()) / fmax)
    assert float(delta.abs().max()) < 1e-6 * fmax
    assert torch.count_nonzero(total) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
@pytest.mark.parametrize("cfg_name,B,k", [("P19", 6, 10), ("TINY", 3, 2)])
def test_dummy_players_get_exact_zeros(cfg_name, B, k, mode):
    """A sensor whose values are all 0, with a zero baseline, changes no input bit when removed: both methods give it
    exactly 0, and so they do to the static player when its baseline equals `static`."""
    cfg = model_config(cfg_name, dropout=0.2)
    d = to_dev(make_batch(cfg, B, seed=5, zero_sensors=k))
    model = _model(cfg, 3, mode)
    N = cfg["d_inp"]
    dummy = (d["src"][:, :, :N] == 0).all(dim=0)                           # [B, N]
    assert dummy.sum(dim=1).min() >= k
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    base = (None, d["static"])
    for a_s, a_st in (A.feature_ablation(*args, baselines=base),
                      A.shapley_value_sampling(*args, baselines=base, n_samples=4)):
        bits = a_s.view(torch.int32)
        assert torch.all(bits[dummy] == 0)
        assert torch.all(a_st.view(torch.int32) == 0)
        assert torch.count_nonzero(a_s[~dummy]) > 0


@pytest.mark.gpu
def test_groups_closed_forms():
    """One group holding every sensor plus the static player (P = 2, both orders) equals the closed form from four
    forwards; P = 1 (one group, no statics) returns F(x) - F(x') from the endpoint forward alone."""
    from raindrop_b200 import lib as L
    cfg = model_config("P19", dropout=0.2)
    d = to_dev(make_batch(cfg, 5, seed=9))
    model = _model(cfg, 2, EXACT)
    N = cfg["d_inp"]
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    game = Game(_module_forward(model), d, np.zeros(N, dtype=np.int64), d["y"])
    v = {k: game(np.array(k)) for k in itertools.product([False, True], repeat=2)}
    closed = torch.stack([0.5 * ((v[True, False] - v[False, False]) + (v[True, True] - v[False, True])),
                          0.5 * ((v[False, True] - v[False, False]) + (v[True, True] - v[True, False]))], dim=1)
    phi = _cat(*A.shapley_value_sampling(*args, target=d["y"], sensor_groups=np.zeros(N, dtype=np.int64),
                                         permutations=[[0, 1], [1, 0]]))
    abl = _cat(*A.feature_ablation(*args, target=d["y"], sensor_groups=torch.zeros(N, dtype=torch.int64)))
    e = {"shapley": normwise(phi, closed),
         "ablation": normwise(abl, torch.stack([v[True, True] - v[False, True], v[True, True] - v[True, False]], dim=1))}
    assert max(e.values()) < 1e-6, e

    cfg8 = model_config("TINY8", dropout=0.2)
    d8 = to_dev(make_batch(cfg8, 4, seed=10))
    m8 = _model(cfg8, 4, EXACT)
    args8 = (m8, d8["src"], None, d8["times"], d8["lengths"])
    g8 = Game(_module_forward(m8), d8, np.zeros(cfg8["d_inp"], dtype=np.int64), d8["y"])
    lib = L.load()
    counts = []
    A.shapley_value_sampling(*args8, sensor_groups=[0] * cfg8["d_inp"], n_samples=1)     # the graph prologue runs once
    for m in (1, 50):
        torch.cuda.synchronize()
        n0 = lib.rd_launch_count()
        phi, phi_st = A.shapley_value_sampling(*args8, target=d8["y"], sensor_groups=[0] * cfg8["d_inp"], n_samples=m)
        torch.cuda.synchronize()
        counts.append(lib.rd_launch_count() - n0)
        assert phi.shape == (4, 1) and phi_st is None
        assert normwise(phi[:, 0], g8(np.array([True])) - g8(np.array([False]))) < 1e-6
    assert counts[0] == counts[1], counts                  # no coalition forward, whatever m


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
def test_chunking_invariance(mode):
    """With the arithmetic mode pinned, one coalition per chunk, 7 per chunk (a ragged tail) and all in one chunk give
    bitwise-equal results: the fp64 running sums add the same values in the same order."""
    cfg = model_config("P19", dropout=0.2)
    B = 8
    d = to_dev(make_batch(cfg, B, seed=3))
    model = _model(cfg, 4, mode)
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    n_coal = 3 * 34
    for fn, kw, n in ((A.shapley_value_sampling, dict(n_samples=3), n_coal), (A.feature_ablation, {}, 35)):
        res = [_cat(*fn(*args, internal_batch_size=ib, **kw)) for ib in (B, 7 * B, n * B)]
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
    for fn in (A.feature_ablation, A.shapley_value_sampling):
        a_int = fn(*args, target=1)
        a_vec = fn(*args, target=torch.ones(B, dtype=torch.int64, device="cuda"))
        assert torch.equal(a_int[0], a_vec[0]) and torch.equal(a_int[1], a_vec[1])
        with torch.no_grad():
            top = model.forward(d["src"], d["static"], d["times"], d["lengths"])[0].argmax(dim=1)
        a_none, a_top = fn(*args, target=None), fn(*args, target=top)
        assert torch.equal(a_none[0], a_top[0]) and torch.equal(a_none[1], a_top[1])
        a_zero = fn(*args, target=top, baselines=(0.0, torch.zeros(1, cfg["d_static"])))
        assert torch.equal(a_zero[0], a_top[0]) and torch.equal(a_zero[1], a_top[1])
    N = cfg["d_inp"]
    base = torch.full((1, 1, 2 * N), 0.3, device="cuda")
    _, _, delta = A.shapley_value_sampling(*args, baselines=(base, None), return_convergence_delta=True)
    assert float(delta.abs().max()) < 1e-5


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
    for fn in (A.feature_ablation, A.shapley_value_sampling):
        with pytest.raises(ValueError):
            fn(model, d["src"], d["static"], d["times"], d["lengths"])
    plan = model._plan
    slot = next(iter(plan._slots.values()))
    snap = {"flat_p": opt.flat_p.detach(), "flat_g": opt.flat_g, "exp_avg": opt.exp_avg, "exp_avg_sq": opt.exp_avg_sq,
            "step": opt.step_count, "rng": plan.rng_state, "slot.src": slot.src, "slot.logits": slot.logits}
    snap.update({"param." + k: p.detach() for k, p in model.named_parameters()})
    snap.update({"grad." + k: p.grad for k, p in model.named_parameters() if p.grad is not None})
    before = {k: v.clone() for k, v in snap.items()}
    model.eval()
    A.feature_ablation(model, d["src"], d["static"], d["times"], d["lengths"])
    A.shapley_value_sampling(model, d["src"], d["static"], d["times"], d["lengths"], n_samples=2)
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
    """A CUDA-graph capture of each call, replayed, reproduces the eager result."""
    cfg = model_config("P19", dropout=0.2)
    B = 8
    d = to_dev(make_batch(cfg, B, seed=11))
    model = _model(cfg, 5, 0)
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    groups = [i // 2 for i in range(cfg["d_inp"])]
    for fn, kw in ((A.shapley_value_sampling, dict(n_samples=3, sensor_groups=groups, internal_batch_size=4 * B,
                                                   return_convergence_delta=True)),
                   (A.feature_ablation, dict(internal_batch_size=4 * B))):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            eager = fn(*args, **kw)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = fn(*args, **kw)
        for t in out:
            t.zero_()
        g.replay()
        torch.cuda.synchronize()
        for x, y in zip(out, eager):
            assert torch.equal(x, y)
