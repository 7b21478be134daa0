"""Shapley-value sampling and leave-one-out ablation of Raindrop_v2 over players of a map of the value cells
(raindrop_b200.attribution feature_mask, time_window_mask; rd_raindrop_v2_cell_coalition_attribution).  Reference
values: tests/golden/cell_attribution.npz, produced by the reference's own files in eval mode with zero baselines
(tools/make_cell_attribution_golden.py): exact Shapley values by subset enumeration for two TINY cases ([T, N] and
per-sample maps), ablation values for the P19, P12 and PAM shapes with per-sample time-window maps.  Tolerances follow
test_sensor_attribution.py."""
import itertools
import json

import numpy as np
import pytest
import torch

from helpers import build_dropin, case_setup, load_golden, normwise, to_dev
from raindrop_b200 import attribution as A
from raindrop_b200.synth import make_batch, model_config

EXACT, FAST = 2, 1
TOL_EXACT, TOL_EXACT_WIDE, TOL_FAST = 2e-3, 1e-2, 2e-2
SHAPLEY = ["tiny_dense", "tiny_t0"]
ABLATION_ONLY = ["p19_b5_leave10", "p12_b2", "pam_b2"]


def _exact_tol(cfg):
    return TOL_EXACT_WIDE if cfg["max_len"] * cfg["d_ob"] >= 1024 else TOL_EXACT


def _fixture(golden_dir):
    z = np.load(golden_dir + "/cell_attribution.npz")
    return z, json.loads(bytes(z["meta"]).decode())


def _all_orders(P):
    return np.array(list(itertools.permutations(range(P))), dtype=np.int64)


def _case_mask(z, meta, name, times):
    """The case's map as the API takes it: [T, N] for tiny_dense, else time_window_mask rebuilt from the meta (checked
    against the stored map)."""
    cells = z[name + ".cells"]
    mp = meta["maps"][name]
    if mp["kind"] == "[T, N]":
        return torch.from_numpy(cells[:, 0, :].copy())
    mask, n_win = A.time_window_mask(times, mp["window"], n_windows=mp["n_windows"], sensor_groups=mp["groups"])
    assert n_win == mp["n_windows"]
    np.testing.assert_array_equal(mask.cpu().numpy(), cells)
    return mask


def _removed(src, static, cells, keep, x0=None, st0=None):
    """The input whose players outside `keep` ([P] bool; ids of `cells` [T, B, N] or [T, N], then the static player)
    are replaced by the baselines (default zeros); cells with id -1 and the mask half are untouched."""
    N = src.shape[2] // 2
    keep = np.asarray(keep, dtype=bool)
    cells = torch.as_tensor(cells, device=src.device).long()
    G = int(cells.max()) + 1
    kx = torch.as_tensor(np.append(keep[:G], True), device=src.device)           # id -1 -> the appended True
    k = kx[cells]
    if k.dim() == 2:
        k = k[:, None, :]
    x = src.clone()
    base = torch.zeros_like(src[:, :, :N]) if x0 is None else x0[:, :, :N]
    x[:, :, :N] = torch.where(k, src[:, :, :N], base)
    st = None
    if static is not None:
        st = static if keep[-1] else (torch.zeros_like(static) if st0 is None else st0)
    return x, st


class Game:
    """v(S) for one batch through a forward (module or oracle), each coalition evaluated once, in fp64 [B]."""

    def __init__(self, forward, d, cells, target, x0=None, st0=None):
        self.forward, self.d, self.cells, self.target, self.x0, self.st0 = forward, d, cells, target, x0, st0
        self.memo = {}

    def __call__(self, keep):
        key = tuple(bool(k) for k in keep)
        if key not in self.memo:
            x, st = _removed(self.d["src"], self.d["static"], self.cells, key, self.x0, self.st0)
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


def _cat(a_players, a_static):
    return a_players if a_static is None else torch.cat([a_players, a_static[:, None]], dim=1)


# ---- CPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SHAPLEY)
def test_oracle_reproduces_cell_attribution_fixture(golden_dir, name):
    """The CPU oracle, averaging over all 7! permutations of (window, group) players plus the static player, reproduces
    the reference's subset-enumeration Shapley values; its leave-one-out values reproduce the ablation fixture."""
    from oracle.raindrop_oracle import build_oracle_model
    z, meta = _fixture(golden_dir)
    _, gm = load_golden(golden_dir, name)
    cfg, batch = case_setup(gm)
    oracle = build_oracle_model(cfg).eval()
    from raindrop_b200.synth import synth_weights
    synth_weights(oracle, cfg, seed=gm["weight_seed"])

    def fwd(s, st, t, ln):
        return oracle.forward_dense(s, st, t, ln)[0]
    target = torch.from_numpy(z[name + ".target"])
    cells = _case_mask(z, meta, name, batch["times"])
    P = int(cells.max()) + 2
    assert P == z[name + ".shapley"].shape[1] == 7
    game = Game(fwd, batch, cells, target)
    phi = shapley_by_permutations(game, P, _all_orders(P))
    assert normwise(phi, z[name + ".shapley"]) < 1e-4, normwise(phi, z[name + ".shapley"])
    assert normwise(ablation_by_loop(game, P), z[name + ".ablation"]) < 1e-4
    ends = torch.from_numpy(z[name + ".endpoint_logits"])
    f = ends.gather(2, target.view(1, -1, 1).expand(2, -1, 1))[:, :, 0].double()
    assert float((phi.sum(dim=1) - (f[1] - f[0])).abs().max()) < 1e-5 * float(ends.abs().max())
    if name == "tiny_t0":                          # target None: the argmax class at x; padding rows carry -1
        assert torch.equal(target, ends[1].argmax(dim=1))
        assert (z[name + ".cells"] == -1).any()


def test_fixture_maps_are_time_window_masks(golden_dir):
    """Every per-sample map of the fixture is what time_window_mask gives for the case's times."""
    z, meta = _fixture(golden_dir)
    for name in SHAPLEY + ABLATION_ONLY:
        _, gm = load_golden(golden_dir, name)
        _, batch = case_setup(gm)
        _case_mask(z, meta, name, batch["times"])


def test_time_window_mask_bins_clamping_and_padding():
    """w = min(floor(t / window), n_windows - 1), id = w*G + g; rows t > 0 with time 0 are padding (-1); row 0 is real
    even when its time is 0 (first_time_zero data); n_windows defaults to max(1, ceil(max(times) / window))."""
    times = torch.tensor([[0.0, 0.0, 1.0],
                          [2.9, 3.0, 2.0],
                          [3.0, 0.0, 8.5],
                          [9.0, 0.0, 0.0]])                             # [T=4, B=3]
    groups = [0, 1, 1]
    mask, n_win = A.time_window_mask(times, 3.0, sensor_groups=groups)
    assert n_win == 3 and mask.dtype == torch.int32 and mask.shape == (4, 3, 3)
    w = torch.tensor([[0, 0, 0], [0, 1, 0], [1, -1, 2], [2, -1, -1]])
    g = torch.tensor(groups)
    expect = torch.where(w[:, :, None] >= 0, w[:, :, None] * 2 + g, -1)
    assert torch.equal(mask.long(), expect)
    mask2, n2 = A.time_window_mask(times, 3.0, n_windows=2, sensor_groups=groups)          # clamped into window 1
    assert n2 == 2 and int(mask2.max()) == 3 and torch.equal(mask2.long(), torch.where(expect >= 4, expect - 2, expect))
    m1, n1 = A.time_window_mask(torch.zeros(3, 2), 1.0, sensor_groups=4)                   # all zero: row 0 real
    assert n1 == 1 and torch.equal(m1[0].long(), torch.arange(4).expand(2, 4)) and bool((m1[1:] == -1).all())
    cfg = model_config("P12")
    b = make_batch(cfg, 4, seed=3, first_time_zero=True)
    assert float(b["times"][0].abs().max()) == 0.0
    mask, n_win = A.time_window_mask(b["times"], 40.0, sensor_groups=cfg["d_inp"])
    assert n_win == int(np.ceil(float(b["times"].max()) / 40.0))
    assert bool((mask[0] >= 0).all()) and bool((mask[0] < cfg["d_inp"]).all())
    pad = (b["times"] == 0) & (torch.arange(cfg["max_len"])[:, None] > 0)
    assert bool((mask[pad] == -1).all()) and bool((mask[~pad] >= 0).all())
    t = b["times"].double()
    w = torch.clamp(torch.floor(t / 40.0), max=n_win - 1).long()
    assert torch.equal(mask[~pad].long(), (w[:, :, None] * cfg["d_inp"] + torch.arange(cfg["d_inp"]))[~pad])


def _cpu_model(train=False):
    cfg = model_config("TINY", dropout=0.2)
    return build_dropin(cfg, 3, device="cpu").train(train), make_batch(cfg, 3, seed=1), cfg


@pytest.mark.parametrize("fn", [A.feature_ablation, A.shapley_value_sampling])
def test_argument_validation(fn):
    model, b, cfg = _cpu_model()
    model.eval()
    T, N = cfg["max_len"], cfg["d_inp"]
    args = (model, b["src"], b["static"], b["times"], b["lengths"])
    good = np.zeros((T, N), dtype=np.int64)
    bad = [dict(feature_mask=good, sensor_groups=np.arange(N)), dict(feature_mask=good.astype(np.float32)),
           dict(feature_mask=good.astype(bool)), dict(feature_mask=np.zeros((T, 2, N), dtype=np.int64)),
           dict(feature_mask=np.zeros((N,), dtype=np.int64)), dict(feature_mask=np.zeros((T, 3, N, 1), dtype=np.int64)),
           dict(feature_mask=good - 2), dict(feature_mask=good - 1)]
    for kw in bad:
        with pytest.raises(ValueError):
            fn(*args, **kw)
    with pytest.raises(ValueError, match="max_len"):
        fn(*args, feature_mask=np.zeros((T + 1, N), dtype=np.int64))
    with pytest.raises(ValueError):
        A.time_window_mask(b["times"], 0.0, sensor_groups=N)
    with pytest.raises(ValueError):
        A.time_window_mask(b["times"], 1.0)
    with pytest.raises(ValueError):
        A.time_window_mask(b["times"], 1.0, n_windows=0, sensor_groups=N)
    with pytest.raises(ValueError):
        A.time_window_mask(b["times"], 1.0, sensor_groups=[0, 2, 2, 2, 2])                  # group 1 empty
    with pytest.raises(ValueError):
        A.time_window_mask(b["times"][:, 0], 1.0, sensor_groups=N)


def test_host_mask_cache_holds_one_mask():
    """The per-plan cache of host feature masks holds one entry: a mask of other content replaces it, the same mask
    reuses it (no copy)."""
    import types
    plan = types.SimpleNamespace()
    dev = torch.device("cpu")
    masks = [np.full((6, 4, 3), i, dtype=np.int32) for i in range(20)]
    for m in masks:
        got = A._device_cells(plan, m, dev)
        np.testing.assert_array_equal(got.numpy(), m)
    assert plan._coal_cells[0][1] == masks[-1].tobytes()
    assert A._device_cells(plan, masks[-1].copy(), dev) is got
    assert not hasattr(plan, "_coal_cells_captured")


@pytest.mark.parametrize("fn", [A.feature_ablation, A.shapley_value_sampling])
def test_no_cuda_raises(monkeypatch, fn):
    from raindrop_b200.lib import RaindropB200Error
    model, b, cfg = _cpu_model()
    model.eval()
    mask, _ = A.time_window_mask(b["times"], 2.0, sensor_groups=cfg["d_inp"])
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RaindropB200Error):
        fn(model, b["src"], b["static"], b["times"], b["lengths"], target=1, feature_mask=mask)


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
def test_golden_cell_attribution(golden_dir, name, mode):
    """Exact Shapley values on the device from all 7! permutations (TINY, a [T, N] map and a per-sample time-window map
    with padding rows) and ablation values for every case, against the reference's fixture."""
    z, meta = _fixture(golden_dir)
    _, gm = load_golden(golden_dir, name)
    cfg, batch = case_setup(gm)
    d = to_dev(batch)
    model = _model(cfg, gm["weight_seed"], mode)
    tgt = torch.from_numpy(z[name + ".target"]).cuda()
    target = None if gm["case"] == "tiny_t0" else tgt
    mask = _case_mask(z, meta, name, d["times"])
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    tol = _exact_tol(cfg) if mode == EXACT else TOL_FAST
    ref = z[name + ".ablation"]
    a_p, a_st = A.feature_ablation(*args, target=target, feature_mask=mask)
    errs = {"ablation": normwise(_cat(a_p, a_st), ref)}
    if name in SHAPLEY:
        P = ref.shape[1]
        phi, phi_st, delta = A.shapley_value_sampling(*args, target=target, permutations=_all_orders(P),
                                                      return_convergence_delta=True, feature_mask=mask)
        errs["shapley"] = normwise(_cat(phi, phi_st), z[name + ".shapley"])
        errs["delta"] = float(delta.abs().max()) / float(np.abs(z[name + ".endpoint_logits"]).max())
    print(name, mode, errs)
    assert max(errs.values()) < tol, errs


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name,B", [("P19", 6), ("TINY8", 5)])
def test_equals_sensor_level_path_bitwise(cfg_name, B):
    """A [T, N] map that repeats sensor_groups over t, and the same as an expanded and as a materialised [T, B, N]
    map, give results bitwise equal to the sensor_groups call (both methods, sampled permutations)."""
    cfg = model_config(cfg_name, dropout=0.2)
    d = to_dev(make_batch(cfg, B, seed=31))
    model = _model(cfg, 3, 0)
    T, N = cfg["max_len"], cfg["d_inp"]
    groups = np.arange(N) // 2
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    rep = np.broadcast_to(groups, (T, N)).copy()
    maps = [rep, torch.as_tensor(rep, dtype=torch.int32, device="cuda")[:, None, :].expand(T, B, N),
            torch.as_tensor(rep, device="cuda")[:, None, :].expand(T, B, N).contiguous()]
    for fn, kw in ((A.shapley_value_sampling, dict(n_samples=3, seed=2)), (A.feature_ablation, {})):
        ref = fn(*args, target=d["y"], sensor_groups=groups, internal_batch_size=4 * B, **kw)
        for mp in maps:
            out = fn(*args, target=d["y"], feature_mask=mp, internal_batch_size=4 * B, **kw)
            for x, y in zip(out, ref):
                assert (x is None and y is None) or torch.equal(x, y), fn.__name__


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name,B,window,opts", [("P19", 5, 8.0, {"first_time_zero": True}), ("TINY8", 4, 1.5, {}),
                                                    ("P12", 2, 40.0, {"first_time_zero": True})])
def test_equals_module_loop(cfg_name, B, window, opts):
    """Exact mode, per-sample time-window map, nonzero baselines: sampled Shapley values and ablation equal the loop of
    B-row module forwards over the same coalition inputs with host-side fp64 sums; cells with id -1 keep x (a baseline
    that differs only there changes no bit of the result)."""
    cfg = model_config(cfg_name, dropout=0.2)
    d = to_dev(make_batch(cfg, B, seed=90 + B, **opts))
    model = _model(cfg, 9, EXACT)
    N = cfg["d_inp"]
    mask, n_win = A.time_window_mask(d["times"], window, sensor_groups=N)
    assert bool((mask == -1).any()) or cfg_name == "TINY8"
    P = n_win * N + (1 if cfg["static"] else 0)
    gen = torch.Generator(device="cuda").manual_seed(5)
    x0 = 0.5 * torch.randn(d["src"].shape, device="cuda", generator=gen)
    st0 = None if d["static"] is None else 0.5 * torch.randn(d["static"].shape, device="cuda", generator=gen)
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    game = Game(_module_forward(model), d, mask, d["y"], x0, st0)
    orders = A.sample_permutations(P, 2, seed=B)
    kw = dict(target=d["y"], baselines=(x0, st0), feature_mask=mask)
    phi = _cat(*A.shapley_value_sampling(*args, n_samples=2, seed=B, internal_batch_size=5 * B, **kw))
    abl = _cat(*A.feature_ablation(*args, internal_batch_size=4 * B, **kw))
    e = {"shapley": normwise(phi, shapley_by_permutations(game, P, orders)), "ablation": normwise(abl, ablation_by_loop(game, P))}
    print(cfg_name, B, P, e)
    assert max(e.values()) < 1e-7, e
    assert torch.count_nonzero(phi) > 0 and torch.count_nonzero(abl) > 0
    pad = torch.cat([mask == -1, torch.zeros_like(mask, dtype=torch.bool)], dim=2)       # value half of the -1 cells
    x0_pad = torch.where(pad, torch.full_like(x0, 7.0), x0)
    kw["baselines"] = (x0_pad, st0)
    assert torch.equal(phi, _cat(*A.shapley_value_sampling(*args, n_samples=2, seed=B, internal_batch_size=5 * B, **kw)))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
def test_efficiency_and_exact_zeros(mode):
    """Sum of the attributions = F(x) - F(x') to 1e-6 of max|F|; a player with no cell (an unused id, an empty window of
    a short sample) and a player whose cells equal their baseline get exactly 0 from both methods."""
    cfg = model_config("P19", dropout=0.2)
    B, N = 12, cfg["d_inp"]
    d = to_dev(make_batch(cfg, B, seed=21))
    model = _model(cfg, 6, mode)
    mask, n_win = A.time_window_mask(d["times"], 6.0, sensor_groups=N)
    mask = torch.where(mask >= N, mask + N, mask)                      # ids N..2N-1 name no cell in any sample
    G = (n_win + 1) * N
    m = mask.permute(1, 0, 2).reshape(B, -1).long()                   # [B, T*N]
    present = torch.zeros(B, G + 1, dtype=torch.bool, device="cuda")
    present = present.scatter_(1, torch.where(m >= 0, m, G), True)[:, :G]
    assert not bool(present[:, N:2 * N].any()) and bool((~present[:, 2 * N:]).any())   # + empty windows of short samples
    x0 = 0.3 * torch.ones_like(d["src"])
    same = mask == 2                                                    # player 2 (sensor 2, window 0): baseline = x
    x0[:, :, :N] = torch.where(same, d["src"][:, :, :N], x0[:, :, :N])
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    phi, phi_st, delta = A.shapley_value_sampling(*args, baselines=(x0, None), n_samples=4, seed=1,
                                                  return_convergence_delta=True, feature_mask=mask)
    abl, _ = A.feature_ablation(*args, baselines=(x0, None), feature_mask=mask)
    with torch.no_grad():
        fmax = float(model.forward(d["src"], d["static"], d["times"], d["lengths"])[0].abs().max())
    print("efficiency residual / max|F|:", float(delta.abs().max()) / fmax)
    assert float(delta.abs().max()) < 1e-6 * fmax
    for a in (phi, abl):
        assert a.shape == (B, G)
        bits = a.view(torch.int32)
        assert torch.all(bits[~present] == 0) and torch.all(bits[:, 2] == 0)
        assert torch.count_nonzero(a[present]) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
def test_chunking_invariance(mode):
    """With the arithmetic mode pinned, one coalition per chunk, 7 per chunk (a ragged tail) and all in one chunk give
    bitwise-equal results over a per-sample time-window map."""
    cfg = model_config("P19", dropout=0.2)
    B = 4
    d = to_dev(make_batch(cfg, B, seed=3))
    model = _model(cfg, 4, mode)
    mask, n_win = A.time_window_mask(d["times"], 12.0, sensor_groups=cfg["d_inp"])
    P = n_win * cfg["d_inp"] + 1
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    for fn, kw, n in ((A.shapley_value_sampling, dict(n_samples=2), 2 * (P - 1)), (A.feature_ablation, {}, P)):
        res = [_cat(*fn(*args, internal_batch_size=ib, feature_mask=mask, **kw)) for ib in (B, 7 * B, n * B)]
        for r in res[1:]:
            assert torch.equal(r, res[0]), normwise(r, res[0])


@pytest.mark.gpu
def test_no_side_effects():
    """Parameters, their .grad, the dropout rng state and a bound FlatAdam (moments, step count, captured slots) are
    untouched by calls with a feature mask."""
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
    mask, _ = A.time_window_mask(d["times"], 10.0, sensor_groups=cfg["d_inp"])
    for fn in (A.feature_ablation, A.shapley_value_sampling):
        with pytest.raises(ValueError):
            fn(model, d["src"], d["static"], d["times"], d["lengths"], feature_mask=mask)
    plan = model._plan
    slot = next(iter(plan._slots.values()))
    snap = {"flat_p": opt.flat_p.detach(), "flat_g": opt.flat_g, "exp_avg": opt.exp_avg, "exp_avg_sq": opt.exp_avg_sq,
            "step": opt.step_count, "rng": plan.rng_state, "slot.src": slot.src, "slot.logits": slot.logits}
    snap.update({"param." + k: p.detach() for k, p in model.named_parameters()})
    snap.update({"grad." + k: p.grad for k, p in model.named_parameters() if p.grad is not None})
    before = {k: v.clone() for k, v in snap.items()}
    model.eval()
    A.feature_ablation(model, d["src"], d["static"], d["times"], d["lengths"], feature_mask=mask)
    A.shapley_value_sampling(model, d["src"], d["static"], d["times"], d["lengths"], n_samples=2, feature_mask=mask)
    torch.cuda.synchronize()
    for k, v in snap.items():
        assert torch.equal(v, before[k]), k
    assert slot.fwd_graph is not None and slot.bwd_graph is not None
    model.train()
    logits, _, _ = model.forward(d["src"], d["static"], d["times"], d["lengths"])      # the captured step still runs
    F.cross_entropy(logits, d["y"]).backward()
    opt.step()


@pytest.mark.gpu
def test_per_batch_host_masks_hold_bounded_memory():
    """A loop of calls with a different host mask each time keeps one mask on the device, and a call with fewer players
    (a batch that does not reach the last window) reuses the scratch instead of reallocating it."""
    cfg = model_config("P19", dropout=0.2)
    B = 4
    model = _model(cfg, 5, 0)
    plan = model._plan
    ptrs, keys = [], []
    d = to_dev(make_batch(cfg, B, seed=40))
    for win in (6.0, 8.0, 10.0, 12.0, 7.0, 16.0):                 # the first window gives the most players
        mask, _ = A.time_window_mask(d["times"].cpu(), win, sensor_groups=cfg["d_inp"])
        A.feature_ablation(model, d["src"], d["static"], d["times"], d["lengths"], feature_mask=mask.numpy())
        ptrs.append(plan._coal_attr_scratch[1].data_ptr())
        keys.append(plan._coal_cells[0][1])
        assert isinstance(plan._coal_cells, tuple) and keys[-1] == mask.numpy().tobytes()
    assert len(set(keys)) == len(keys)
    assert len(set(ptrs)) == 1, ptrs
    assert not hasattr(plan, "_coal_cells_captured")


@pytest.mark.gpu
def test_cuda_graph_capture():
    """A CUDA-graph capture of each call with a host feature mask (cached on the device by the eager call), replayed,
    reproduces the eager result, also after a call with another mask has replaced the plan's cached mask."""
    cfg = model_config("P19", dropout=0.2)
    B = 8
    d = to_dev(make_batch(cfg, B, seed=11))
    model = _model(cfg, 5, 0)
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    mask, _ = A.time_window_mask(d["times"].cpu(), 10.0, sensor_groups=[i // 2 for i in range(cfg["d_inp"])])
    for fn, kw in ((A.shapley_value_sampling, dict(n_samples=2, internal_batch_size=4 * B, return_convergence_delta=True)),
                   (A.feature_ablation, dict(internal_batch_size=4 * B))):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            eager = fn(*args, feature_mask=mask.numpy(), **kw)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = fn(*args, feature_mask=mask.numpy(), **kw)
        for t in out:
            t.zero_()
        g.replay()
        torch.cuda.synchronize()
        for x, y in zip(out, eager):
            assert torch.equal(x, y)
        # a call with another host mask replaces the plan's cached mask; the graph still reads the one it captured
        # (wider windows: fewer players, so the call reuses the captured scratch)
        other, _ = A.time_window_mask(d["times"].cpu(), 20.0, sensor_groups=cfg["d_inp"])
        fn(*args, feature_mask=other.numpy(), **kw)
        assert model._plan._coal_cells[0][1] == other.numpy().tobytes()
        for t in out:
            t.zero_()
        g.replay()
        torch.cuda.synchronize()
        for x, y in zip(out, eager):
            assert torch.equal(x, y)
    assert len(model._plan._coal_cells_captured) == 2              # the mask copy read by each of the two graphs


@pytest.mark.gpu
def test_launches_do_not_grow_with_players():
    """An ablation call whose coalitions fit in one chunk makes the same launches for 35 players (one window) as for
    over a hundred (6-unit windows): the kept-player test of a cell is O(1) and costs no launch of its own."""
    from raindrop_b200 import lib as L
    cfg = model_config("P19", dropout=0.2)
    B = 4
    d = to_dev(make_batch(cfg, B, seed=12))
    model = _model(cfg, 5, 0)
    args = (model, d["src"], d["static"], d["times"], d["lengths"])
    lib = L.load()
    counts = []
    for win in (1e9, 6.0):
        mask, n_win = A.time_window_mask(d["times"], win, sensor_groups=cfg["d_inp"])
        P = n_win * cfg["d_inp"] + 1
        A.feature_ablation(*args, feature_mask=mask, internal_batch_size=P * B)               # warm
        torch.cuda.synchronize()
        n0 = lib.rd_launch_count()
        A.feature_ablation(*args, feature_mask=mask, internal_batch_size=P * B)
        torch.cuda.synchronize()
        counts.append((P, lib.rd_launch_count() - n0))
    print("players, launches:", counts)
    assert counts[1][0] > 100 and counts[0][1] == counts[1][1], counts
