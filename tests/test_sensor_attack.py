"""Worst-case sensor removal of Raindrop_v2 (raindrop_b200.sensor_attack, rd_raindrop_v2_sensor_attack).

CPU: the exported symbols, the scratch query, the host argument checks, and a numpy restatement of the search driven by
any logits function: against brute force over all subsets on the float64 oracle model, and on hand-built logits tables
with ties (the order, the deduplication, the success rule, the rows of the fixed round shapes).  GPU: greedy, beam and
exhaustive results against the restatement driven by the module's own forward on torch-built removed copies (bitwise),
a wide beam against exhaustive search, exhaustive against greedy, the targeted mode, y = None, remove_mask=False,
remove_static and a sensors subset, chunking, CUDA-graph replay without side effects, and the large shapes.  Every GPU
test pins plan.obprop_mode: the auto mode picks the ob-prop arithmetic from the row count."""
import ctypes as C
import itertools
import math
import os
import subprocess

import numpy as np
import pytest
import torch

from helpers import build_dropin, to_dev
from raindrop_b200 import sensor_attack as SA
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


# ---- numpy restatement ------------------------------------------------------------------------------------------------
def row_score(z, y, targeted):
    """(s, success) of logits z [C] against class y, in float32 as the device computes them."""
    z = np.asarray(z, np.float32)
    if not np.isfinite(z).all():
        return np.float32(np.inf), False
    other = np.max(np.delete(z, y))
    s = (other - z[y]) if targeted else (z[y] - other)
    arg = int(np.argmax(z))                             # the first maximum
    return np.float32(s), (arg == y) if targeted else (arg != y)


def first_argmax(z):
    z = np.asarray(z, np.float32)
    best, arg = z[0], 0
    for c in range(1, len(z)):
        if z[c] > best:
            best, arg = z[c], c
    return arg


def search(logits_fn, B, P, R, W, exhaustive, cls=None, targeted=False):
    """The search of the module docstring.  logits_fn(rows) -> float32 [len(rows), C] for rows [(b, sorted tuple of
    removed players)].  Returns dict(removed [B, P] bool, n_removed [B], logits [B, C], clean [B, C], score [B],
    best_score [B, R+1], beams: per round the list of beams, rows: per round the rows per sample)."""
    clean = np.asarray(logits_fn([(b, ()) for b in range(B)]), np.float32)
    Cn = clean.shape[1]
    y = [first_argmax(clean[b]) for b in range(B)] if cls is None else [int(c) for c in cls]
    beams = [[()] for _ in range(B)]
    out = dict(removed=np.zeros((B, P), bool), n_removed=np.full(B, -1, np.int64), logits=np.zeros((B, Cn), np.float32),
               clean=clean, score=np.zeros(B, np.float32), best_score=np.zeros((B, R + 1), np.float32), beams=[],
               rows=[])
    done = [False] * B
    for r in range(R + 1):
        per = []
        if r == 0:
            slots = [[((), -1)] for _ in range(B)]
        elif exhaustive:
            slots = [[(c, -1) for c in itertools.combinations(range(P), r)] for _ in range(B)]
        else:
            Wr = min(W, math.comb(P, r - 1))
            slots = [[(beams[b][w] if w < len(beams[b]) else None, p) for w in range(Wr) for p in range(P)]
                     for b in range(B)]
        out["rows"].append(len(slots[0]))
        rows = []
        for b in range(B):
            for S, p in slots[b]:
                if S is None or p in S:          # an empty beam slot, or p already removed: evaluated and ignored
                    continue
                rows.append((b, tuple(sorted(S + ((p,) if p >= 0 else ())))))
        z = np.asarray(logits_fn(rows), np.float32)
        for b in range(B):
            cands = {}
            for i, (bb, c) in enumerate(rows):
                if bb == b:
                    s, ok = row_score(z[i], y[b], targeted)
                    if c not in cands or (s, c) < cands[c][:2]:
                        cands[c] = (s, c, ok, z[i])
            order = sorted(cands.values(), key=lambda e: (e[0], e[1]))
            out["best_score"][b, r] = order[0][0]
            wins = [e for e in order if e[2]]
            res = None
            if not done[b] and wins:
                res, done[b] = wins[0], True
                out["n_removed"][b] = r
            elif not done[b] and r == R:
                res = order[0]
            if res is not None:
                out["removed"][b] = False
                out["removed"][b, list(res[1])] = True
                out["logits"][b], out["score"][b] = res[3], res[0]
            beams[b] = [e[1] for e in order[:(1 if r == 0 else W)]]
            per.append(list(beams[b]))
        out["beams"].append(per)
    return out


def brute_force(logits_fn, B, P, R, cls=None, targeted=False):
    """n_removed and best_score over all subsets of at most R players."""
    clean = np.asarray(logits_fn([(b, ()) for b in range(B)]), np.float32)
    y = [first_argmax(clean[b]) for b in range(B)] if cls is None else list(cls)
    nr = np.full(B, -1, np.int64)
    best = np.zeros((B, R + 1), np.float32)
    for r in range(R + 1):
        sets = list(itertools.combinations(range(P), r))
        z = np.asarray(logits_fn([(b, c) for b in range(B) for c in sets]), np.float32).reshape(B, len(sets), -1)
        for b in range(B):
            sc = [row_score(z[b, i], y[b], targeted) for i in range(len(sets))]
            best[b, r] = min(s for s, _ in sc)
            if nr[b] < 0 and any(ok for _, ok in sc):
                nr[b] = r
    return nr, best


def removed_copies(src, static, times, lengths, rows, players, remove_mask):
    """The batch rows [(b, removed players)] as removed copies (torch, on the inputs' device)."""
    N = src.shape[2] // 2
    idx = torch.tensor([b for b, _ in rows], dtype=torch.int64, device=src.device)
    gone = np.zeros((len(rows), N), bool)
    st_gone = np.zeros(len(rows), bool)
    for i, (_, c) in enumerate(rows):
        for p in c:
            if players[p] < 0:
                st_gone[i] = True
            else:
                gone[i, players[p]] = True
    g = torch.from_numpy(gone).to(src.device)[None]
    x = src[:, idx]
    vals = torch.where(g, 0.0, x[:, :, :N])
    mask = torch.where(g, 0.0, x[:, :, N:]) if remove_mask else x[:, :, N:]
    st = None
    if static is not None:
        st = torch.where(torch.from_numpy(st_gone).to(src.device)[:, None], 0.0, static[idx])
    return torch.cat([vals, mask], 2).contiguous(), st, times[:, idx].contiguous(), lengths[idx].contiguous()


def module_logits(model, d, players, remove_mask, chunk=4096):
    def fn(rows):
        out = []
        for i in range(0, len(rows), chunk):
            with torch.no_grad():
                out.append(model.forward(*removed_copies(d["src"], d["static"], d["times"], d["lengths"],
                                                         rows[i:i + chunk], players, remove_mask))[0].cpu())
        return torch.cat(out).numpy()
    return fn


# ---- CPU --------------------------------------------------------------------------------------------------------------
def test_symbols_exported():
    lib_path = os.path.join(ROOT, "raindrop_b200", "csrc", "librd_b200.so")
    out = subprocess.run(["nm", "-D", "--defined-only", lib_path], capture_output=True, text=True, check=True).stdout
    names = {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert {"rd_sensor_attack_scratch_bytes", "rd_raindrop_v2_sensor_attack"} <= names


def test_scratch_query():
    from raindrop_b200 import lib as L
    cfg = model_config("P19", dropout=0.2)
    model = build_dropin(cfg, 1, device="cpu")
    lib = L.load()
    dims = model._plan.dims(128, False)
    q = lambda P, W, R, c: lib.rd_sensor_attack_scratch_bytes(C.byref(dims), P, W, R, c)     # noqa: E731
    sizes = [q(34, 4, 3, c) for c in (1, 2, 17, 136)]
    assert 0 < sizes[0] and all(a < b for a, b in zip(sizes, sizes[1:]))
    assert q(34, 1, 3, 8) < q(34, 32, 3, 8) and q(34, 4, 1, 8) < q(34, 4, 32, 8)
    assert q(129, 1, 3, 8) > 0 and q(4096, 1, 1, 1) > 0
    for P, W, R, c in ((0, 1, 1, 1), (4097, 1, 1, 1), (34, 0, 1, 1), (34, 33, 1, 1), (34, 1, 0, 1), (34, 1, 33, 1),
                       (3, 1, 4, 1), (34, 1, 1, 0), (34, 1, 1, -2), (34, 1, 1, 1 << 30)):
        assert q(P, W, R, c) == 0, (P, W, R, c)


def _cpu_model(name="TINY"):
    cfg = model_config(name, dropout=0.2)
    return build_dropin(cfg, 3, device="cpu").eval(), make_batch(cfg, 3, seed=1), cfg


def test_argument_validation():
    model, b, cfg = _cpu_model()
    args = (b["src"], b["static"], b["times"], b["lengths"])
    P = cfg["d_inp"]
    with pytest.raises(ValueError, match="eval"):
        SA.sensor_removal_attack(model.train(), *args)
    model.eval()
    bad = [dict(y=[0, 1, 0], target=1), dict(max_removed=0), dict(max_removed=P + 1), dict(max_removed=1.5),
           dict(beam_width=0), dict(beam_width=33), dict(beam_width=True), dict(sensors=[True] * (P - 1)),
           dict(sensors=[False] * P), dict(internal_batch_size=0), dict(max_removed=P + 2, remove_static=True)]
    for kw in bad:
        with pytest.raises(ValueError):
            SA.sensor_removal_attack(model, *args, **kw)
    tiny8, b8, _ = _cpu_model("TINY8")
    with pytest.raises(ValueError, match="static"):
        SA.sensor_removal_attack(tiny8, b8["src"], None, b8["times"], b8["lengths"], remove_static=True)
    # too many exhaustive subsets: sum_{r <= R} C(P, r) > 2^31 - 1 at P = 129, R = 6
    with pytest.raises(ValueError, match="exhaustive"):
        SA._check_search(129, 6, 1, True)
    assert SA._check_search(129, 5, 1, True) == (5, 1)                 # 275,234,705 sets
    assert SA._check_search(129, 6, 1, False) == (6, 1)
    with pytest.raises(ValueError):
        SA._check_class("y", torch.tensor([0, 2, 1]), 3, 2, "cpu")
    with pytest.raises(ValueError):
        SA._check_class("y", torch.tensor([0.0, 1.0, 1.0]), 3, 2, "cpu")
    with pytest.raises(ValueError):
        SA._check_class("target", 2, 3, 2, "cpu")
    assert SA.round_rows(5, 3, 3, False) == [1, 5, 15, 15]
    assert SA.round_rows(5, 3, 3, True) == [1, 5, 10, 10]
    assert SA.player_sensors(5, [True, False, True, False, False], True).tolist() == [0, 2, -1]


def test_no_cuda_raises(monkeypatch):
    from raindrop_b200.lib import RaindropB200Error
    model, b, _ = _cpu_model()
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RaindropB200Error):
        SA.sensor_removal_attack(model, b["src"], b["static"], b["times"], b["lengths"])


def test_robust_accuracy():
    res = SA.SensorRemovalResult(None, torch.tensor([0, 1, 3, -1, 2]), None, None, None, None, None, None, 3, 1, False)
    acc = SA.robust_accuracy(res)
    assert acc.dtype == np.float64 and acc.tolist() == [0.8, 0.6, 0.4, 0.2]


def _oracle_logits(cfg, wseed, batch, players, remove_mask=True):
    from oracle.raindrop_oracle import build_oracle_model
    from raindrop_b200.synth import synth_weights
    o = build_oracle_model(cfg).eval()
    synth_weights(o, cfg, seed=wseed)
    o = o.double()
    src, st = batch["src"].double(), None if batch["static"] is None else batch["static"].double()

    def fn(rows):
        with torch.no_grad():
            x = removed_copies(src, st, batch["times"].double(), batch["lengths"], rows, players, remove_mask)
            return o.forward_dense(*x)[0].float().numpy()
    return fn


@pytest.mark.parametrize("targeted", [False, True], ids=["untargeted", "targeted"])
def test_restatement_wide_beam_is_brute_force_on_oracle(targeted):
    """With W >= C(P, r) for every r <= R the beam is exhaustive: n_removed and best_score equal brute force over all
    subsets, and the result equals exhaustive mode's."""
    cfg = model_config("TINY", dropout=0.2)
    batch = make_batch(cfg, 4, seed=2)
    P, R = cfg["d_inp"] + 1, 3
    players = list(range(cfg["d_inp"])) + [-1]
    fn = _oracle_logits(cfg, 9, batch, players)
    cls = [1, 0, 1, 0] if targeted else None
    W = max(math.comb(P, r) for r in range(R + 1))
    wide = search(fn, 4, P, R, W, False, cls, targeted)
    ex = search(fn, 4, P, R, 1, True, cls, targeted)
    nr, best = brute_force(fn, 4, P, R, cls, targeted)
    assert np.array_equal(wide["n_removed"], nr) and np.array_equal(ex["n_removed"], nr)
    assert np.array_equal(wide["best_score"], best) and np.array_equal(ex["best_score"], best)
    for k in ("removed", "logits", "score"):
        assert np.array_equal(wide[k], ex[k]), k
    greedy = search(fn, 4, P, R, 1, False, cls, targeted)
    assert (greedy["best_score"] >= best).all()
    assert ((greedy["n_removed"] < 0) | (nr <= greedy["n_removed"]) & (nr >= 0)).all()


def _table_fn(table, C=2):
    """logits_fn of a hand-built table {removed tuple: logits}; sets not in it get [1, 0] (no success, s = 1)."""
    def fn(rows):
        return np.array([table.get(c, [1.0, 0.0][:C]) for _, c in rows], np.float32)
    return fn


def test_restatement_ties_dedup_and_success_rule():
    P = 4
    # every single removal ties at s = 0 (z = [1, 1]: the first argmax is still y = 0, no success); among pairs,
    # (0, 2), (0, 3) and (1, 2) succeed with s = -1 and (2, 3) ties at s = 0; the clean row scores 1
    table = {(p,): [1.0, 1.0] for p in range(P)}
    table.update({(0, 2): [1.0, 2.0], (0, 3): [1.0, 2.0], (1, 2): [1.0, 2.0], (2, 3): [0.5, 0.5]})
    greedy = search(_table_fn(table), 1, P, 2, 1, False, [0])
    assert greedy["beams"][1] == [[(0,)]]                               # the tie goes to the smallest tuple
    assert greedy["n_removed"].tolist() == [2] and np.flatnonzero(greedy["removed"][0]).tolist() == [0, 2]
    assert greedy["best_score"][0].tolist() == [1.0, 0.0, -1.0]
    assert greedy["rows"] == [1, 4, 4]
    beam = search(_table_fn(table), 1, P, 2, 3, False, [0])
    assert beam["beams"][1] == [[(0,), (1,), (2,)]]
    # round 2 rows: 3 slots x 4 players, (0, 1) and (0, 2) / (1, 2) reached twice: the beam holds distinct sets
    assert beam["rows"] == [1, 4, 12]
    assert beam["beams"][2] == [[(0, 2), (0, 3), (1, 2)]]
    assert np.flatnonzero(beam["removed"][0]).tolist() == [0, 2]
    # a tie at s = 0 where the first argmax is not y: z = [1, 1] against y = 1 succeeds
    ok = search(_table_fn({(3,): [1.0, 1.0]}), 1, P, 1, 1, False, [1])
    assert ok["n_removed"].tolist() == [0]                              # the clean row [1, 0] already misses y = 1
    tgt = search(_table_fn({(3,): [1.0, 1.0], (1,): [0.0, 1.0]}), 1, P, 1, 2, False, [1], targeted=True)
    assert tgt["n_removed"].tolist() == [1] and np.flatnonzero(tgt["removed"][0]).tolist() == [1]
    # (3,) ties at s = 0 but argmax is 0: only (1,) succeeds, although (3,) is not worse in s
    tgt = search(_table_fn({(3,): [1.0, 1.0], (1,): [1.0, 1.0 + 2 ** -20]}), 1, P, 1, 1, False, [1], targeted=True)
    assert tgt["best_score"][0, 1] < 0 and np.flatnonzero(tgt["removed"][0]).tolist() == [1]
    # a non-finite logit scores +inf and never succeeds; without a success the result is round R's best
    nan = search(_table_fn({(p,): [np.nan, 5.0] for p in range(P)}), 1, P, 1, 1, False, [0])
    assert nan["n_removed"].tolist() == [-1] and nan["best_score"][0, 1] == np.inf
    assert np.flatnonzero(nan["removed"][0]).tolist() == [0] and nan["score"][0] == np.inf


# ---- GPU --------------------------------------------------------------------------------------------------------------
def _setup(name, mode=EXACT, wseed=9, dseed=3):
    cfg_name, B, opts = CASES[name]
    cfg = model_config(cfg_name, dropout=0.2)
    d = to_dev(make_batch(cfg, B, seed=dseed, **opts))
    model = build_dropin(cfg, wseed).eval()
    model._plan.obprop_mode = mode
    return cfg, d, model


def _args(d):
    return d["src"], d["static"], d["times"], d["lengths"]


def _check(res, want, model, d, remove_mask=True):
    assert torch.equal(res.n_removed.cpu(), torch.from_numpy(want["n_removed"]))
    assert torch.equal(res.success.cpu(), torch.from_numpy(want["n_removed"] >= 0))
    assert torch.equal(res.removed.cpu(), torch.from_numpy(want["removed"]))
    assert np.array_equal(res.best_score.cpu().numpy(), want["best_score"])
    assert np.array_equal(res.score.cpu().numpy(), want["score"])
    assert np.array_equal(res.logits.cpu().numpy().view(np.int32), want["logits"].view(np.int32))
    assert np.array_equal(res.clean_logits.cpu().numpy().view(np.int32), want["clean"].view(np.int32))
    # the returned logits are bitwise the module's forward on the returned set
    rows = [(b, tuple(np.flatnonzero(want["removed"][b]).tolist())) for b in range(d["src"].shape[1])]
    with torch.no_grad():
        f = model.forward(*removed_copies(*_args(d), rows, res.players.tolist(), remove_mask))[0]
    assert torch.equal(res.logits, f)


def _budget(P, mode, name):
    if mode == "exhaustive":
        return min(3 if name in ("tiny_b6", "tiny8_b5") else 2, P)
    return min(3, P)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["greedy", "beam3", "exhaustive"])
@pytest.mark.parametrize("name", list(CASES))
def test_matches_restatement(name, mode):
    cfg, d, model = _setup(name)
    B, P = d["src"].shape[1], cfg["d_inp"]
    R, W = _budget(P, mode, name), 3 if mode == "beam3" else 1
    y = d["y"]
    res = SA.sensor_removal_attack(model, *_args(d), y, max_removed=R, beam_width=W, exhaustive=mode == "exhaustive")
    want = search(module_logits(model, d, list(range(P)), True), B, P, R, W, mode == "exhaustive", y.tolist())
    _check(res, want, model, d)
    assert res.players.tolist() == list(range(P)) and res.best_score.shape == (B, R + 1)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny_b6", "tiny8_b5"])
def test_wide_beam_equals_exhaustive(name):
    cfg, d, model = _setup(name)
    P, R = cfg["d_inp"], 3
    W = max(math.comb(P, r) for r in range(R + 1))
    a = SA.sensor_removal_attack(model, *_args(d), max_removed=R, beam_width=W)
    b = SA.sensor_removal_attack(model, *_args(d), max_removed=R, exhaustive=True)
    for k in ("removed", "n_removed", "success", "logits", "clean_logits", "score", "best_score"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_exhaustive_dominates_greedy(name):
    cfg, d, model = _setup(name, FAST)
    R = 2
    g = SA.sensor_removal_attack(model, *_args(d), d["y"], max_removed=R)
    e = SA.sensor_removal_attack(model, *_args(d), d["y"], max_removed=R, exhaustive=True)
    assert (e.best_score <= g.best_score).all()
    assert torch.equal(e.best_score[:, :2], g.best_score[:, :2])          # rounds 0 and 1 see every set
    won = g.success
    assert (e.success[won]).all() and (e.n_removed[won] <= g.n_removed[won]).all()
    assert (SA.robust_accuracy(e) <= SA.robust_accuracy(g)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny_b6", "tiny8_b5", "p19_b9"])
def test_modes_match_restatement(name):
    cfg, d, model = _setup(name)
    B, N = d["src"].shape[1], cfg["d_inp"]
    ast = d["static"] is not None
    sensors = np.arange(N) % 3 != 1
    runs = [
        dict(kw=dict(target=1), cls=[1] * B, targeted=True, players=list(range(N))),
        dict(kw=dict(), cls=None, targeted=False, players=list(range(N))),
        dict(kw=dict(remove_mask=False), cls=None, targeted=False, players=list(range(N)), mask=False),
        dict(kw=dict(sensors=torch.from_numpy(sensors), remove_static=ast, beam_width=2), cls=None, targeted=False,
             players=np.flatnonzero(sensors).tolist() + ([-1] if ast else []), W=2),
    ]
    for run in runs:
        P, W, R = len(run["players"]), run.get("W", 1), 3
        res = SA.sensor_removal_attack(model, *_args(d), max_removed=R, **run["kw"])
        assert res.players.tolist() == run["players"]
        fn = module_logits(model, d, run["players"], run.get("mask", True))
        want = search(fn, B, P, R, W, False, run["cls"], run["targeted"])
        _check(res, want, model, d, run.get("mask", True))
        if run["cls"] is None:                      # against the clean prediction: never flipped by no removal
            assert (res.n_removed != 0).all()
    tres = SA.sensor_removal_attack(model, *_args(d), target=torch.zeros(B, dtype=torch.int64), max_removed=1)
    clean = tres.clean_logits.argmax(1)
    assert torch.equal(tres.n_removed == 0, clean == 0)             # targeted: the clean row succeeds when it is t


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_chunking_graph_and_no_side_effects(name):
    cfg, d, model = _setup(name, FAST)
    B, P = d["src"].shape[1], cfg["d_inp"]
    plan = model._prepare(torch.device("cuda"))
    snap = {"rng": plan.rng_state.clone()}
    snap.update({"param." + k: p.detach().clone() for k, p in model.named_parameters()})
    kw = dict(max_removed=3, beam_width=3)
    keys = ("removed", "n_removed", "success", "logits", "clean_logits", "score", "best_score")
    res = [SA.sensor_removal_attack(model, *_args(d), d["y"], internal_batch_size=ib, **kw)
           for ib in (B, 2 * B, 7 * B, 3 * P * B, None)]
    for r in res[1:]:
        for k in keys:
            assert torch.equal(getattr(r, k), getattr(res[0], k)), k
    ex = [SA.sensor_removal_attack(model, *_args(d), max_removed=2, exhaustive=True, internal_batch_size=ib)
          for ib in (B, 5 * B, None)]
    for r in ex[1:]:
        for k in keys:
            assert torch.equal(getattr(r, k), getattr(ex[0], k)), k
    gkw = dict(internal_batch_size=2 * B, **kw)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        SA.sensor_removal_attack(model, *_args(d), **gkw)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    eager = SA.sensor_removal_attack(model, *_args(d), **gkw)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = SA.sensor_removal_attack(model, *_args(d), **gkw)
    SA.sensor_removal_attack(model, *_args(d), max_removed=1, internal_batch_size=B)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        for k in keys:
            assert torch.equal(getattr(out, k), getattr(eager, k)), k
    assert torch.equal(plan.rng_state, snap["rng"])
    for k, p in model.named_parameters():
        assert torch.equal(p.detach(), snap["param." + k]) and p.grad is None, k


@pytest.mark.gpu
def test_no_side_effects_on_a_trained_model():
    """Parameters, their .grad, the dropout rng state and a bound FlatAdam are untouched by the attack."""
    from raindrop_b200.optim import FlatAdam
    import torch.nn.functional as F
    cfg = model_config("P19", dropout=0.2)
    B = 16
    model = build_dropin(cfg, 8).train()
    opt = FlatAdam(model, lr=1e-3)
    for it in range(3):
        d = to_dev(make_batch(cfg, B, seed=60 + it))
        logits, _, _ = model.forward(d["src"], d["static"], d["times"], d["lengths"])
        F.cross_entropy(logits, d["y"]).backward()
        opt.step()
    plan = model._plan
    snap = {"flat_p": opt.flat_p.detach(), "flat_g": opt.flat_g, "exp_avg": opt.exp_avg, "exp_avg_sq": opt.exp_avg_sq,
            "step": opt.step_count, "rng": plan.rng_state}
    snap.update({"param." + k: p.detach() for k, p in model.named_parameters()})
    snap.update({"grad." + k: p.grad for k, p in model.named_parameters() if p.grad is not None})
    before = {k: v.clone() for k, v in snap.items()}
    model.eval()
    SA.sensor_removal_attack(model, *_args(d), d["y"], max_removed=2, beam_width=2)
    torch.cuda.synchronize()
    for k, v in snap.items():
        assert torch.equal(v, before[k]), k
    model.train()
    logits, _, _ = model.forward(d["src"], d["static"], d["times"], d["lengths"])
    F.cross_entropy(logits, d["y"]).backward()
    opt.step()


@pytest.mark.gpu
def test_large_shape_129_players_greedy():
    cfg = model_config("LARGE", dropout=0.2)
    B = 2
    d = to_dev(make_batch(cfg, B, seed=3))
    model = build_dropin(cfg, 9).eval()
    model._plan.obprop_mode = FAST
    res = SA.sensor_removal_attack(model, *_args(d), max_removed=2, remove_static=True)
    assert res.removed.shape == (B, 129) and res.players[-1] == -1
    sizes = res.removed.sum(1)
    assert torch.equal(sizes, torch.where(res.n_removed >= 0, res.n_removed, 2))
    rows = [(b, tuple(torch.nonzero(res.removed[b]).view(-1).tolist())) for b in range(B)]
    with torch.no_grad():
        f = model.forward(*removed_copies(*_args(d), rows, res.players.tolist(), True))[0]
    assert torch.equal(res.logits, f)
    want = search(module_logits(model, d, res.players.tolist(), True), B, 129, 2, 1, False)
    _check(res, want, model, d)


@pytest.mark.gpu
def test_p19_b128_budget_3():
    cfg = model_config("P19", dropout=0.2)
    B = 128
    d = to_dev(make_batch(cfg, B, seed=12))
    model = build_dropin(cfg, 9).eval()
    model._plan.obprop_mode = FAST
    res = SA.sensor_removal_attack(model, *_args(d), d["y"], max_removed=3, beam_width=4)
    acc = SA.robust_accuracy(res)
    assert acc.shape == (4,) and (np.diff(acc) <= 0).all()
    with torch.no_grad():
        clean = model.forward(*_args(d))[0]
    assert torch.equal(res.clean_logits, clean)
    assert acc[0] == pytest.approx((clean.argmax(1) == d["y"]).double().mean().item(), abs=1e-12)
    rows = [(b, tuple(torch.nonzero(res.removed[b]).view(-1).tolist())) for b in range(B)]
    with torch.no_grad():
        f = model.forward(*removed_copies(*_args(d), rows, res.players.tolist(), True))[0]
    assert torch.equal(res.logits, f)
