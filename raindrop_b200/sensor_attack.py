"""Worst-case sensor removal for Raindrop_v2: the fewest missing sensors that flip a prediction, searched on the device
in one call per batch (rd_raindrop_v2_sensor_attack) -- greedily, by beam search, or exhaustively.

    res = sensor_removal_attack(model.eval(), src, static, times, lengths, y, max_removed=3)           # greedy
    res = sensor_removal_attack(model.eval(), src, static, times, lengths, y, max_removed=3, beam_width=4)
    res = sensor_removal_attack(model.eval(), src, static, times, lengths, y, max_removed=2, exhaustive=True)
    acc = robust_accuracy(res)        # acc[r]: share of samples still correct with r adversarially missing players

Players.  As in raindrop_b200.ablation: the sensors selected by `sensors` (default: all d_inp) in increasing index, and
with remove_static=True the static vector as one more player, the last.  P is their number.

Removing a player writes +0.0 into its value column at every time step and, with remove_mask=True (the default), into
its mask column, so the sensor looks never observed; remove_mask=False is the reference's leave-sensors-out removal.
The static player is replaced by zeros.  times and lengths are copied bit for bit.  These are the ablation semantics,
and the removed copies are written by the same expansion kernel.

Objective.  Each row is scored from its eval-mode logits z against a reference class, in fp32:
  untargeted (default): y is the given label, or the clean prediction (first argmax) when y is None;
      s = z_y - max_{c != y} z_c, and the row succeeds when the first argmax of z is not y;
  targeted (target=t): s = max_{c != t} z_c - z_t, and the row succeeds when the first argmax is t.
A row with a non-finite logit has s = +inf and never succeeds.  Lower s is a stronger attack.  Candidates are ordered
by (s, sorted tuple of removed player indices), ascending; every selection uses this order, which makes the results
independent of the chunking and of the row order.

Search with beam width W and budget R = max_removed.  Round 0 evaluates the empty set (the clean forward,
clean_logits); if it already succeeds (targeted mode, or a given y that is already misclassified), n_removed = 0.
Round r = 1 .. R extends every beam set S by every player p not in S; the new beam is the W smallest distinct candidates
(S + {p} = S' + {q} happens).  best_score[b, r] is the lowest score of round r.  In the first round with a success,
n_removed[b] = r and the result is the smallest successful candidate of that round, with its logits.  Samples that
succeeded keep searching, so best_score is complete.  With no success within R rounds, n_removed = -1 and the result
is the best candidate of round R.  W = 1 is the greedy attack; with W >= C(P, r) for every r <= R the beam holds every
set and the search is exhaustive.  Round r runs W_r * P rows per sample, W_r = min(W, C(P, r - 1)): rows whose p is in S
and rows of empty beam slots are evaluated and ignored, so every round's shape is fixed.

Exhaustive mode (exhaustive=True) evaluates all C(P, r) sets in round r, with the same scoring and selection: the exact
smallest number of removals that flips each sample (when it is at most R) and the exact curve best_score[b, r].  It
needs sum_{r <= R} C(P, r) <= 2^31 - 1.

This is an empirical attack on the model that ships: robust_accuracy is an upper bound on the accuracy under r missing
players for greedy and beam search, and exact for exhaustive search.  ablation.certify gives certified lower bounds for
the ablation-smoothed classifier instead.
"""
import ctypes as C
import math
from dataclasses import dataclass

import numpy as np
import torch

from . import lib as L
from .ablation import MAX_SUBSETS, _device_sensors, _players
from .adversarial import _sensor_mask
from .attribution import _Call, _check_call


@dataclass
class SensorRemovalResult:
    """sensor_removal_attack's output (device tensors unless noted): removed [B, P] bool (the result set), n_removed [B]
    int64 (the first round with a success, -1: none within max_removed), success [B] bool, logits [B, C] (of the result
    set) and clean_logits [B, C], score [B] (of the result set) and best_score [B, R+1] (the lowest score per round),
    fp32; players [P] int64 on the host (the sensor of each player, -1 for the static player); max_removed, beam_width
    and exhaustive."""
    removed: object
    n_removed: object
    success: object
    logits: object
    clean_logits: object
    score: object
    best_score: object
    players: object
    max_removed: int
    beam_width: int
    exhaustive: bool


def _check_int(name, v):
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
        raise ValueError("%s must be an int, got %r" % (name, v))
    return int(v)


def round_rows(P, beam_width, max_removed, exhaustive):
    """Candidates of rounds 0 .. R per sample: 1, then C(P, r) (exhaustive) or min(W, C(P, r - 1)) * P."""
    if exhaustive:
        return [math.comb(P, r) for r in range(max_removed + 1)]
    return [1] + [min(beam_width, math.comb(P, r - 1)) * P for r in range(1, max_removed + 1)]


def _check_search(P, max_removed, beam_width, exhaustive):
    R = _check_int("max_removed", max_removed)
    W = _check_int("beam_width", beam_width)
    if not 1 <= R <= min(P, L.SENSOR_ATTACK_MAX_REMOVED):
        raise ValueError("max_removed must be in [1, min(n_players = %d, %d)], got %d"
                         % (P, L.SENSOR_ATTACK_MAX_REMOVED, R))
    if not 1 <= W <= L.SENSOR_ATTACK_MAX_BEAM:
        raise ValueError("beam_width must be in [1, %d], got %d" % (L.SENSOR_ATTACK_MAX_BEAM, W))
    if exhaustive:
        total = sum(round_rows(P, W, R, True))
        if total > MAX_SUBSETS:
            raise ValueError("exhaustive mode needs sum_{r <= max_removed} C(n_players, r) <= 2^31 - 1, got %d for "
                             "n_players = %d, max_removed = %d" % (total, P, R))
    return R, W


def _check_class(name, v, B, n_classes, device):
    """An int or integer [B] class indices as a contiguous int64 device tensor; the range of a tensor is checked on the
    host (one sync), skipped under CUDA-graph capture (the eager call before it checked it)."""
    if isinstance(v, bool):
        raise ValueError("%s must hold integer class indices" % name)
    if isinstance(v, (int, np.integer)):
        if not 0 <= int(v) < n_classes:
            raise ValueError("%s %d out of range for %d classes" % (name, int(v), n_classes))
        return torch.full((B,), int(v), dtype=torch.int64, device=device)
    t = torch.as_tensor(v)
    if t.is_floating_point() or t.is_complex() or t.dtype == torch.bool:
        raise ValueError("%s must hold integer class indices" % name)
    if tuple(t.shape) != (B,):
        raise ValueError("%s must be an int or have shape [B=%d], got %s" % (name, B, tuple(t.shape)))
    if not (t.device.type == "cuda" and torch.cuda.is_current_stream_capturing()):
        lo, hi = torch.stack(torch.aminmax(t)).tolist()
        if lo < 0 or hi >= n_classes:
            raise ValueError("%s values must lie in [0, %d), got [%d, %d]" % (name, n_classes, lo, hi))
    return t.to(device=device, dtype=torch.int64).contiguous()


def player_sensors(N, sensors, remove_static):
    """The sensor of each player, int64 [P] on the host (-1: the static player)."""
    s = _sensor_mask(sensors, N, "cpu")
    idx = torch.arange(N, dtype=torch.int64) if s is None else torch.nonzero(s).view(-1)
    return torch.cat([idx, torch.tensor([-1] if remove_static else [], dtype=torch.int64)])


def sensor_removal_attack(model, src, static, times, lengths, y=None, *, target=None, max_removed=3, beam_width=1,
                          exhaustive=False, sensors=None, remove_static=False, remove_mask=True, internal_batch_size=None):
    """The fewest players whose removal flips each sample's prediction (see the module docstring), as a
    SensorRemovalResult.

    y:          None (the clean prediction) or the reference classes (an int or [B] integers); untargeted.
    target:     an int or [B] class indices: the targeted attack (give y or target, not both).
    max_removed: R, the budget, 1 <= R <= min(P, 32).
    beam_width: W, 1 <= W <= 32 (1: greedy).  Not used with exhaustive=True.
    exhaustive: every set of at most R players (sum_{r <= R} C(P, r) <= 2^31 - 1).
    sensors:    None (every sensor is a player) or a bool [d_inp]: the sensors that are players (a host mask when the
                call is captured in a CUDA graph).
    remove_static: the static vector is a player too, the last (needs a model with a static branch).
    remove_mask: a removed sensor's mask column is zeroed too (True), or only its values (False).
    internal_batch_size: (candidate, sample) rows per chunk, i.e. max(1, internal_batch_size // B) candidates per chunk.
                Default: the largest chunk whose scratch fits in 1 GiB.  The result does not depend on it once
                model._plan.obprop_mode is pinned.

    Stream-ordered and sync-free apart from the host checks (a device tensor of classes costs one sync for its range
    check, skipped under capture); changes neither the parameters, their .grad, the model's rng state nor a bound
    FlatAdam, and can be captured in a CUDA graph (after an eager call with the same arguments and shapes).  Raises
    ValueError for a model in training mode or invalid arguments, and RaindropB200Error without CUDA."""
    _check_call("sensor_removal_attack", model, src, static, None, internal_batch_size)
    if y is not None and target is not None:
        raise ValueError("give y (untargeted) or target (targeted), not both")
    plan = model._plan
    P = _players(model, sensors, remove_static)
    R, W = _check_search(P, max_removed, beam_width, bool(exhaustive))
    with torch.no_grad():
        cl = _Call(model, src, static, times, lengths, None, False)
        lib, B, dev = cl.lib, src.shape[1], cl.device
        ncls = plan.n_classes
        cls = None
        if y is not None or target is not None:
            cls = _check_class("y" if target is None else "target", y if target is None else target, B, ncls, dev)
        sens = _device_sensors(plan, sensors, dev)
        dims = plan.dims(B, False)
        n = max(round_rows(P, W, R, bool(exhaustive)))
        cc, scratch = cl.chunk_scratch("_sensor_attack_scratch", "rd_sensor_attack_scratch_bytes", dims, n,
                                       internal_batch_size, P, W, R)
        removed = torch.empty(B, P, dtype=torch.uint8, device=dev)
        n_removed = torch.empty(B, dtype=torch.int64, device=dev)
        logits = torch.empty(B, ncls, dtype=torch.float32, device=dev)
        clean = torch.empty(B, ncls, dtype=torch.float32, device=dev)
        score = torch.empty(B, dtype=torch.float32, device=dev)
        best = torch.empty(B, R + 1, dtype=torch.float32, device=dev)
        yy, tt = (cls, None) if target is None else (None, cls)
        L.check(lib.rd_raindrop_v2_sensor_attack(C.byref(dims), C.byref(cl.params), cl.x.data_ptr(), L.ptr(cl.st),
                                                 cl.tm.data_ptr(), cl.ln.data_ptr(), plan.node_scale.data_ptr(),
                                                 L.ptr(sens), P, int(bool(remove_static)), int(bool(remove_mask)),
                                                 L.ptr(yy), L.ptr(tt), W, R, int(bool(exhaustive)), cc,
                                                 scratch.data_ptr(), removed.data_ptr(), n_removed.data_ptr(),
                                                 logits.data_ptr(), clean.data_ptr(), score.data_ptr(), best.data_ptr(),
                                                 L.stream_ptr(dev)),
                "rd_raindrop_v2_sensor_attack")
    return SensorRemovalResult(removed.view(torch.bool), n_removed, n_removed >= 0, logits, clean, score, best,
                               player_sensors(plan.N, sensors, remove_static), R, W, bool(exhaustive))


def robust_accuracy(result):
    """float64 [R+1] on the host: entry r is the share of samples with n_removed == -1 or n_removed > r.  With y = the
    labels, the empirical accuracy under r adversarially missing players (an upper bound for greedy and beam search,
    exact for exhaustive search)."""
    nr = torch.as_tensor(result.n_removed).detach().cpu().numpy().astype(np.int64)
    if nr.size == 0:
        raise ValueError("the result holds no samples")
    r = np.arange(int(result.max_removed) + 1)
    held = (nr[:, None] == -1) | (nr[:, None] > r[None, :])
    return held.mean(axis=0).astype(np.float64)
