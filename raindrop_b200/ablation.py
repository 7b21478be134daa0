"""Certified robustness of Raindrop_v2 to missing, faulty or corrupted sensors by randomized ablation (Levine & Feizi,
AAAI 2020): class votes over random (or all) k-subsets of sensors computed on the device in one call per batch
(rd_raindrop_v2_ablation_counts), the certificates on the host, and ablation training as a TrainStep whose whole step is
one CUDA graph.

    res = certify(model.eval(), src, static, times, lengths, keep=5)            # n0 = 100, n = 100,000, alpha = 0.001
    certified = (res.prediction == y) & (res.radius >= 2)                     # provably correct if any 2 sensors change
    res = certify(model.eval(), src, static, times, lengths, keep=3, exhaustive=True)    # all C(P, 3) subsets: exact

    step = AblationTrainStep(model.train(), batch_size=128, keep=5)            # train on ablated copies
    step.load_batch(batch)
    step.step()

Players.  The players are the sensors n with sensors[n] set (sensors=None: all d_inp), in increasing n; with
ablate_static=True the static vector is one more player, the last.  P is their number.  Sensors that are not players
are always kept and lie outside the threat model.

Ablating a player writes +0.0 into its value column src[:, b, n] at every time step and, with ablate_mask=True (the
default), into its mask column src[:, b, N + n]: an ablated sensor then looks exactly like one that was never observed.
With ablate_mask=False it is the reference's leave-sensors-out removal (values zeroed, mask kept).  The static player is
replaced by zeros.  times, lengths and everything else are copied bit for bit.

Base classifier and votes.  f is the eval-mode model.  Replicate m of sample b keeps k players (1 <= k <= P) and
ablates the others; it votes for the first maximum of its logits, and a row with a non-finite logit votes for no class.
g(x) is the class f returns most often over a uniform k-subset.

Sampled subsets (exactly uniform).  Each (replicate, sample) row runs a partial Fisher-Yates shuffle over 0 .. P-1:
position i = 0 .. k-1 swaps with position i + U(P - i), and the first k positions are kept.  U(r) is Lemire's unbiased
bounded integer, with rejection, over the 32-bit Philox words of key {seed, step + m} at site 101, word j of sample b at
index (b << 32) + j.  A row depends on (seed, step + m, b) alone, so the counts depend on neither B nor the chunking, and
counts(a + b, s) = counts(a, s) + counts(b, s + a).

Exhaustive subsets (derandomized).  exhaustive=True runs each of the J = C(P, k) subsets once: replicate m takes the
subset of lexicographic rank step + m, list(itertools.combinations(range(P), k))[step + m].  The seed is ignored; J must
be <= 2^31 - 1 and step + n <= J.

Certificates.  With Delta(rho) = 1 - C(P - rho, k) / C(P, k), the share of subsets that meet rho given players:
  sampled: c_A from n0 selection replicates at (seed, step), p_lower the one-sided Clopper-Pearson bound of n estimation
      replicates at (seed, step + n0), rounded up to j / J (the true probability is a multiple of 1/J); the radius is
      the largest rho in [0, P - k] with 2 (j - J + C(P - rho, k)) > J, else prediction -1 and radius -1.
  exhaustive: exact counts; rho is certified when every other class c has n_A - Delta_n > n_c + Delta_n, or equality
      with c_A < c (Delta_n = J - C(P - rho, k)); n_A = 0 abstains.  Deterministic, no alpha.
Both state: for every x' that differs from x only in the data of at most `radius` players, g(x') = prediction.  A
player's data is its value column, plus its mask column when ablate_mask, plus the statics for the static player; every
other part of x' (times and lengths included) is identical.  The sampled certificate holds with probability 1 - alpha.
"""
import ctypes as C
import math
from dataclasses import dataclass
from fractions import Fraction

import numpy as np
import torch

from . import lib as L
from .adversarial import _check_key, _sensor_mask
from .attribution import _Call, _check_call
from .smoothing import AugmentedTrainStep, _check_alpha, _check_n, _counts, predict_from_counts, selection_lower_bound
from .uncertainty import _device_key

MAX_SUBSETS = (1 << 31) - 1      # exhaustive mode: C(P, k) subsets at most


@dataclass
class AblationCertifyResult:
    """A certificate per sample: prediction [B] int64 (c_A, or -1 = abstain); radius [B] int64 (a number of players,
    -1 when abstaining); p_lower [B] float64 (the Clopper-Pearson bound before rounding; NaN in exhaustive mode);
    counts0 [B, C] the selection votes and counts [B, C] the estimation votes (int64 device tensors; in exhaustive mode
    both are the exact counts); n_players and keep."""
    prediction: object
    radius: object
    p_lower: object
    counts0: object
    counts: object
    n_players: int
    keep: int


def _players(model, sensors, ablate_static):
    """P for a model and a player selection, checked on the host (sensors None or a bool [d_inp])."""
    if ablate_static and not model.static:
        raise ValueError("ablate_static needs a model with a static branch")
    s = _sensor_mask(sensors, model._plan.N, "cpu")
    P = (model._plan.N if s is None else int(s.sum())) + int(bool(ablate_static))
    if P < 1:
        raise ValueError("no players: select at least one sensor or ablate_static")
    if P > L.ABLATION_MAX_PLAYERS:
        raise ValueError("%d players, at most %d" % (P, L.ABLATION_MAX_PLAYERS))
    return P


def _device_sensors(plan, sensors, device):
    """The sensors mask as a device tensor, cached per plan in one entry that another mask replaces (as _device_key
    caches the key): a CUDA-graph capture after an eager call with the same mask copies nothing.  A mask read by a call
    under capture is held for the plan's lifetime."""
    if sensors is None:
        return None
    s = _sensor_mask(sensors, plan.N, "cpu")
    k = (s.numpy().tobytes(), device.index)
    cached = plan.__dict__.get("_ablation_sensors")
    if cached is None or cached[0] != k:
        cached = plan.__dict__["_ablation_sensors"] = (k, s.to(device))
    got = cached[1]
    if device.type == "cuda" and torch.cuda.is_current_stream_capturing():
        held = plan.__dict__.setdefault("_ablation_sensors_captured", [])
        if not any(t is got for t in held):
            held.append(got)
    return got


def _check_keep(keep, P):
    keep = int(keep)
    if not 1 <= keep <= P:
        raise ValueError("keep must be in [1, n_players = %d], got %d" % (P, keep))
    return keep


def _check_subsets(P, keep):
    J = math.comb(P, keep)
    if J > MAX_SUBSETS:
        raise ValueError("exhaustive mode needs C(n_players, keep) <= 2^31 - 1, got C(%d, %d) = %d" % (P, keep, J))
    return J


def ablation_counts(model, src, static, times, lengths, *, keep, n_samples=None, exhaustive=False, seed=0, step=0,
                    sensors=None, ablate_static=False, ablate_mask=True, internal_batch_size=None):
    """Votes of the ablation-smoothed classifier: counts [B, C] int64 on the model's device, counts[b, c] = how many of
    n_samples ablated replicates of sample b (each keeping `keep` players) the eval-mode model classifies as c (first
    maximum of the logits; a replicate with a non-finite logit votes for no class).

    keep:       k, the players each replicate keeps, 1 <= k <= P.
    n_samples:  replicates per sample, >= 1.  Required in sampled mode; exhaustive mode defaults to J - step.
    exhaustive: replicate m takes the subset of lexicographic rank step + m of the J = C(P, k) <= 2^31 - 1 subsets
                (step + n_samples <= J); False: a uniform random subset drawn at key (seed, step + m).
    seed, step: the key (see the module docstring).  The model's dropout stream is neither read nor advanced.
    sensors:    None (every sensor is a player) or a bool [d_inp]: the sensors that are players (a host mask when the
                call is captured in a CUDA graph).
    ablate_static: the static vector is a player too, the last (needs a model with a static branch).
    ablate_mask: an ablated sensor's mask column is zeroed too (True), or only its values (False).
    internal_batch_size: (replicate, sample) rows per chunk, i.e. max(1, internal_batch_size // B) replicates per chunk.
                Default: the largest chunk whose scratch fits in 1 GiB.  The counts do not depend on it once
                model._plan.obprop_mode is pinned.

    Stream-ordered and sync-free apart from the host checks; changes neither the parameters, their .grad, the model's
    rng state nor a bound FlatAdam, and can be captured in a CUDA graph (after an eager call with the same key and
    shapes).  Raises ValueError for a model in training mode or invalid arguments, and RaindropB200Error without CUDA."""
    _check_call("ablation_counts", model, src, static, None, internal_batch_size)
    P = _players(model, sensors, ablate_static)
    keep = _check_keep(keep, P)
    seed, step = _check_key(seed, step)
    if exhaustive:
        J = _check_subsets(P, keep)
        if n_samples is None:
            n_samples = J - step
        n_samples = _check_n("n_samples", n_samples)
        if step + n_samples > J:
            raise ValueError("exhaustive mode needs step + n_samples <= C(%d, %d) = %d, got %d + %d"
                             % (P, keep, J, step, n_samples))
    else:
        if n_samples is None:
            raise ValueError("sampled mode needs n_samples")
        n_samples = _check_n("n_samples", n_samples)
        if step + n_samples > 1 << 64:
            raise ValueError("step + n_samples must be <= 2^64")
    plan = model._plan
    with torch.no_grad():
        cl = _Call(model, src, static, times, lengths, None, False)
        lib, B, dev = cl.lib, src.shape[1], cl.device
        sens = _device_sensors(plan, sensors, dev)
        dims = plan.dims(B, False)
        cc, scratch = cl.chunk_scratch("_ablation_scratch", "rd_ablation_scratch_bytes", dims, n_samples,
                                       internal_batch_size, P)
        key = _device_key(plan, seed, step, dev)
        counts = torch.empty(B, plan.n_classes, dtype=torch.int64, device=dev)
        L.check(lib.rd_raindrop_v2_ablation_counts(C.byref(dims), C.byref(cl.params), cl.x.data_ptr(), L.ptr(cl.st),
                                                   cl.tm.data_ptr(), cl.ln.data_ptr(), plan.node_scale.data_ptr(),
                                                   L.ptr(sens), P, int(bool(ablate_static)), int(bool(ablate_mask)), keep,
                                                   int(bool(exhaustive)), key.data_ptr(), n_samples, cc,
                                                   scratch.data_ptr(), counts.data_ptr(), L.stream_ptr(dev)),
                "rd_raindrop_v2_ablation_counts")
    return counts


def certify_from_counts(counts0, counts, n_players, keep, alpha=0.001, n=None):
    """The sampled certificate from selection votes counts0 and estimation votes counts ([B, C], tensors or arrays),
    on the host: c_A and the Clopper-Pearson p_lower as smoothing.certify_from_counts computes them (n: the estimation
    draws per sample, default the row sums), p_lower rounded up to j / J with j = ceil(p_lower J), J = C(P, k), and the
    radius the largest rho in [0, P - k] with 2 (j - J + C(P - rho, k)) > J in exact integers; prediction -1 and
    radius -1 when no rho qualifies.  Returns (prediction int64 [B], radius int64 [B], p_lower float64 [B])."""
    P = int(n_players)
    if P < 1:
        raise ValueError("n_players must be >= 1, got %d" % P)
    keep = _check_keep(keep, P)
    alpha = _check_alpha(alpha)
    ca, p_lower = selection_lower_bound(counts0, counts, alpha, n)
    J = math.comb(P, keep)
    pred = np.full(len(ca), -1, dtype=np.int64)
    radius = np.full(len(ca), -1, dtype=np.int64)
    for b, pl in enumerate(p_lower):
        j = math.ceil(Fraction(float(pl)) * J)
        rho = -1
        while rho + 1 <= P - keep and 2 * (j - J + math.comb(P - rho - 1, keep)) > J:
            rho += 1
        if rho >= 0:
            pred[b], radius[b] = ca[b], rho
    return pred, radius, p_lower.astype(np.float64)


def certify_exact_from_counts(counts, n_players, keep):
    """The exhaustive certificate from the exact votes counts [B, C] over all J = C(P, k) subsets, in exact integers on
    the host: c_A the first argmax, and the radius the largest rho in [0, P - k] at which every class c != c_A has
    n_A - Delta_n > n_c + Delta_n, or equality with c_A < c (Delta_n = J - C(P - rho, k)); a sample with n_A = 0
    abstains (prediction -1, radius -1).  Returns (prediction int64 [B], radius int64 [B])."""
    P = int(n_players)
    if P < 1:
        raise ValueError("n_players must be >= 1, got %d" % P)
    keep = _check_keep(keep, P)
    c = _counts(counts)
    J = math.comb(P, keep)
    if (c.sum(axis=1) > J).any():
        raise ValueError("a row has more than C(%d, %d) = %d votes" % (P, keep, J))
    pred = np.full(c.shape[0], -1, dtype=np.int64)
    radius = np.full(c.shape[0], -1, dtype=np.int64)
    for b in range(c.shape[0]):
        ca = int(np.argmax(c[b]))
        nA = int(c[b, ca])
        if nA == 0:
            continue

        def holds(rho):
            dn = J - math.comb(P - rho, keep)
            return all(nA - dn > int(c[b, o]) + dn or (nA - dn == int(c[b, o]) + dn and ca < o)
                       for o in range(c.shape[1]) if o != ca)
        rho = 0                                        # rho = 0 always holds: c_A is the first argmax
        while rho + 1 <= P - keep and holds(rho + 1):
            rho += 1
        pred[b], radius[b] = ca, rho
    return pred, radius


def predict(model, src, static, times, lengths, *, keep, n_samples=1000, alpha=0.001, seed=0, step=0, sensors=None,
            ablate_static=False, ablate_mask=True, internal_batch_size=None):
    """Cohen's PREDICT on ablation votes: smoothing.predict_from_counts of ablation_counts (sampled mode; arguments as
    there).  Returns int64 [B] on the host: the class, or -1 (abstain).  The probability of returning a class other
    than g(x) is at most alpha."""
    alpha = _check_alpha(alpha)
    counts = ablation_counts(model, src, static, times, lengths, keep=keep, n_samples=n_samples, seed=seed, step=step,
                             sensors=sensors, ablate_static=ablate_static, ablate_mask=ablate_mask,
                             internal_batch_size=internal_batch_size)
    return predict_from_counts(counts, alpha)


def certify(model, src, static, times, lengths, *, keep, n0=100, n_samples=100_000, alpha=0.001, exhaustive=False,
            seed=0, step=0, sensors=None, ablate_static=False, ablate_mask=True, internal_batch_size=None):
    """The certified number of players of each sample (see the module docstring).  Sampled: n0 selection replicates at
    key (seed, step) pick c_A, n_samples estimation replicates at (seed, step + n0) bound P(f = c_A), and
    certify_from_counts turns the bound into a radius; it holds with probability >= 1 - alpha.  exhaustive: one
    enumeration of all C(P, keep) subsets (n0, n_samples, alpha, seed and step are not used) and
    certify_exact_from_counts; it holds always.  Other arguments as ablation_counts.  Returns an
    AblationCertifyResult."""
    kw = dict(keep=keep, sensors=sensors, ablate_static=ablate_static, ablate_mask=ablate_mask,
              internal_batch_size=internal_batch_size)
    _check_call("certify", model, src, static, None, internal_batch_size)
    P = _players(model, sensors, ablate_static)
    if exhaustive:
        counts = ablation_counts(model, src, static, times, lengths, exhaustive=True, **kw)
        pred, radius = certify_exact_from_counts(counts, P, keep)
        return AblationCertifyResult(pred, radius, np.full(len(pred), np.nan), counts, counts, P, int(keep))
    alpha = _check_alpha(alpha)
    n0 = _check_n("n0", n0)
    n_samples = _check_n("n_samples", n_samples)
    seed, step = _check_key(seed, step)
    counts0 = ablation_counts(model, src, static, times, lengths, n_samples=n0, seed=seed, step=step, **kw)
    counts = ablation_counts(model, src, static, times, lengths, n_samples=n_samples, seed=seed, step=step + n0, **kw)
    pred, radius, p_lower = certify_from_counts(counts0, counts, P, keep, alpha, n=n_samples)
    return AblationCertifyResult(pred, radius, p_lower, counts0, counts, P, int(keep))


class AblationTrainStep(AugmentedTrainStep):
    """Training on randomly ablated inputs (Levine & Feizi 2020) on static device buffers: each step keeps a uniform
    random `keep`-subset of the players of every sample of the loaded batch (ablation_counts' sampled subsets, one
    replicate at the device key {seed, step}) and runs TrainStep's forward, backward and Adam on the ablated copy -- all
    on the device, one CUDA graph per step.  A base classifier trained this way keeps its accuracy on the ablated inputs
    that certify votes over, which is what makes its certificates large.

    The ablated copy lands in noisy_src / noisy_static (AugmentedTrainStep); keep_table [B, P] uint8 holds the step's
    kept players.  noise_seed: the Philox seed (default: 64 bits from os.urandom); save and restore the key with
    noise_key_state() / set_noise_key().  At keep = P a step is TrainStep's bit for bit.  adam_eps is Adam's epsilon.
    One GPU only."""

    augmentation = "ablation"

    def __init__(self, model, batch_size, keep, sensors=None, ablate_static=False, ablate_mask=True, noise_seed=None,
                 lr=1e-4, use_graph=True, betas=(0.9, 0.999), adam_eps=1e-8, group=None):
        self.refuse_distributed(group)
        self.n_players = _players(model, sensors, ablate_static)
        self.keep = _check_keep(keep, self.n_players)
        self.ablate_static, self.ablate_mask = bool(ablate_static), bool(ablate_mask)
        super().__init__(model, batch_size, noise_seed, lr, use_graph, betas, adam_eps, group)
        self.sensors = _sensor_mask(sensors, self.plan.N, self.device)
        self.keep_table = torch.zeros(self.B, self.n_players, dtype=torch.uint8, device=self.device)

    def _augment(self, st):
        L.check(self.lib.rd_debug_ablation_inputs(C.byref(self.noise_dims), self.src.data_ptr(), L.ptr(self.static),
                                                  self.times.data_ptr(), self.lengths.data_ptr(), L.ptr(self.sensors),
                                                  self.n_players, int(self.ablate_static), int(self.ablate_mask),
                                                  self.keep, 0, self.noise_key.data_ptr(), 0, 1,
                                                  self.keep_table.data_ptr(), self.noisy_src.data_ptr(),
                                                  L.ptr(self.noisy_static), None, None, st),
                "rd_debug_ablation_inputs")
