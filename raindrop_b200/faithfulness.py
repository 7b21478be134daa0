"""Faithfulness of Raindrop_v2's attributions, computed on the device: does removing the players an explanation ranks
highest actually move the prediction the most?

* deletion_curves (rd_raindrop_v2_removal_curves): the deletion and insertion curves of Petsiuk et al. 2018 (RISE) over
  the players of the attribution calls, their trapezoid AUCs and the AOPC of Samek et al. 2017;
* infidelity (rd_raindrop_v2_removal_infidelity): the infidelity of Yeh et al. 2019 (captum.metrics.infidelity) under
  random removal perturbations, the game every removal-based attribution of this package explains.

Players, removal, target and baselines are those of attribution.feature_ablation, shapley_value_sampling and
kernel_shap: sensor groups (sensor_groups) or a map of the value cells (feature_mask), and the static vector as player
G when the model has statics.  Use the same target and baselines as the attribution under test.

    phi, phi_st = shapley_value_sampling(model.eval(), src, static, times, lengths, target=y)
    curves = deletion_curves(model, src, static, times, lengths, (phi, phi_st), target=y)
    curves.deletion_auc(), curves.insertion_auc("probability"), curves.aopc()
    inf = infidelity(model, src, static, times, lengths, (phi, phi_st), target=y, n_samples=1000)
    attr_src, attr_st = integrated_gradients(model, src, static, times, lengths, target=y)
    ig = player_attributions(attr_src, attr_st)          # IG summed per sensor player: [B, P]

Every device sum is in a fixed order: the results are bitwise independent of internal_batch_size with
model._plan.obprop_mode pinned, and both calls can be captured in a CUDA graph.
"""
import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from . import attribution as A
from . import lib as L
from .adversarial import _check_key
from .uncertainty import _device_key

MAX_PLAYERS = L.REMOVAL_MAX_PLAYERS
ORDERS = {"descending": L.REMOVAL_DESCENDING, "ascending": L.REMOVAL_ASCENDING, "absolute": L.REMOVAL_ABSOLUTE}
OUTPUTS = ("logit", "probability")
SITE_REMOVAL = 107           # Philox site of infidelity's removal sets
DEFAULT_ALL_COUNTS = 64      # steps=None: every count 0..P up to this many players, else 21 fractions


def removal_counts(n_players, steps=None):
    """int32 numpy [K]: the removal counts of a curve over n_players = P players.  steps None: 0..P when P <= 64,
    otherwise round(f P) for f = 0, 0.05, ..., 1; an int K >= 2: round(f P) for K evenly spaced fractions f in [0, 1]
    (K <= P + 1); or a strictly increasing integer array in [0, P].  round(v) is floor(v + 1/2)."""
    P = int(n_players)
    if P < 1:
        raise ValueError("n_players must be >= 1, got %d" % P)
    if steps is None:
        if P <= DEFAULT_ALL_COUNTS:
            return np.arange(P + 1, dtype=np.int32)
        steps = 21
    if isinstance(steps, (int, np.integer)) and not isinstance(steps, bool):
        K = int(steps)
        if not 2 <= K <= P + 1:
            raise ValueError("steps as a count must be in [2, n_players + 1 = %d], got %d" % (P + 1, K))
        return np.floor(np.linspace(0.0, 1.0, K) * P + 0.5).astype(np.int32)
    s = torch.as_tensor(steps)
    if s.is_floating_point() or s.is_complex() or s.dtype == torch.bool or s.dim() != 1 or s.numel() < 1:
        raise ValueError("steps must be None, an int or a 1-D integer array of removal counts")
    c = s.cpu().numpy().astype(np.int64)
    if c.min() < 0 or c.max() > P:
        raise ValueError("steps must lie in [0, n_players = %d], got [%d, %d]" % (P, c.min(), c.max()))
    if np.any(np.diff(c) <= 0):
        raise ValueError("steps must be strictly increasing")
    return c.astype(np.int32)


def player_attributions(attr_src, attr_static=None, sensor_groups=None, feature_mask=None):
    """[B, P] float64: per-cell attributions (integrated_gradients' attr_src [T, B, 2N], value half read) summed per
    player of sensor_groups (default one per sensor) or of feature_mask ([T, N] or [T, B, N], -1 = no player), with the
    static attributions (attr_static [B, d_static] summed per sample, or [B]) as player G.  The sums run on the host in
    float64 in a fixed order (numpy's add.at, cells in index order), so they are deterministic."""
    a = torch.as_tensor(attr_src)
    if a.dim() != 3 or a.shape[2] % 2:
        raise ValueError("attr_src must be [T, B, 2*d_inp], got %s" % (tuple(a.shape),))
    T, B, N = a.shape[0], a.shape[1], a.shape[2] // 2
    v = a.detach()[:, :, :N].double().cpu().numpy()                        # [T, B, N]
    if feature_mask is None:
        groups, G = A._check_groups(sensor_groups, N)
        ids = np.broadcast_to(groups[None, None, :], (T, B, N))
    else:
        if sensor_groups is not None:
            raise ValueError("give sensor_groups or feature_mask, not both")
        m, G = A._check_feature_mask(feature_mask, T, B, N)
        m = m.cpu().numpy().astype(np.int64)
        ids = np.broadcast_to(m[:, None, :] if m.ndim == 2 else m, (T, B, N))
    out = np.zeros((B, G + (attr_static is not None)), dtype=np.float64)
    bidx = np.broadcast_to(np.arange(B)[None, :, None], (T, B, N))
    sel = ids >= 0
    np.add.at(out, (bidx[sel], ids[sel]), v[sel])
    if attr_static is not None:
        s = torch.as_tensor(attr_static).detach().double().cpu().numpy()
        if s.shape[:1] != (B,) or s.ndim > 2:
            raise ValueError("attr_static must be [B=%d] or [B, d_static], got %s" % (B, s.shape))
        out[:, G] = s.reshape(B, -1).sum(axis=1) if s.ndim == 2 else s
    return torch.from_numpy(out).to(a.device)


def _host_scores(attributions, B, P):
    """The scores under test as a [B, P] or [P] tensor (no copy yet), checked against the call's B and P."""
    if isinstance(attributions, (tuple, list)):
        if len(attributions) != 2:
            raise ValueError("attributions as a tuple must be (attr_players [B, G], attr_static [B] or None)")
        ap, ast = (torch.as_tensor(t) if t is not None else None for t in attributions)
        if ast is not None:
            if ast.dim() != 1:
                raise ValueError("attr_static must be [B], got %s" % (tuple(ast.shape),))
            ap = torch.cat([ap, ast.to(device=ap.device, dtype=ap.dtype)[:, None]], dim=1)
        phi = ap
    else:
        phi = torch.as_tensor(attributions)
    if phi.is_complex() or phi.dtype == torch.bool:
        raise ValueError("attributions must be real scores")
    if tuple(phi.shape) not in ((B, P), (P,)):
        raise ValueError("attributions must be [B=%d, P=%d], [P] or (attr_players, attr_static) for %d players, got %s"
                         % (B, P, P, tuple(phi.shape)))
    return phi


class _Removal:
    """The operands a removal call shares: the players and the scores, checked on the host (__init__), then the
    attribution-call operands (_Call) and the device copies (load)."""

    def __init__(self, fn, model, src, static, baselines, attributions, sensor_groups, feature_mask,
                 internal_batch_size):
        A._check_call(fn, model, src, static, baselines, internal_batch_size)
        self.groups, self.cells, self.G, self.P = A._players(model, src, sensor_groups, feature_mask)
        if self.P > MAX_PLAYERS:
            raise ValueError("%s takes at most %d players, got %d" % (fn, MAX_PLAYERS, self.P))
        self.phi = _host_scores(attributions, src.shape[1], self.P)

    def load(self, model, src, static, times, lengths, target, baselines):
        self.cl = cl = A._Call(model, src, static, times, lengths, target, baselines)
        device, B, P = cl.device, src.shape[1], self.P
        phi = self.phi.detach().to(device=device, dtype=torch.float32)
        self.phi = phi.expand(B, P).contiguous() if phi.dim() == 1 else phi.contiguous()
        if self.groups is not None:
            self.player, self.stride_t, self.stride_b = A._device_int32(cl.plan, "players", self.groups, device), 0, 0
        else:
            self.player, self.stride_t, self.stride_b = A._cell_players(cl.plan, self.cells, device)
        return cl

    def head(self, dims):
        cl = self.cl
        return (C.byref(dims), C.byref(cl.params), cl.x.data_ptr(), L.ptr(cl.st), cl.tm.data_ptr(), cl.ln.data_ptr(),
                cl.plan.node_scale.data_ptr(), cl.x0.data_ptr(), L.ptr(cl.st0), L.ptr(cl.tgt), self.player.data_ptr(),
                self.stride_t, self.stride_b, self.P, self.phi.data_ptr())


@dataclass
class RemovalCurves:
    """Deletion and insertion curves of a batch.  counts [K] (int32 numpy) removal counts; rank [B, P] int32 (player g's
    position in the order); target [B] int64; deletion_logits / insertion_logits [B, K, C] fp32; deletion / insertion
    [B, K] = F at the target; clean [B] = F(x).  summaries [B, 6] fp64 (the device's deletion AUC, insertion AUC and
    AOPC of the logit, then of the probability) back the methods below."""
    counts: object
    rank: object
    target: object
    deletion_logits: object
    insertion_logits: object
    deletion: object
    insertion: object
    clean: object
    summaries: object

    def _col(self, output, i):
        if output not in OUTPUTS:
            raise ValueError("output must be one of %s, got %r" % (", ".join(OUTPUTS), output))
        return self.summaries[:, i + (3 if output == "probability" else 0)]

    def deletion_auc(self, output="logit"):
        """[B] fp64: trapezoid area under the deletion curve over x_k = counts[k] / P (lower is more faithful)."""
        return self._col(output, 0)

    def insertion_auc(self, output="logit"):
        """[B] fp64: trapezoid area under the insertion curve over x_k = counts[k] / P (higher is more faithful)."""
        return self._col(output, 1)

    def aopc(self, output="logit"):
        """[B] fp64: (1/K) sum_k (F(x) - deletion[b, k]), the area over the perturbation curve."""
        return self._col(output, 2)


def deletion_curves(model, src, static, times, lengths, attributions, target=None, baselines=None, sensor_groups=None,
                    feature_mask=None, steps=None, order="descending", internal_batch_size=None):
    """Deletion and insertion curves of F = logits[b, target[b]] of an eval-mode Raindrop_v2 over the players ranked by
    `attributions`: a [B, P] tensor, the (attr_players [B, G], attr_static [B] or None) pair the coalition calls return,
    or a [P] vector shared by the batch (e.g. a dataset-level sensor importance).  Scores are read in fp32.

    order:  "descending" (phi high to low: most relevant first), "ascending" or "absolute" (|phi| high to low); ties go
            to the lower player index, -0 equals +0 and NaN sorts after every number.
    steps:  the removal counts (removal_counts): None, an int K or a strictly increasing integer array in [0, P].
    Deletion point (k, b) removes the players of rank < counts[k]; insertion point (k, b) removes all others.  So deletion
    at count 0 is x and at count P is x' on every player cell; cells of no player keep x.
    Players, target, baselines and internal_batch_size ((sample, curve point) rows per chunk) as for kernel_shap.

    The call runs the endpoint forward, one rank launch and, per chunk of (curve, count) pairs, a keep-table launch, an
    expansion launch and one eval forward, then the fp64 summaries, all on the device: stream-ordered, sync-free (a
    device target or feature mask costs one sync for its range check) and CUDA-graph capturable with device scores.
    It changes neither the parameters, their .grad, the dropout rng state nor a bound FlatAdam.  Raises ValueError for
    a model in training mode or bad arguments, TypeError for another model class and RaindropB200Error without CUDA."""
    if order not in ORDERS:
        raise ValueError("order must be one of %s, got %r" % (", ".join(ORDERS), order))
    r = _Removal("deletion_curves", model, src, static, baselines, attributions, sensor_groups, feature_mask,
                 internal_batch_size)
    counts = removal_counts(r.P, steps)
    cl = r.load(model, src, static, times, lengths, target, baselines)
    lib, plan, device, B, K = cl.lib, cl.plan, cl.device, src.shape[1], counts.shape[0]
    counts_d = A._device_int32(plan, "removal_counts", counts, device)
    dims = plan.dims(B, False)
    cc, scratch = cl.chunk_scratch("_removal_scratch", "rd_removal_curves_scratch_bytes", dims, 2 * K,
                                   internal_batch_size, r.P, key=device.index)
    C_ = plan.n_classes
    rank = torch.empty(B, r.P, device=device, dtype=torch.int32)
    curve_logits = torch.empty(2, K, B, C_, device=device, dtype=torch.float32)
    ends = torch.empty(2, B, C_, device=device, dtype=torch.float32)
    values = torch.empty(2, B, K, device=device, dtype=torch.float32)
    summaries = torch.empty(B, L.REMOVAL_SUMMARIES, device=device, dtype=torch.float64)
    tgt = torch.empty(B, device=device, dtype=torch.int64)
    L.check(lib.rd_raindrop_v2_removal_curves(*r.head(dims), ORDERS[order], counts_d.data_ptr(), K, cc, scratch.data_ptr(),
                                              rank.data_ptr(), curve_logits.data_ptr(), ends.data_ptr(),
                                              values.data_ptr(), summaries.data_ptr(), tgt.data_ptr(),
                                              L.stream_ptr(device)),
            "rd_raindrop_v2_removal_curves")
    return RemovalCurves(counts=counts, rank=rank, target=tgt, deletion_logits=curve_logits[0].transpose(0, 1),
                         insertion_logits=curve_logits[1].transpose(0, 1), deletion=values[0], insertion=values[1],
                         clean=ends[1].gather(1, tgt[:, None])[:, 0], summaries=summaries)


def infidelity_from_moments(moments, normalize=False):
    """Infidelity [..] (float64 tensor) from the moments [.., 6] = [sum 1, sum a, sum d, sum a^2, sum ad, sum d^2] of M
    replicates:  plain  (sum a^2 - 2 sum ad + sum d^2) / M;  normalize  min over beta of sum (beta a - d)^2 / M =
    (sum d^2 - (sum ad)^2 / sum a^2) / M with beta = sum ad / sum a^2 (Captum's scale-invariant form; beta = 0 when
    sum a^2 = 0).  Moments of split calls add up (see infidelity)."""
    m = torch.as_tensor(moments).double()
    n, saa, sad, sdd = m[..., 0], m[..., 3], m[..., 4], m[..., 5]
    if not normalize:
        return (saa - 2.0 * sad + sdd) / n
    beta = infidelity_beta(m)
    return (sdd - beta * sad) / n


def infidelity_beta(moments):
    """The normalising scale beta = sum ad / sum a^2 of normalize=True (0 when sum a^2 = 0), float64."""
    m = torch.as_tensor(moments).double()
    saa, sad = m[..., 3], m[..., 4]
    return torch.where(saa != 0, sad / torch.where(saa != 0, saa, 1.0), torch.zeros_like(sad))


@dataclass
class InfidelityResult:
    """moments [B, 6] fp64 = [sum 1, sum a, sum d, sum a^2, sum ad, sum d^2] over the replicates; infidelity [B] fp64;
    beta [B] fp64 (1 without normalize); target [B] int64; clean_logits [B, C] fp32 (the logits at x)."""
    moments: object
    infidelity: object
    beta: object
    target: object
    clean_logits: object


def infidelity(model, src, static, times, lengths, attributions, target=None, baselines=None, sensor_groups=None,
               feature_mask=None, n_samples=1000, p_remove=0.5, seed=0, step=0, normalize=False,
               internal_batch_size=None):
    """Infidelity (Yeh et al. 2019) of attributions under removal perturbations: replicate m removes from sample b the
    random set S of players, each independently with probability p_remove, and compares
        a = sum_{g in S} phi[b, g]   with   d = F(x) - F(x with S removed)
    as mean (a - d)^2 over the replicates (normalize: Captum's scale-invariant min over beta of mean (beta a - d)^2).
    Player g of sample b is removed in replicate m iff the 32-bit Philox word b*P + g at site 107, key
    (seed, step + m), is below floor(p_remove 2^32); p_remove in (0, 1] (1 removes every player).  So moments of
    n_samples = M1 + M2 at step s are the moments of M1 at s plus those of M2 at s + M1.

    attributions, players, target and baselines as for deletion_curves; internal_batch_size is (sample, replicate)
    rows per chunk.  a and d are fp64 (d from the fp32 logits) and the moments are added on the device in replicate
    order.  The call runs one forward on the B rows of x and, per chunk of replicates, a keep-table launch, an expansion
    launch, one eval forward and one moment launch; everything else is as for deletion_curves."""
    r = _Removal("infidelity", model, src, static, baselines, attributions, sensor_groups, feature_mask,
                 internal_batch_size)
    n_samples = int(n_samples)
    if n_samples < 1:
        raise ValueError("n_samples must be >= 1, got %d" % n_samples)
    if n_samples >= 1 << 31:
        raise ValueError("n_samples must be < 2^31")
    p_remove = float(p_remove)
    if not 0.0 < p_remove <= 1.0:
        raise ValueError("p_remove must lie in (0, 1], got %r" % p_remove)
    seed, step = _check_key(seed, step)
    cl = r.load(model, src, static, times, lengths, target, baselines)
    lib, plan, device, B = cl.lib, cl.plan, cl.device, src.shape[1]
    key = _device_key(plan, seed, step, device)
    dims = plan.dims(B, False)
    cc, scratch = cl.chunk_scratch("_removal_scratch", "rd_removal_infidelity_scratch_bytes", dims, n_samples,
                                   internal_batch_size, r.P, key=device.index)
    clean = torch.empty(B, plan.n_classes, device=device, dtype=torch.float32)
    moments = torch.empty(B, L.REMOVAL_MOMENTS, device=device, dtype=torch.float64)
    tgt = torch.empty(B, device=device, dtype=torch.int64)
    L.check(lib.rd_raindrop_v2_removal_infidelity(*r.head(dims), key.data_ptr(), p_remove, n_samples, cc,
                                                  scratch.data_ptr(), clean.data_ptr(), moments.data_ptr(), tgt.data_ptr(),
                                                  L.stream_ptr(device)),
            "rd_raindrop_v2_removal_infidelity")
    beta = infidelity_beta(moments) if normalize else torch.ones(B, device=device, dtype=torch.float64)
    return InfidelityResult(moments=moments, infidelity=infidelity_from_moments(moments, normalize), beta=beta,
                            target=tgt, clean_logits=clean)
