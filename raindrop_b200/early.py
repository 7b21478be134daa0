"""Early prediction with Raindrop_v2: the model's prediction on every prefix of a record -- "how early would it have
known?" -- computed on the device in one call per batch (rd_raindrop_v2_prefix_logits), per-horizon AUROC / AUPRC and
first alarms on the host, and training on truncated records as a TrainStep whose whole step is one CUDA graph.

    res = prefix_predict(model.eval(), src, static, times, lengths, horizons=[6, 12, 24, float("inf")])
    m = horizon_metrics(res, y)                       # m["auroc"][k], m["auprc"][k] for horizon k
    alarm = first_alarm(res, threshold=0.5)           # per sample: the first prefix with P(class 1) >= 0.5, or -1

    step = PrefixTrainStep(model.train(), batch_size=128, min_fraction=0.25, p_full=0.5)
    step.load_batch(batch)                            # optional batch["rows"]: caller-given cutoffs per slot
    step.step()

Prefix r of a record (0 <= r <= T) is the record cut after row r: rows t < r bit for bit, +0.0 in both halves of src
and in times at rows t >= r (how a shorter record is padded), the statics unchanged and lengths = min(lengths,
#{t < r : times > 0}) -- the rule lengths follow (code/Raindrop.py:317) applied to the truncated record; r >= T is the
record itself.  A prefix is given by row count (rows) or by horizon in the units of times (horizons: the leading rows
with times <= h).  A prefix of length 0 (a horizon before the first observation) is computed as the model computes any
length-0 sample: finite, but outside the reference's envelope (SURVEY.md section 7), so its prediction means little.
"""
import ctypes as C
import math
from dataclasses import dataclass

import numpy as np
import torch

from . import lib as L
from .attribution import _Call, _check_call
from .ood import _auroc, _average_precision
from .smoothing import AugmentedTrainStep


@dataclass
class PrefixResult:
    """prefix_predict's output (device tensors): logits [B, K, C] fp32, cutoffs [B, K] int32 (the rows each prefix
    keeps) and lengths [B, K] int64 (the prefix's length).  Each is a transposed view of the [K, B, ...] buffer the
    device writes."""
    logits: object
    cutoffs: object
    lengths: object


def _table(plan, kind, arr, dtype, device):
    """Device copy of a host prefix table, cached per plan (a CUDA-graph capture of a call copies nothing)."""
    cache = plan.__dict__.setdefault("_prefix_" + kind, {})
    key = (arr.shape, arr.tobytes(), device.index)
    got = cache.get(key)
    if got is None:
        got = cache[key] = torch.tensor(arr, dtype=dtype, device=device)
    return got


def _check_prefixes(horizons, rows, T):
    """Host checks of the prefixes (one sync for a device tensor) -> (kind, values): horizons as float32, rows as int32,
    a numpy array for host input and a tensor for device input; neither: every row count 1 .. T."""
    if horizons is not None and rows is not None:
        raise ValueError("give horizons or rows, not both")
    if horizons is None and rows is None:
        return "rows", np.arange(1, T + 1, dtype=np.int32)
    kind, v = ("horizons", horizons) if horizons is not None else ("rows", rows)
    t = v if torch.is_tensor(v) else torch.as_tensor(np.asarray(v))
    # reading a device tensor's values syncs, which a CUDA-graph capture cannot: the eager call before it checked them
    check_values = not (t.device.type == "cuda" and torch.cuda.is_current_stream_capturing())
    if t.dim() != 1 or t.numel() < 1 or t.numel() >= 1 << 31:
        raise ValueError("%s must be a 1-D sequence of 1 .. 2^31 - 1 prefixes, got shape %s" % (kind, tuple(t.shape)))
    if kind == "horizons":
        if t.is_complex() or t.dtype == torch.bool:
            raise ValueError("horizons must be real numbers")
        t = t.to(torch.float32)
        if check_values and bool(torch.isnan(t).any()):
            raise ValueError("horizons must not be NaN (+-inf are allowed)")
    else:
        if t.is_floating_point() or t.is_complex() or t.dtype == torch.bool:
            raise ValueError("rows must hold integer row counts")
        if check_values:
            lo, hi = torch.stack(torch.aminmax(t.to(torch.int64))).tolist()
            if lo < 0 or hi > T:
                raise ValueError("rows must lie in [0, max_len=%d], got [%d, %d]" % (T, lo, hi))
        t = t.to(torch.int32)
    return kind, (t.numpy() if t.device.type == "cpu" else t)


def prefix_predict(model, src, static, times, lengths, *, horizons=None, rows=None, internal_batch_size=None):
    """The eval-mode logits of K prefixes of every sample (see the module docstring), as a PrefixResult.

    horizons:   [K] times h (tensor or sequence, compared with times in float32; +-inf allowed, NaN refused): prefix k
                keeps the leading rows with times <= h_k.
    rows:       [K] row counts in [0, max_len]: prefix k keeps rows t < rows[k].
    Give at most one of the two; with neither, the prefixes are every row count 1 .. max_len.  A host sequence is copied
    to the device once per plan and content (a device tensor is read where it is).
    internal_batch_size: (prefix, sample) rows per chunk, i.e. max(1, internal_batch_size // B) prefixes per chunk.
                Default: the largest chunk whose scratch fits in 1 GiB.  The result does not depend on it once
                model._plan.obprop_mode is pinned (mode 0 picks the ob-prop arithmetic from the chunk's row count).

    Stream-ordered and sync-free apart from the host checks (a device tensor of prefixes costs one sync for its check,
    skipped under CUDA-graph capture; the device clips rows to [0, max_len] and a NaN horizon keeps no row);
    changes neither the parameters, their .grad, the model's rng state nor a bound FlatAdam, and can be captured in a
    CUDA graph (after an eager call with the same prefixes and shapes).  Raises ValueError for a model in training mode
    or invalid arguments, and RaindropB200Error without CUDA."""
    _check_call("prefix_predict", model, src, static, None, internal_batch_size)
    plan = model._plan
    kind, values = _check_prefixes(horizons, rows, plan.T)
    with torch.no_grad():
        cl = _Call(model, src, static, times, lengths, None, False)
        lib, B, dev = cl.lib, src.shape[1], cl.device
        if torch.is_tensor(values):
            table = values.to(dev).contiguous()
        else:
            table = _table(plan, kind, values, torch.float32 if kind == "horizons" else torch.int32, dev)
        K = table.numel()
        dims = plan.dims(B, False)
        kc, scratch = cl.chunk_scratch("_prefix_scratch", "rd_prefix_scratch_bytes", dims, K, internal_batch_size)
        logits = torch.empty(K, B, plan.n_classes, dtype=torch.float32, device=dev)
        cutoffs = torch.empty(K, B, dtype=torch.int32, device=dev)
        plen = torch.empty(K, B, dtype=torch.int64, device=dev)
        hz, rw = (table, None) if kind == "horizons" else (None, table)
        L.check(lib.rd_raindrop_v2_prefix_logits(C.byref(dims), C.byref(cl.params), cl.x.data_ptr(), L.ptr(cl.st),
                                                 cl.tm.data_ptr(), cl.ln.data_ptr(), plan.node_scale.data_ptr(),
                                                 L.ptr(hz), L.ptr(rw), K, kc, scratch.data_ptr(), logits.data_ptr(),
                                                 cutoffs.data_ptr(), plen.data_ptr(), L.stream_ptr(dev)),
                "rd_raindrop_v2_prefix_logits")
    return PrefixResult(logits.transpose(0, 1), cutoffs.t(), plen.t())


def _class_probs(result, cls):
    """softmax(logits)[..., cls] [B, K] in float64 on the host."""
    lg = torch.as_tensor(result.logits).detach().cpu().double()
    if lg.dim() != 3:
        raise ValueError("result.logits must be [B, K, C], got shape %s" % (tuple(lg.shape),))
    if isinstance(cls, bool) or not isinstance(cls, (int, np.integer)) or not 0 <= int(cls) < lg.shape[2]:
        raise ValueError("cls must be a class index in [0, %d), got %r" % (lg.shape[2], cls))
    return torch.softmax(lg, dim=2)[:, :, int(cls)].numpy()


def horizon_metrics(result, y, cls=1):
    """AUROC (Mann-Whitney, ties count 1/2) and AUPRC (average precision) of P(cls) at each prefix, with the samples of
    label cls as the positives, float64 on the host.  Returns dict(auroc=[K], auprc=[K]) numpy arrays.  Raises
    ValueError when y does not hold both positives and negatives."""
    p = _class_probs(result, cls)
    yy = np.asarray(torch.as_tensor(y).detach().cpu()).reshape(-1)
    if yy.shape[0] != p.shape[0]:
        raise ValueError("y must have the batch's %d labels, got %d" % (p.shape[0], yy.shape[0]))
    pos = yy == int(cls)
    if pos.all() or not pos.any():
        raise ValueError("y must hold samples of class %d and of other classes" % int(cls))
    K = p.shape[1]
    return dict(auroc=np.array([_auroc(p[pos, k], p[~pos, k]) for k in range(K)]),
                auprc=np.array([_average_precision(p[pos, k], p[~pos, k]) for k in range(K)]))


def first_alarm(result, threshold, cls=1):
    """Per sample, the first prefix index k whose softmax probability of cls is >= threshold, or -1 when none is (int64
    [B], host).  With prefixes in increasing order, it is the earliest prefix at which the alarm fires."""
    threshold = float(threshold)
    if math.isnan(threshold):
        raise ValueError("threshold must not be NaN")
    hit = _class_probs(result, cls) >= threshold
    return np.where(hit.any(axis=1), hit.argmax(axis=1), -1).astype(np.int64)


def _check_fraction(name, v):
    v = float(v)
    if not 0.0 <= v <= 1.0:
        raise ValueError("%s must lie in [0, 1], got %r" % (name, v))
    return v


class PrefixTrainStep(AugmentedTrainStep):
    """Training on truncated records on static device buffers: each step cuts every slot of the loaded batch at a cutoff
    drawn on the device and runs TrainStep's forward, backward and Adam on the truncated copy -- all on the device, one
    CUDA graph per step.  A model trained this way has seen short records with the statistics of a prefix, which is
    what prefix_predict asks of it.

    Slot b keeps its whole record with probability p_full; otherwise its cutoff is uniform over lo_b .. R_b, with R_b
    the rows up to its last observation (times > 0) and lo_b = max(f_b + 1, ceil(min_fraction R_b)), f_b the first
    observed row, so every drawn prefix holds an observation (Philox site 104 at the device key {seed, step}; see
    rd_debug_prefix_inputs).  An optional batch["rows"] [B] (integers) gives caller-chosen cutoffs: slot b with
    rows[b] >= 0 is cut after min(rows[b], max_len) rows, one with rows[b] < 0 draws -- so a caller with per-hour labels
    can train on (sample, cutoff, label) slots.

    The truncated copy lands in noisy_src / noisy_static, prefix_times and prefix_lengths, which the training forward
    reads; cutoffs [1, B] holds the step's cutoffs.  noise_seed: the Philox seed (default: 64 bits from os.urandom);
    save and restore the key with noise_key_state() / set_noise_key().  At p_full = 1 a step is TrainStep's bit for bit.
    adam_eps is Adam's epsilon.  One GPU only."""

    augmentation = "early-prediction"

    def __init__(self, model, batch_size, min_fraction=0.25, p_full=0.5, noise_seed=None, lr=1e-4, use_graph=True,
                 betas=(0.9, 0.999), adam_eps=1e-8, group=None):
        self.refuse_distributed(group)
        self.min_fraction = _check_fraction("min_fraction", min_fraction)
        self.p_full = _check_fraction("p_full", p_full)
        super().__init__(model, batch_size, noise_seed, lr, use_graph, betas, adam_eps, group)
        self.prefix_times = torch.zeros_like(self.times)
        self.prefix_lengths = torch.zeros_like(self.lengths)
        self.rows = torch.full((self.B,), -1, dtype=torch.int32, device=self.device)
        self.cutoffs = torch.zeros(1, self.B, dtype=torch.int32, device=self.device)

    def load_batch(self, batch, non_blocking=True):
        """TrainStep.load_batch plus the caller-given cutoffs batch["rows"] ([B] integers, < 0: drawn; default: every
        slot draws)."""
        super().load_batch(batch, non_blocking)
        if batch.get("rows") is not None:
            r = torch.as_tensor(batch["rows"])
            if r.is_floating_point() or r.is_complex() or r.dtype == torch.bool or tuple(r.shape) != (self.B,):
                raise ValueError("rows must be [B=%d] integers, got %s %s" % (self.B, r.dtype, tuple(r.shape)))
            self.rows.copy_(r, non_blocking=non_blocking)
        else:
            self.rows.fill_(-1)

    def _inputs(self):
        return self.noisy_src, self.noisy_static, self.prefix_times, self.prefix_lengths

    def _state(self):
        return super()._state() + (self.prefix_times, self.prefix_lengths, self.cutoffs)

    def _augment(self, st):
        L.check(self.lib.rd_debug_prefix_inputs(C.byref(self.noise_dims), self.src.data_ptr(), L.ptr(self.static),
                                                self.times.data_ptr(), self.lengths.data_ptr(), None,
                                                self.rows.data_ptr(), 1, self.noise_key.data_ptr(), self.p_full,
                                                self.min_fraction, self.cutoffs.data_ptr(), self.noisy_src.data_ptr(),
                                                L.ptr(self.noisy_static), self.prefix_times.data_ptr(),
                                                self.prefix_lengths.data_ptr(), st),
                "rd_debug_prefix_inputs")
