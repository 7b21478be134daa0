"""Adversarial robustness of Raindrop_v2: projected gradient descent (PGD) attacks computed on the device in one call per
batch (rd_raindrop_v2_pgd), and PGD adversarial training (Madry et al. 2018) as a TrainStep whose whole step is one CUDA
graph.

    res = pgd(model.eval(), src, static, times, lengths, y, eps=0.1)               # PGD-10, L-inf, random start
    robust_acc = 1.0 - res.success.float().mean()
    fgsm = pgd(model.eval(), src, static, times, lengths, y, eps=0.1, n_steps=1, step_size=0.1, random_start=False)

    step = AdversarialTrainStep(model.train(), batch_size=128, eps=0.1, n_steps=3)
    step.load_batch(batch)                                                          # or DeviceDataset.fill(step, idx)
    step.step()

Threat model: only the value half of src moves, and only at observed cells (mask src[..., N:] > 0; padded rows have
mask 0), optionally restricted to some sensors, plus the static vector when perturb_static.  The mask half, times and
lengths never change.  eps is in the units the model sees: per-feature standard deviations after normalisation.
norm "linf": |delta| <= eps per element; "l2": ||delta_b||_2 <= eps per sample over its perturbable elements.  Each
sample is attacked on its own cross-entropy, and the returned input is its iterate of highest loss (x_0 included), so
without a random start the loss never falls below the clean one.  The lift relu(v * R_u) has gradient exactly 0 at a
cell whose d_ob channels are all inactive (for d_ob = 1, every value of the wrong sign): such a cell does not move from
delta = 0, which is why random_start is on by default.
"""
import ctypes as C
import math
import os
from dataclasses import dataclass

import numpy as np
import torch
import torch.distributed as dist

from . import lib as L
from .attribution import _Call, _check_call
from .train import TrainStep
from .uncertainty import _device_key

NORMS = {"linf": 0, "l2": 1}      # RD_PGD_LINF, RD_PGD_L2


@dataclass
class AdversarialResult:
    """src [T, B, 2N] and static [B, d_static] (None without a static branch): the adversarial inputs; logits [B, C] at
    them and loss [B] their cross-entropy; clean_logits [B, C] at the clean inputs; success [B] bool: argmax(logits) != y."""
    src: object
    static: object
    logits: object
    clean_logits: object
    loss: object
    success: object


def _check_attack(eps, norm, n_steps, step_size):
    """Host checks of the attack's settings -> (eps, norm id, n_steps, step size)."""
    eps = float(eps)
    if not (math.isfinite(eps) and eps >= 0):
        raise ValueError("eps must be finite and >= 0, got %r" % eps)
    if norm not in NORMS:
        raise ValueError("norm must be one of %s, got %r" % (", ".join(NORMS), norm))
    n_steps = int(n_steps)
    if not 0 <= n_steps < 1 << 31:
        raise ValueError("n_steps must be in [0, 2^31), got %d" % n_steps)
    if step_size is None:
        step_size = 2.5 * eps / n_steps if n_steps > 0 else 0.0
    step_size = float(step_size)
    if not (math.isfinite(step_size) and step_size >= 0):
        raise ValueError("step_size must be finite and >= 0, got %r" % step_size)
    return eps, NORMS[norm], n_steps, step_size


def _check_key(seed, step):
    seed, step = int(seed), int(step)
    if not (0 <= seed < 1 << 64 and 0 <= step < 1 << 64):
        raise ValueError("seed and step must be in [0, 2^64)")
    return seed, step


def _sensor_mask(sensors, N, device):
    """None, or a bool [N] (tensor or array) -> a contiguous bool device tensor (read as uint8 by the kernels)."""
    if sensors is None:
        return None
    s = torch.as_tensor(sensors)
    if s.dtype != torch.bool:
        raise ValueError("sensors must be a bool mask, got dtype %s" % s.dtype)
    if tuple(s.shape) != (N,):
        raise ValueError("sensors must have shape [d_inp=%d], got %s" % (N, tuple(s.shape)))
    return s.to(device).contiguous()


def pgd(model, src, static, times, lengths, y=None, *, eps, norm="linf", n_steps=10, step_size=None, random_start=True,
        seed=0, step=0, sensors=None, perturb_static=False, internal_batch_size=None):
    """Untargeted PGD on each sample's cross-entropy of an eval-mode Raindrop_v2 (see the module docstring for the
    threat model).  Returns an AdversarialResult of tensors on the model's device.

    y:          [B] labels, or None = the class the model predicts on the clean input.
    eps:        the perturbation budget, >= 0.  norm: "linf" or "l2".
    n_steps:    K >= 0 gradient steps; step_size: alpha, default 2.5 eps / K.  The returned input is the iterate of
                highest loss among x_0 .. x_K (ties: the earliest).  FGSM is n_steps=1, step_size=eps, random_start=False.
    random_start: start from a uniform draw in the eps-ball (linf: per element; l2: uniform in the ball), drawn from
                the Philox stream at key (seed, step) and indexed by (sample, t, sensor), so it does not depend on the
                chunking.  The model's dropout stream is neither read nor advanced.
    sensors:    None (every sensor) or a bool [d_inp]: only those sensors' observed cells are perturbed.
    perturb_static: perturb the static vector too (needs a model with a static branch).
    internal_batch_size: samples per chunk.  Default: the largest chunk whose scratch fits in 1 GiB.  Results are
                bitwise independent of it once model._plan.obprop_mode is pinned (mode 0 picks the ob-prop arithmetic
                from the chunk's row count).

    Stream-ordered and sync-free apart from the host checks (a device-tensor y costs one sync for its range check); it
    changes neither the parameters, their .grad, the model's rng state nor a bound FlatAdam.  Raises ValueError for a
    model in training mode or invalid arguments, and RaindropB200Error without CUDA."""
    _check_call("pgd", model, src, static, None, internal_batch_size)
    eps, norm_id, n_steps, alpha = _check_attack(eps, norm, n_steps, step_size)
    seed, step = _check_key(seed, step)
    if perturb_static and not model.static:
        raise ValueError("perturb_static needs a model with a static branch")
    plan = model._plan
    if sensors is not None:
        _sensor_mask(sensors, plan.N, "cpu")          # shape and dtype checked before anything touches the device
    with torch.no_grad():
        cl = _Call(model, src, static, times, lengths, y, False)
        lib, B, dev = cl.lib, src.shape[1], cl.device
        sens = _sensor_mask(sensors, plan.N, dev)
        dims = plan.dims(B, False)
        spc, scratch = cl.chunk_scratch("_pgd_scratch", "rd_pgd_scratch_bytes", dims, B, internal_batch_size,
                                        per_sample=True)
        key = _device_key(plan, seed, step, dev) if random_start else None
        f32 = dict(device=dev, dtype=torch.float32)
        src_adv = torch.empty_like(cl.x)
        st_adv = torch.empty_like(cl.st) if cl.st is not None else None
        logits = torch.empty(B, plan.n_classes, **f32)
        clean = torch.empty(B, plan.n_classes, **f32)
        loss = torch.empty(B, **f32)
        L.check(lib.rd_raindrop_v2_pgd(C.byref(dims), C.byref(cl.params), cl.x.data_ptr(), L.ptr(cl.st), cl.tm.data_ptr(),
                                       cl.ln.data_ptr(), plan.node_scale.data_ptr(), L.ptr(cl.tgt), L.ptr(sens), None,
                                       int(bool(perturb_static)), norm_id, eps, alpha, n_steps, int(bool(random_start)),
                                       L.ptr(key), spc, scratch.data_ptr(), src_adv.data_ptr(), L.ptr(st_adv),
                                       logits.data_ptr(), clean.data_ptr(), loss.data_ptr(), L.stream_ptr(dev)),
                "rd_raindrop_v2_pgd")
        target = cl.tgt if cl.tgt is not None else clean.argmax(dim=1)
        success = logits.argmax(dim=1) != target
    return AdversarialResult(src_adv, st_adv, logits, clean, loss, success)


class AdversarialTrainStep(TrainStep):
    """PGD adversarial training (Madry et al. 2018) on static device buffers: each step attacks the loaded batch with
    pgd's algorithm in eval arithmetic on the live parameters, then runs TrainStep's forward, backward and Adam on the
    adversarial batch -- all on the device, one CUDA graph per step.

    The clean batch goes where TrainStep keeps it (load_batch, DeviceDataset.fill: src, static, times, lengths, y); the
    attacked copy lands in adv_src / adv_static, which the training forward reads.  An optional batch["attack"] bool [B]
    (default: every slot) attacks only some slots; the others train on their clean input.  After a step, adv_loss [B],
    adv_logits and clean_logits [B, C] hold the attack's per-sample results.  attack_seed: the Philox seed of the random
    start (default: 64 bits from os.urandom); the key {seed, step} lives on the device and every step advances it, so a
    resumed run restores it with attack_key_state() / set_attack_key().  adam_eps is Adam's epsilon.  One GPU only."""

    def __init__(self, model, batch_size, eps, norm="linf", n_steps=10, step_size=None, random_start=True, attack_seed=None,
                 lr=1e-4, use_graph=True, betas=(0.9, 0.999), adam_eps=1e-8, group=None):
        if dist.is_initialized() and dist.get_world_size(group) > 1:
            raise L.RaindropB200Error("AdversarialTrainStep runs on one GPU; data-parallel adversarial training is not supported")
        self.attack_eps, self.norm_id, self.n_steps, self.step_size = _check_attack(eps, norm, n_steps, step_size)
        self.norm, self.random_start = norm, bool(random_start)
        seed = int.from_bytes(os.urandom(8), "little") if attack_seed is None else int(attack_seed)
        _check_key(seed, 0)
        super().__init__(model, batch_size, lr=lr, betas=betas, eps=adam_eps, group=group, use_graph=use_graph,
                         distributed=False)
        dev, lib, B = self.device, self.lib, self.B
        self.attack_dims = self.plan.dims(B, False)
        self.attack = torch.ones(B, dtype=torch.bool, device=dev)
        self.adv_src = torch.zeros_like(self.src)
        self.adv_static = torch.zeros_like(self.static) if self.static is not None else None
        self.adv_logits = torch.zeros_like(self.logits)
        self.clean_logits = torch.zeros_like(self.logits)
        self.adv_loss = torch.zeros(B, dtype=torch.float32, device=dev)
        nbytes = lib.rd_pgd_scratch_bytes(C.byref(self.attack_dims), B)
        if nbytes == 0:
            L.check(-2, "rd_pgd_scratch_bytes")
        self.pgd_scratch = torch.empty(nbytes // 4, dtype=torch.float32, device=dev)
        self.attack_key = torch.tensor(np.array([seed, 0], dtype=np.uint64).view(np.int64), device=dev)

    def load_batch(self, batch, non_blocking=True):
        """TrainStep.load_batch plus the attacked slots batch["attack"] (bool [B], default: every slot)."""
        super().load_batch(batch, non_blocking)
        if batch.get("attack") is not None:
            self.attack.copy_(torch.as_tensor(batch["attack"], dtype=torch.bool), non_blocking=non_blocking)
        else:
            self.attack.fill_(True)

    def _inputs(self):
        return self.adv_src, self.adv_static, self.times, self.lengths

    def _state(self):
        extra = (self.attack_key, self.adv_src, self.adv_logits, self.clean_logits, self.adv_loss)
        return super()._state() + extra + ((self.adv_static,) if self.adv_static is not None else ())

    def _attack(self, st):
        L.check(self.lib.rd_raindrop_v2_pgd(C.byref(self.attack_dims), C.byref(self.P), self.src.data_ptr(),
                                            L.ptr(self.static), self.times.data_ptr(), self.lengths.data_ptr(),
                                            self.plan.node_scale.data_ptr(), self.y.data_ptr(), None,
                                            self.attack.data_ptr(), 0, self.norm_id, self.attack_eps, self.step_size,
                                            self.n_steps, int(self.random_start), self.attack_key.data_ptr(), self.B,
                                            self.pgd_scratch.data_ptr(), self.adv_src.data_ptr(), L.ptr(self.adv_static),
                                            self.adv_logits.data_ptr(), self.clean_logits.data_ptr(),
                                            self.adv_loss.data_ptr(), st),
                "rd_raindrop_v2_pgd")
        self.attack_key[1:].add_(1)

    def _enqueue(self):
        self._attack(L.stream_ptr(self.device))
        super()._enqueue()

    def attack_key_state(self):
        """(seed, step) of the random-start stream, to be saved with a checkpoint (reads the device key: synchronises)."""
        seed, step = (int(v) for v in self.attack_key.cpu().numpy().view(np.uint64))
        return seed, step

    def set_attack_key(self, seed, step):
        """Restores a saved attack_key_state(); the next step draws the random start of that step."""
        seed, step = _check_key(seed, step)
        self.attack_key.copy_(torch.tensor(np.array([seed, step], dtype=np.uint64).view(np.int64)))
