"""Training-step plumbing around the C ABI: the ops code/Raindrop.py:319-324 performs per batch
(forward, CrossEntropyLoss, backward, Adam) plus the one collective the CUDA build adds -- a single
NCCL all-reduce over the flat fp32 bucket of the gradients that exist (SURVEY.md section 8e).

Two ways to run a step:
  * the reference's own loop (model.forward -> criterion -> loss.backward() -> optimizer.step()),
    with `allreduce_gradients(model)` between backward and step when world_size > 1;
  * `TrainStep`: the same arithmetic on static buffers, straight through the C ABI (no autograd
    bookkeeping, no allocation), optionally captured into ONE CUDA graph -- the launch-latency
    killer at the reference's batch sizes (B = 128: ~70 kernels of a few microseconds each).
"""
import ctypes as C

import torch
import torch.distributed as dist

from . import functional as RF
from . import lib as L
from .data import DeviceDataset  # noqa: F401  (re-exported: the batch assembler lives with the input pipeline)


def allreduce_gradients(model, group=None):
    """Sum-all-reduce + 1/world scaling of the gradients produced by the last backward.  Uses the
    flat bucket the backward wrote (one collective); falls back to a gather if autograd had to
    copy (gradient accumulation)."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    world = dist.get_world_size(group)
    params = model.used_parameters()
    flat = model._flat_grad
    aliased = flat is not None and all(p.grad is not None for p in params)
    if aliased:
        lo, hi = flat.data_ptr(), flat.data_ptr() + flat.numel() * 4
        aliased = all(lo <= p.grad.data_ptr() < hi for p in params)
    if aliased:
        dist.all_reduce(flat, group=group)
        flat.mul_(1.0 / world)
        return
    grads = [p.grad for p in params if p.grad is not None]
    buf = torch.cat([g.reshape(-1) for g in grads])
    dist.all_reduce(buf, group=group)
    buf.mul_(1.0 / world)
    off = 0
    for g in grads:
        g.copy_(buf[off:off + g.numel()].view_as(g))
        off += g.numel()


def shard_slice(n, rank, world):
    """Contiguous slice of `n` samples owned by `rank` (sizes differ by at most one)."""
    base, extra = divmod(n, world)
    start = rank * base + min(rank, extra)
    return slice(start, start + base + (1 if rank < extra else 0))


def evaluate_sharded(model, P, Pstatic, Ptime, group=None):
    """`evaluate_standard` (code/utils_rd.py:310-320: the WHOLE validation set as one batch) with the samples
    sharded over the ranks and the logits all-gathered, so every rank returns the full [n, n_classes]."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    n = P.shape[1]
    sl = shard_slice(n, rank, world)
    dev = next(model.parameters()).device
    with torch.no_grad():
        Pt = Ptime[:, sl].to(dev)
        lengths = torch.sum(Pt > 0, dim=0)
        out, _, _ = model.forward(P[:, sl].to(dev), None if Pstatic is None else Pstatic[sl].to(dev), Pt, lengths)
    if world == 1:
        return out
    sizes = [s_.stop - s_.start for s_ in (shard_slice(n, r, world) for r in range(world))]
    biggest = max(sizes)                       # all_gather needs equal shapes: pad the short shards, trim afterwards
    padded = torch.zeros(biggest, out.shape[1], dtype=out.dtype, device=out.device)
    padded[: out.shape[0]] = out
    bufs = [torch.empty_like(padded) for _ in range(world)]
    dist.all_gather(bufs, padded, group=group)
    return torch.cat([b_[:k] for b_, k in zip(bufs, sizes)], 0)


class TrainStep:
    """fwd + loss + bwd + (all-reduce) + Adam for a fixed batch size on static device buffers.

    Data parallel (world > 1): the flat gradient bucket is ordered head | encoder | lin_value pairs.  The front part
    is complete when `rd_raindrop_v2_bwd(RD_BWD_ENCODER)` returns, so its NCCL all-reduce is issued on a side
    stream and runs while the observation-propagation backward (`RD_BWD_OBPROP`) computes the tail part
    (SURVEY.md section 8e); the tail is reduced afterwards and both join before the Adam launch."""

    def __init__(self, model, batch_size, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, group=None, use_graph=True,
                 distributed=True):
        lib = L.load()
        self.lib, self.model, self.B = lib, model, int(batch_size)
        dev = next(model.parameters()).device
        if dev.type != "cuda":
            raise L.RaindropB200Error("TrainStep needs the model on a CUDA device")
        self.device = dev
        self.plan = model._prepare(dev)
        self.betas, self.eps = betas, float(eps)
        self.group = group
        self.world = dist.get_world_size(group) if (distributed and dist.is_initialized()) else 1
        # ---- flatten the used parameters into one bucket (views keep the nn.Parameters alive) ----
        params = model.used_parameters()
        self.offsets, total = [], 0
        for p in params:
            self.offsets.append(total)
            total += (p.numel() + 3) // 4 * 4
        self.split = self.offsets[len(params) - RF.N_OBPROP_FIELDS]     # [0, split): head + encoder, [split, total): ob-prop
        self.flat_p = torch.zeros(total, dtype=torch.float32, device=dev)
        for p, off in zip(params, self.offsets):
            view = self.flat_p[off:off + p.numel()].view(p.shape)
            view.copy_(p.data)
            p.data = view
        self.flat_g = torch.zeros_like(self.flat_p)
        self.exp_avg = torch.zeros_like(self.flat_p)
        self.exp_avg_sq = torch.zeros_like(self.flat_p)
        self.step_count = torch.zeros(2, dtype=torch.int64, device=dev)          # {count, ticket}
        self.lr_dev = torch.full((1,), float(lr), dtype=torch.float32, device=dev)   # read by the Adam kernel every step
        self._lr = float(lr)
        # ---- static I/O buffers ------------------------------------------------------------------
        T, N = self.plan.T, self.plan.N
        self.src = torch.zeros(T, self.B, 2 * N, dtype=torch.float32, device=dev)
        self.times = torch.zeros(T, self.B, dtype=torch.float32, device=dev)
        self.lengths = torch.ones(self.B, dtype=torch.int64, device=dev)
        self.static = torch.zeros(self.B, self.plan.d_static, dtype=torch.float32, device=dev) if self.plan.static else None
        self.y = torch.zeros(self.B, dtype=torch.int64, device=dev)
        self.logits = torch.zeros(self.B, self.plan.n_classes, dtype=torch.float32, device=dev)
        self.d_logits = torch.zeros_like(self.logits)
        self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
        # ---- kernel-side structs --------------------------------------------------------------------
        self.dims = self.plan.dims(self.B, True)
        self.P, self.G = L.RdParams(), L.RdGrads()
        self.P.R_u = self.plan.R_u.data_ptr()
        for (key, path), p, off in zip(self.plan.fields, params, self.offsets):
            RF._set_field(self.P, path, p.data_ptr())
            RF._set_field(self.G, path, self.flat_g.data_ptr() + 4 * off)
        self.ws = torch.empty(lib.rd_workspace_bytes(C.byref(self.dims)) // 4, dtype=torch.float32, device=dev)
        self.scratch = torch.empty(lib.rd_backward_scratch_bytes(C.byref(self.dims)) // 4, dtype=torch.float32, device=dev)
        self.side = torch.cuda.Stream(device=dev) if self.world > 1 else None
        self.graph = None
        self.use_graph = use_graph
        self.kernel_launches = None

    # learning rate lives in a device scalar, so a scheduler can change it under a captured graph
    @property
    def lr(self):
        return self._lr

    @lr.setter
    def lr(self, value):
        self.set_lr(value)

    def set_lr(self, value):
        self._lr = float(value)
        self.lr_dev.fill_(self._lr)

    def load_batch(self, batch, non_blocking=True):
        """Host (pinned) or device tensors -> the static device buffers."""
        self.src.copy_(batch["src"], non_blocking=non_blocking)
        self.times.copy_(batch["times"], non_blocking=non_blocking)
        self.lengths.copy_(batch["lengths"], non_blocking=non_blocking)
        self.y.copy_(batch["y"], non_blocking=non_blocking)
        if self.static is not None:
            self.static.copy_(batch["static"], non_blocking=non_blocking)

    def _inputs(self):
        """(src, static, times, lengths) the forward and backward read: the loaded batch (AdversarialTrainStep reads its
        perturbed copy, PrefixTrainStep its truncated one)."""
        return self.src, self.static, self.times, self.lengths

    def _bwd(self, phases, st):
        _, static, _, lengths = self._inputs()
        L.check(self.lib.rd_raindrop_v2_bwd(C.byref(self.dims), C.byref(self.P), L.ptr(static), lengths.data_ptr(),
                                            self.plan.node_scale.data_ptr(), self.ws.data_ptr(), self.d_logits.data_ptr(),
                                            C.byref(self.G), self.scratch.data_ptr(), phases, st), "rd_raindrop_v2_bwd")

    def _forward(self, st):
        """forward incl. CrossEntropyLoss + d(loss)/d(logits) (fused into the head kernel)"""
        src, static, times, lengths = self._inputs()
        L.check(self.lib.rd_raindrop_v2_fwd(C.byref(self.dims), C.byref(self.P), src.data_ptr(), L.ptr(static),
                                            times.data_ptr(), lengths.data_ptr(), self.plan.node_scale.data_ptr(),
                                            self.plan.rng_state.data_ptr(), self.ws.data_ptr(), self.logits.data_ptr(),
                                            self.y.data_ptr(), self.loss.data_ptr(), self.d_logits.data_ptr(), st),
                "rd_raindrop_v2_fwd")

    def _adam(self, st):
        L.check(self.lib.rd_adam_step(self.flat_p.data_ptr(), self.flat_g.data_ptr(), self.exp_avg.data_ptr(),
                                      self.exp_avg_sq.data_ptr(), self.flat_p.numel(), self._lr, self.lr_dev.data_ptr(),
                                      self.betas[0], self.betas[1], self.eps, 1.0 / self.world, self.step_count.data_ptr(),
                                      st),
                "rd_adam_step")

    def _enqueue(self):
        st = L.stream_ptr(self.device)
        self._forward(st)
        if self.world > 1:
            cur = torch.cuda.current_stream(self.device)
            self._bwd(L.BWD_ENCODER, st)
            self.side.wait_stream(cur)
            with torch.cuda.stream(self.side):           # bucket 1 hides behind the ob-prop backward
                dist.all_reduce(self.flat_g[:self.split], group=self.group)
            self._bwd(L.BWD_OBPROP, st)
            dist.all_reduce(self.flat_g[self.split:], group=self.group)
            cur.wait_stream(self.side)
        else:
            self._bwd(L.BWD_ALL, st)
        self._adam(st)

    def _state(self):
        """What a step changes besides its scratch: snapshotted around capture()'s warm-up steps."""
        return (self.flat_p, self.exp_avg, self.exp_avg_sq, self.step_count, self.plan.rng_state, self.loss, self.logits)

    def _snapshot(self):
        return [t.clone() for t in self._state()]

    def _restore(self, snap):
        for t, s_ in zip(self._state(), snap):
            t.copy_(s_)

    def capture(self, warmup=3):
        """Warm up on a side stream, then capture one step into a CUDA graph.  Warm-up iterations are real
        steps (they load modules, size NCCL channels, ...), so parameters, Adam moments, the step counter and
        the dropout stream are snapshotted before and restored after: capture() has no effect on training."""
        s = torch.cuda.Stream(device=self.device)
        snap = self._snapshot() if warmup > 0 else None
        s.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(s):
            for _ in range(warmup):
                self._enqueue()
            if snap is not None:
                self._restore(snap)
        torch.cuda.current_stream(self.device).wait_stream(s)
        torch.cuda.synchronize(self.device)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._enqueue()
        self.graph = g

    def step(self):
        """Runs one training step on whatever is in the static buffers; returns the loss tensor."""
        if self.use_graph:
            if self.graph is None:
                self.capture()
            self.graph.replay()
        else:
            self._enqueue()
        return self.loss
