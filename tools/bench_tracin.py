"""Times TracIn (raindrop_b200.influence.tracin) on one GPU: one checkpoint, n_query queries against a DeviceDataset of
n_train synthetic samples.  Prints one JSON line per shape: seconds per checkpoint, train samples/s, the split of the
time (rows = forward + data-gradient backward + materialisation, the forward alone, dot = remainder image + wgmma dot +
reduce), the dot kernel's achieved bytes/s and TFLOP/s against the H100 SXM data sheet (3.35 TB/s, 495 TFLOP/s TF32
dense; 3xTF32 issues three TF32 products per fp32 product), the share of the row kernels' time spent in the
materialisation kernels (torch.profiler over the first four train chunks, applied to the rows time as an estimate), the
paper bound of writing each train row once and reading it once per query block, and the loop of one-sample module backwards timed on
`--loop` samples and extrapolated to n_train.  The card's name and power limit are printed with the numbers.

    python tools/bench_tracin.py --shape P19 --n-query 128 --n-train 31000
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

from helpers import build_dropin, to_dev  # noqa: E402
from raindrop_b200 import influence as IF  # noqa: E402
from raindrop_b200 import lib as L  # noqa: E402
from raindrop_b200.data import BatchBuffers, DeviceDataset  # noqa: E402
from raindrop_b200.synth import make_batch, model_config  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


PSG_KERNELS = ("psg_tile_kernel", "psg_ln_kernel", "psg_head_kernel", "psg_pad_kernel")


def materialisation_share(model, ds, idx, tc, R, ldg, n):
    """Share of the row computation's GPU kernel time spent in the materialisation kernels (psg_tile / ln / head / pad),
    from a torch.profiler run (CUDA activity) over the rows of the first n train samples, in tracin's chunks."""
    from torch.profiler import ProfilerActivity, profile
    st_w = 0 if ds.Pstatic is None else ds.Pstatic.shape[1]

    def fetch(a, b):
        buf = BatchBuffers(ds.T, b - a, ds.width, st_w)
        ds.fill(buf, idx[a:b])
        return buf.src, buf.static, buf.times, buf.lengths, buf.y
    with torch.no_grad(), profile(activities=[ProfilerActivity.CUDA]) as prof:
        for t0 in range(0, n, tc):
            IF._rows_aligned(model, fetch, t0, min(n, t0 + tc), R, ldg)
        torch.cuda.synchronize()
    mat = tot = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        t = e.cuda_time_total if t is None else t
        if t <= 0 or "Memcpy" in e.key or "Memset" in e.key:
            continue
        tot += t
        if any(k in e.key for k in PSG_KERNELS):
            mat += t
    return mat / tot if tot else float("nan")


def run(shape, nq, nt, loop_n):
    cfg = model_config(shape, dropout=0.2)
    model = build_dropin(cfg, 21)
    model.eval()
    dq = to_dev(make_batch(cfg, nq, seed=1))
    dt = make_batch(cfg, nt, seed=2)
    ds = DeviceDataset(dt["src"], dt["static"], dt["times"], dt["y"])
    q = dict(src=dq["src"], static=dq["static"], times=dq["times"], lengths=dq["lengths"], y=None)
    IF.tracin(model, q, (ds, torch.arange(min(nt, 64))))          # warm-up: modules, tensor maps, allocator
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    S = IF.tracin(model, q, ds)
    torch.cuda.synchronize()
    total = time.perf_counter() - t0

    # the split, with CUDA events, over the same chunk plan
    lib, plan = L.load(), model._plan
    layout = IF.grad_layout(model)
    ldg = IF._bucket_length(layout)
    off, ln = IF.plan_segments(layout)
    n_seg = len(off)
    offs, lens = (C.c_int64 * n_seg)(*off.tolist()), (C.c_int64 * n_seg)(*ln.tolist())
    qb, tc, R = IF._blocks(lib, plan, ldg, n_seg, nq, nt, None)
    ev = lambda: torch.cuda.Event(enable_timing=True)
    t_rows = t_fwd = t_dot = 0.0
    scores = torch.zeros(nq, nt, dtype=torch.float64, device="cuda")
    idx = torch.arange(nt, device="cuda")
    with torch.no_grad():
        for q0 in range(0, nq, qb):
            q1 = min(nq, q0 + qb)
            qf = lambda a, b: (dq["src"][:, a:b], None if dq["static"] is None else dq["static"][a:b], dq["times"][:, a:b],
                               dq["lengths"][a:b], None)
            Gq = IF._rows_aligned(model, qf, q0, q1, R, ldg)
            for t0_ in range(0, nt, tc):
                t1_ = min(nt, t0_ + tc)
                bufs = []
                for s0 in range(t0_, t1_, R):
                    buf = BatchBuffers(ds.T, min(t1_, s0 + R) - s0, ds.width, 0 if ds.Pstatic is None else ds.Pstatic.shape[1])
                    ds.fill(buf, idx[s0:s0 + buf.src.shape[1]])
                    bufs.append(buf)
                tf = lambda a, b: (lambda bb: (bb.src, bb.static, bb.times, bb.lengths, bb.y))(bufs[(a - t0_) // R])
                e = [ev() for _ in range(6)]
                e[0].record()
                for buf in bufs:
                    model.forward(buf.src, buf.static, buf.times, buf.lengths)
                e[1].record()
                Gt = IF._rows_aligned(model, tf, t0_, t1_, R, ldg)
                e[2].record()
                nb = lib.rd_per_sample_grad_dot_scratch_bytes(q1 - q0, t1_ - t0_, ldg, n_seg)
                sc = torch.empty((nb + 3) // 4, dtype=torch.float32, device="cuda")
                e[3].record()
                L.check(lib.rd_per_sample_grad_dot(Gq.data_ptr(), q1 - q0, Gt.data_ptr(), t1_ - t0_, ldg, offs, lens, n_seg,
                                                   1.0, scores.data_ptr() + 8 * (q0 * nt + t0_), nt, sc.data_ptr(),
                                                   L.stream_ptr()), "dot")
                e[4].record()
                torch.cuda.synchronize()
                t_fwd += e[0].elapsed_time(e[1]) / 1e3
                t_rows += e[1].elapsed_time(e[2]) / 1e3
                t_dot += e[3].elapsed_time(e[4]) / 1e3
                del Gt, sc
    assert torch.equal(scores, S), "the split run must reproduce tracin bitwise"
    # the materialisation apart from forward and backward: kernel times of a profiled run over the first train chunks
    mat_share = materialisation_share(model, ds, idx, tc, R, ldg, min(nt, 4 * tc))
    K = int(ln.sum())
    dot_bytes = 4 * nt * K * ((nq + qb - 1) // qb) + 4 * 2 * nq * K * ((nt + tc - 1) // tc)   # Gt per query block; Gq, Gq_lo per chunk
    dot_flop = 2.0 * nq * nt * K
    # the loop a user would write without this: one-sample module backwards, timed on loop_n samples
    dl = to_dev(make_batch(cfg, loop_n, seed=3))
    model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for b in range(loop_n):
        sl = slice(b, b + 1)
        logits, _, _ = model.forward(dl["src"][:, sl], None if dl["static"] is None else dl["static"][sl],
                                     dl["times"][:, sl], dl["lengths"][sl])
        g = torch.autograd.grad(F.cross_entropy(logits, dl["y"][sl]), model.used_parameters())
        torch.cat([x.reshape(-1) for x in g])
    torch.cuda.synchronize()
    loop = (time.perf_counter() - t0) / loop_n * (nt + nq)
    return dict(shape=shape, card=card(), n_query=nq, n_train=nt, bucket=ldg, query_block=qb, train_chunk=tc,
                seconds_per_checkpoint=total, train_samples_per_s=nt / total,
                split_s=dict(forward_only=t_fwd, rows=t_rows, dot=t_dot),
                dot_bytes_per_s=dot_bytes / t_dot, dot_hbm_fraction=dot_bytes / t_dot / 3.35e12,
                dot_tflops_fp32_products=dot_flop / t_dot / 1e12,
                dot_tf32_fraction=3 * dot_flop / t_dot / 495e12,
                materialisation_share_of_row_kernels=mat_share, materialisation_s_estimated=mat_share * t_rows,
                paper_bound_s_per_train_sample=8 * ldg / 3.35e12, measured_s_per_train_sample=total / nt,
                one_sample_loop_s_extrapolated=loop, loop_samples_timed=loop_n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="P19")
    ap.add_argument("--n-query", type=int, default=128)
    ap.add_argument("--n-train", type=int, default=31000)
    ap.add_argument("--loop", type=int, default=64)
    a = ap.parse_args()
    print(json.dumps(run(a.shape, a.n_query, a.n_train, a.loop)), flush=True)


if __name__ == "__main__":
    main()
