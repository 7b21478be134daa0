#!/usr/bin/env python
"""SWA / SWAG: the collect and sample launches against HBM bandwidth, and swag_predictive against the torch loop a user
writes without it.

    python tools/bench_swag.py [--config P19] [--batches 128,3880] [--samples 30] [--rank 20] [--steps 5]

collect / sample: rd_swag_collect and rd_swag_sample on the model's bucket (n floats) and on a synthetic bucket of
         --big-n floats, CUDA events with an L2 flush outside each pair, median over --steps * 10 launches.  Bytes from
         the shapes: collect reads theta (4n) and both fp64 moments (16n), writes them (16n) and one column (4n); sample
         reads the moments (16n) and k columns (4kn) and writes theta_s (4n).  Achieved bytes/s is quoted against the
         3.35 TB/s of the H100 SXM data sheet.
predictive: one swag_predictive call (S samples, rank-K posterior) at each batch size, with the default chunking (the
         largest chunk of rows whose scratch fits in 1 GiB) and in one chunk of B rows, against the torch loop: per
         sample the weights drawn with torch ops in float64, load_state_dict, the module's eval forward and a float64
         softmax accumulation; CUDA events, median over --steps calls after two warm-up calls.
Prints one JSON line, with the card's name, power limit and SM clock read in the same run.
"""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import L2_FLUSH_BYTES, build_model, timed_steps  # noqa: E402
from raindrop_b200.synth import make_batch, model_config  # noqa: E402

HBM_GBS = 3350.0     # H100 SXM data sheet


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return "nvidia-smi unavailable (%r)" % (exc,)


def kernel_rates(n, rank, steps, flush, dev):
    """(collect_us, sample_us, collect_GBs, sample_GBs) of the two launches on a bucket of n floats, k = rank."""
    from raindrop_b200 import lib as L
    lib = L.load()
    theta = torch.randn(n, device=dev)
    mean = torch.zeros(n, dtype=torch.float64, device=dev)
    sq = torch.zeros_like(mean)
    D = torch.zeros(rank, n, device=dev)
    out = torch.empty(n, device=dev)
    key = torch.zeros(2, dtype=torch.int64, device=dev)
    st = L.stream_ptr(dev)
    c = [0]

    def collect():
        L.check(lib.rd_swag_collect(theta.data_ptr(), n, c[0], rank, mean.data_ptr(), sq.data_ptr(), D.data_ptr(), st),
                "rd_swag_collect")
        c[0] += 1

    def sample():
        L.check(lib.rd_swag_sample(mean.data_ptr(), sq.data_ptr(), D.data_ptr(), n, rank, 0.5, key.data_ptr(), 0,
                                   out.data_ptr(), st), "rd_swag_sample")

    for _ in range(rank + 1):
        collect()
    sample()
    torch.cuda.synchronize()
    tc = float(np.median(timed_steps(collect, steps, flush))) * 1e3
    ts = float(np.median(timed_steps(sample, steps, flush))) * 1e3
    bc, bs = 40.0 * n, (20.0 + 4.0 * rank) * n
    return tc, ts, bc / tc * 1e-3, bs / ts * 1e-3


def torch_predictive(model, post, args, S, scale=0.5, seed=0):
    """The loop without the library's call: torch weight draws, load_state_dict, module forward, softmax average."""
    g = torch.Generator(device=post.mean.device).manual_seed(seed)
    sd = torch.sqrt(torch.clamp(post.sq_mean - post.mean * post.mean, min=0))
    k = post.k
    Dk = post.dev[:k].double()
    names = [key for key, _, _ in post.layout]
    acc = None
    with torch.no_grad():
        for _ in range(S):
            z1 = torch.randn(post.n, generator=g, device=sd.device, dtype=torch.float64)
            z2 = torch.randn(k, generator=g, device=sd.device, dtype=torch.float64)
            th = post.mean + math.sqrt(scale) * (sd * z1 + (Dk.t() @ z2) / math.sqrt(k - 1))
            th = th.float()
            state = {name: th[off:off + math.prod(shape)].view(shape) for name, (_, off, shape) in zip(names, post.layout)}
            model.load_state_dict(state, strict=False)
            p = torch.softmax(model(*args)[0].double(), dim=1)
            acc = p if acc is None else acc + p
    return acc / S


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--config", default="P19")
    ap.add_argument("--batches", default="128,3880")
    ap.add_argument("--samples", type=int, default=30)
    ap.add_argument("--rank", type=int, default=20)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--big-n", type=int, default=1 << 24)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_swag measures the H100 path: no CUDA device")
    from raindrop_b200 import swag as SW
    dev = torch.device("cuda", torch.cuda.current_device())
    cfg = model_config(args.config, dropout=0.2)
    model = build_model(cfg, dev).eval()
    model._plan.obprop_mode = 0
    flush = torch.empty(L2_FLUSH_BYTES // 4, device=dev)

    post = SW.SWAG(model, rank=args.rank)
    base = [p.detach().clone() for p in model.used_parameters()]
    g = torch.Generator(device=dev).manual_seed(0)
    with torch.no_grad():
        for _ in range(args.rank + 5):        # a trajectory around the weights: k = rank columns
            for p, b in zip(model.used_parameters(), base):
                p.copy_(b + 1e-3 * torch.randn(b.shape, generator=g, device=dev))
            post.collect(model)
        for p, b in zip(model.used_parameters(), base):
            p.copy_(b)
    out = dict(metric="swag", config=args.config, n=post.n, rank=args.rank, samples=args.samples)
    for tag, n in (("bucket", post.n), ("big", args.big_n)):
        tc, ts, gc, gs = kernel_rates(n, args.rank, args.steps * 10, flush, dev)
        out[tag] = dict(n=n, collect_us=tc, sample_us=ts, collect_GBs=gc, sample_GBs=gs,
                        collect_of_peak=gc / HBM_GBS, sample_of_peak=gs / HBM_GBS)

    for B in (int(b) for b in args.batches.split(",")):
        q = make_batch(cfg, B, seed=22, device=dev)
        qa = (q["src"], q["static"], q["times"], q["lengths"])
        state = {}

        def ours():
            state["res"] = SW.swag_predictive(model, post, *qa, n_samples=args.samples)

        def one_chunk():
            SW.swag_predictive(model, post, *qa, n_samples=args.samples, internal_batch_size=B)

        def loop():
            state["torch"] = torch_predictive(model, post, qa, args.samples)

        saved = [p.detach().clone() for p in model.used_parameters()]
        for fn in (ours, one_chunk, loop):
            fn()
            fn()
        torch.cuda.synchronize()
        t_ours = float(np.median(timed_steps(ours, args.steps, flush)))
        t_one = float(np.median(timed_steps(one_chunk, args.steps, flush)))
        t_loop = float(np.median(timed_steps(loop, args.steps, flush)))
        with torch.no_grad():
            for p, s in zip(model.used_parameters(), saved):
                p.copy_(s)
        out["B%d" % B] = dict(swag_predictive_ms=t_ours, one_chunk_ms=t_one, torch_loop_ms=t_loop,
                              speedup_vs_torch=t_loop / t_ours,
                              mean_probs_max_abs_diff_independent_draws=float((state["res"].mean_probs.double() - state["torch"]).abs().max()))
    out["card"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
