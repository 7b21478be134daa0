#!/usr/bin/env python
"""Randomized-smoothing votes (raindrop_b200.smoothing.smooth_counts) and Gaussian-augmentation training
(SmoothingTrainStep) on the P19 synthetic configuration:

    python tools/bench_smoothing.py [--reps 3] [--loop-reps 500] [--steps 20] [--warmup 3]
    python tools/bench_smoothing.py --ablate 5 [--exhaustive] ...

1. smooth_counts at B = 1 and 128 with n = 1,000 and 10,000 replicates (sigma 0.25), as one device call and as the
   host loop a user writes without it: per replicate torch-generated noise on the observed values, one eval forward of
   raindrop_b200.models_rd.Raindrop_v2, argmax and bincount.  The call: host clock around work that ends in a device
   synchronise, median of --reps calls after one warm-up call.  The loop costs the same per replicate whatever n is, so
   it runs --loop-reps replicates (median of three such runs) and its time for n is that per-replicate time times n
   (reported as extrapolated).
2. SmoothingTrainStep against TrainStep at B = 128, both as captured CUDA graphs in one process, alternating step by
   step with CUDA events (median over --steps replays).
Prints one JSON line with the medians and the card's name and power limit, read in the same run.

--ablate K times randomized ablation (raindrop_b200.ablation) keeping K of the 34 sensors instead: ablation_counts at
the same B and n against its module loop (per replicate a torch.randperm subset per sample, the other sensors' values
and masks zeroed, one eval forward, argmax and bincount) and against smooth_counts at the same n, and AblationTrainStep
against TrainStep.  --exhaustive adds the exhaustive enumeration of all C(34, K) subsets at B = 128.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import build_model  # noqa: E402
from raindrop_b200.synth import make_batch, model_config  # noqa: E402

SIGMA = 0.25


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return "nvidia-smi unavailable (%r)" % (exc,)


def host_loop_counts(model, src, static, times, lengths, sigma, n, gen):
    """The same votes by the module: n eval forwards of B rows on x + sigma z (observed values only)."""
    N = src.shape[2] // 2
    mask = (src[:, :, N:] > 0).float()
    C = model._plan.n_classes
    counts = torch.zeros(src.shape[1], C, dtype=torch.int64, device=src.device)
    cols = torch.arange(src.shape[1], device=src.device) * C
    with torch.no_grad():
        for _ in range(n):
            x = src.clone()
            x[:, :, :N] += sigma * torch.randn(mask.shape, device=src.device, generator=gen) * mask
            votes = model(x, static, times, lengths)[0].argmax(1)
            counts += torch.bincount(cols + votes, minlength=counts.numel()).view_as(counts)
    return counts


def host_loop_ablation(model, src, static, times, lengths, keep, n):
    """The same votes by the module: n eval forwards of B rows, each sample keeping `keep` random sensors."""
    N = src.shape[2] // 2
    B, C = src.shape[1], model._plan.n_classes
    counts = torch.zeros(B, C, dtype=torch.int64, device=src.device)
    cols = torch.arange(B, device=src.device) * C
    with torch.no_grad():
        for _ in range(n):
            kept = torch.zeros(B, N, dtype=torch.bool, device=src.device)
            for b in range(B):
                kept[b, torch.randperm(N, device=src.device)[:keep]] = True
            x = src * torch.cat([kept, kept], 1).to(src.dtype)[None]
            votes = model(x, static, times, lengths)[0].argmax(1)
            counts += torch.bincount(cols + votes, minlength=counts.numel()).view_as(counts)
    return counts


def time_calls(fn, reps):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--loop-reps", type=int, default=500)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ablate", type=int, metavar="K", help="time randomized ablation keeping K sensors")
    ap.add_argument("--exhaustive", action="store_true", help="--ablate: also the enumeration of all C(34, K) subsets")
    args = ap.parse_args()
    if args.ablate is not None:
        return main_ablation(args)
    from raindrop_b200.smoothing import SmoothingTrainStep, smooth_counts
    from raindrop_b200.train import TrainStep
    device = torch.device("cuda", 0)
    cfg = model_config("P19", dropout=0.2)
    result = {"card": card(), "config": "P19 synthetic, sigma %g, observed values" % SIGMA}
    model = build_model(cfg, device).eval()
    gen = torch.Generator(device=device).manual_seed(1)
    for B in (1, 128):
        b = {k: (v.to(device) if v is not None else None) for k, v in make_batch(cfg, B, seed=3000).items()}
        a = (b["src"], b["static"], b["times"], b["lengths"])
        loop_ms = time_calls(lambda: host_loop_counts(model, *a, SIGMA, args.loop_reps, gen), 3) / args.loop_reps
        result["host_loop_ms_per_replicate_B%d" % B] = loop_ms
        for n in (1000, 10000):
            ms = time_calls(lambda: smooth_counts(model, *a, sigma=SIGMA, n_samples=n, seed=1), args.reps)
            result["call_ms_B%d_n%d" % (B, n)] = ms
            result["host_loop_ms_B%d_n%d_extrapolated" % (B, n)] = loop_ms * n
            result["call_speedup_B%d_n%d" % (B, n)] = loop_ms * n / ms
            result["samples_per_s_B%d_n%d" % (B, n)] = 1e3 * B / ms

    B = 128
    batch = {k: (v.to(device) if v is not None else None) for k, v in make_batch(cfg, B, seed=2000).items()}
    runs = {"train": TrainStep(build_model(cfg, device).train(), B),
            "smoothing": SmoothingTrainStep(build_model(cfg, device).train(), B, sigma=SIGMA, noise_seed=1)}
    for s in runs.values():
        s.load_batch(batch)
        s.capture(warmup=args.warmup)
    times = {n: [] for n in runs}
    for _ in range(args.steps):
        for n, s in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            s.graph.replay()
            e1.record()
            e1.synchronize()
            times[n].append(e0.elapsed_time(e1))
    for n, t in times.items():
        result["step_ms_" + n] = float(np.median(t))
    print(json.dumps(result))


def time_steps(runs, steps, warmup, batch):
    for s in runs.values():
        s.load_batch(batch)
        s.capture(warmup=warmup)
    times = {n: [] for n in runs}
    for _ in range(steps):
        for n, s in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            s.graph.replay()
            e1.record()
            e1.synchronize()
            times[n].append(e0.elapsed_time(e1))
    return {"step_ms_" + n: float(np.median(t)) for n, t in times.items()}


def main_ablation(args):
    import math
    from raindrop_b200.ablation import AblationTrainStep, ablation_counts
    from raindrop_b200.smoothing import smooth_counts
    from raindrop_b200.train import TrainStep
    device = torch.device("cuda", 0)
    cfg = model_config("P19", dropout=0.2)
    K = args.ablate
    result = {"card": card(), "config": "P19 synthetic, ablation keeping %d of %d sensors" % (K, cfg["d_inp"])}
    model = build_model(cfg, device).eval()
    for B in (1, 128):
        b = {k: (v.to(device) if v is not None else None) for k, v in make_batch(cfg, B, seed=3000).items()}
        a = (b["src"], b["static"], b["times"], b["lengths"])
        loop_ms = time_calls(lambda: host_loop_ablation(model, *a, K, args.loop_reps), 3) / args.loop_reps
        result["host_loop_ms_per_replicate_B%d" % B] = loop_ms
        for n in (1000, 10000):
            # the two calls alternate, so that both see the same clocks
            ab, sm = [], []
            for _ in range(args.reps):
                ab.append(time_calls(lambda: ablation_counts(model, *a, keep=K, n_samples=n, seed=1), 1))
                sm.append(time_calls(lambda: smooth_counts(model, *a, sigma=SIGMA, n_samples=n, seed=1), 1))
            ms, ms_sm = float(np.median(ab)), float(np.median(sm))
            result["call_ms_B%d_n%d" % (B, n)] = ms
            result["smooth_counts_ms_B%d_n%d" % (B, n)] = ms_sm
            result["ratio_to_smooth_counts_B%d_n%d" % (B, n)] = ms / ms_sm
            result["host_loop_ms_B%d_n%d_extrapolated" % (B, n)] = loop_ms * n
            result["call_speedup_B%d_n%d" % (B, n)] = loop_ms * n / ms
        if args.exhaustive and B == 128:
            J = math.comb(cfg["d_inp"], K)
            result["exhaustive_subsets"] = J
            result["exhaustive_call_ms_B128"] = time_calls(
                lambda: ablation_counts(model, *a, keep=K, exhaustive=True), args.reps)
    B = 128
    batch = {k: (v.to(device) if v is not None else None) for k, v in make_batch(cfg, B, seed=2000).items()}
    result.update(time_steps({"train": TrainStep(build_model(cfg, device).train(), B),
                              "ablation": AblationTrainStep(build_model(cfg, device).train(), B, keep=K, noise_seed=1)},
                             args.steps, args.warmup, batch))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
