#!/usr/bin/env python
"""PGD attacks (raindrop_b200.adversarial.pgd) and PGD adversarial training (AdversarialTrainStep) on the P19 synthetic
configuration:

    python tools/bench_adversarial.py [--reps 5] [--steps 20] [--warmup 3]

1. PGD-10 L-inf (eps 0.1, random start) at B = 128 and at B = 3880 (the P19 validation split), as one device call and
   as the host loop a user writes without it: per iteration one module forward and one torch.autograd.grad through
   raindrop_b200.models_rd.Raindrop_v2, then the sign step, clip and mask in torch.  Host clock around work that ends
   in a device synchronise, median of --reps calls after one warm-up call each.
2. AdversarialTrainStep at K = 1, 3, 10 against TrainStep at B = 128, all as captured CUDA graphs in one process,
   alternating step by step with CUDA events (median over --steps replays).
Prints one JSON line with the medians and the card's name and power limit, read in the same run.
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

EPS, K = 0.1, 10


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return "nvidia-smi unavailable (%r)" % (exc,)


def host_loop_pgd(model, src, static, times, lengths, y, eps, n_steps, alpha, seed):
    """PGD-K L-inf by module autograd: the same attack as pgd() (random start, best iterate by per-sample loss)."""
    N = src.shape[2] // 2
    mask = (src[:, :, N:] > 0).float()
    g = torch.Generator(device=src.device).manual_seed(seed)
    delta = (torch.rand(src[:, :, :N].shape, device=src.device, generator=g) * 2 - 1) * eps * mask
    best_loss = torch.full((src.shape[1],), -float("inf"), device=src.device)
    best = src.clone()
    for k in range(n_steps + 1):
        x = src.clone()
        x[:, :, :N] = src[:, :, :N] + delta
        x.requires_grad_(k < n_steps)
        logits = model(x, static, times, lengths)[0]
        loss = torch.nn.functional.cross_entropy(logits, y, reduction="none")
        better = loss.detach() > best_loss
        best_loss = torch.where(better, loss.detach(), best_loss)
        best[:, better] = x.detach()[:, better]
        if k == n_steps:
            break
        grad = torch.autograd.grad(loss.sum(), x)[0][:, :, :N]
        delta = (delta + alpha * grad.sign()).clamp(-eps, eps) * mask
    return best, best_loss


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
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    from raindrop_b200.adversarial import AdversarialTrainStep, pgd
    from raindrop_b200.train import TrainStep
    device = torch.device("cuda", 0)
    cfg = model_config("P19", dropout=0.2)
    result = {"card": card(), "config": "P19 synthetic, PGD-%d L-inf eps %g, random start" % (K, EPS)}
    model = build_model(cfg, device).eval()
    for B in (128, 3880):
        b = {k: (v.to(device) if v is not None else None) for k, v in make_batch(cfg, B, seed=3000).items()}
        a = (b["src"], b["static"], b["times"], b["lengths"])
        result["pgd_call_ms_B%d" % B] = time_calls(lambda: pgd(model, *a, b["y"], eps=EPS, n_steps=K, seed=1), args.reps)
        result["pgd_host_loop_ms_B%d" % B] = time_calls(
            lambda: host_loop_pgd(model, *a, b["y"], EPS, K, 2.5 * EPS / K, 1), args.reps)

    B = 128
    batch = {k: (v.to(device) if v is not None else None) for k, v in make_batch(cfg, B, seed=2000).items()}
    runs = {"train": TrainStep(build_model(cfg, device).train(), B)}
    for k in (1, 3, 10):
        runs["adv_k%d" % k] = AdversarialTrainStep(build_model(cfg, device).train(), B, eps=EPS, n_steps=k, attack_seed=1)
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


if __name__ == "__main__":
    main()
