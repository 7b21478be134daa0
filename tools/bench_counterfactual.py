#!/usr/bin/env python
"""Counterfactual search (raindrop_b200.counterfactual.counterfactual) on the P19 synthetic configuration:

    python tools/bench_counterfactual.py [--n-search 5] [--n-steps 100] [--batches 128,3880]

At each batch size (3880 is the P19 validation split) the default search (runner-up target, beta 0.1, step 0.01,
c_init 1, one replica) runs as one device call and as the host loop a user writes without it: per FISTA step one module
forward and one torch.autograd.grad through raindrop_b200.models_rd.Raindrop_v2 (model.requires_grad_(False)), then the
proximal step, momentum, tracking and bisection in torch.  Host clock around work that ends in a device synchronise, one
timed call each after a short warm-up call.  Prints one JSON line with the times, the validity rates, and the card's name
and power limit, read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import build_model  # noqa: E402
from raindrop_b200.counterfactual import counterfactual  # noqa: E402
from raindrop_b200.synth import make_batch, model_config  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return "nvidia-smi unavailable (%r)" % (exc,)


def _margins(logits, target):
    z = logits.clone()
    z.scatter_(1, target[:, None], -float("inf"))
    cs = z.argmax(dim=1)
    return logits.gather(1, target[:, None])[:, 0] - logits.gather(1, cs[:, None])[:, 0], cs


def host_loop(model, src, static, times, lengths, beta, c_init, alpha, n_search, n_steps, kappa=0.0):
    """The same search (unit weights, no box, one replica) by module autograd.  Returns (valid [B], distance [B])."""
    N = src.shape[2] // 2
    B = src.shape[1]
    x = src[:, :, :N]
    pert = (src[:, :, N:] > 0).float()
    with torch.no_grad():
        clean = model(src, static, times, lengths)[0]
    z = clean.clone()
    z.scatter_(1, z.argmax(1, keepdim=True), -float("inf"))
    target = z.argmax(1)
    c = torch.full((B,), c_init, dtype=torch.float64, device=src.device)
    lo, hi = torch.zeros_like(c), torch.full_like(c, float("inf"))
    best_d = torch.full_like(c, float("inf"))
    best = src.clone()
    for _ in range(n_search):
        xd = torch.zeros_like(x)
        yd = torch.zeros_like(x)
        found = torch.zeros(B, dtype=torch.bool, device=src.device)
        for k in range(n_steps + 1):
            inp = src.clone()
            inp[:, :, :N] = torch.where(yd == 0, x, x + yd)
            inp.requires_grad_(k < n_steps)
            logits = model(inp, static, times, lengths)[0]
            m, cs = _margins(logits.detach().double(), target)
            valid = (m > 0) & (m >= kappa)
            found |= valid
            d = beta * yd.double().abs().sum(dim=(0, 2)) + (yd.double() ** 2).sum(dim=(0, 2))
            better = valid & (d < best_d)
            best_d = torch.where(better, d, best_d)
            best[:, better] = inp.detach()[:, better]
            if k == n_steps:
                break
            sel = (c * (m <= kappa).double()).float()
            hinge = (sel * (logits.gather(1, cs[:, None])[:, 0] - logits.gather(1, target[:, None])[:, 0])).sum()
            g = torch.autograd.grad(hinge, inp)[0][:, :, :N] * pert + 2 * yd
            v = yd - alpha * g
            xn = torch.sign(v) * torch.clamp(v.abs() - alpha * beta, min=0.0) * pert
            yd = xn + (k / (k + 3)) * (xn - xd)
            xd = xn
        hi = torch.where(found, torch.minimum(hi, c), hi)
        lo = torch.where(found, lo, torch.maximum(lo, c))
        c = torch.where(found | torch.isfinite(hi), (lo + hi) / 2, 10 * c)
    return torch.isfinite(best_d), best_d


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-search", type=int, default=5)
    ap.add_argument("--n-steps", type=int, default=100)
    ap.add_argument("--batches", default="128,3880")
    ap.add_argument("--skip-host-above", type=int, default=1 << 30, help="no host loop above this batch size")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_counterfactual.py needs a GPU")
    device = torch.device("cuda")
    cfg = model_config("P19", dropout=0.2)
    model = build_model(cfg, device).eval()
    model.requires_grad_(False)
    kw = dict(beta=0.1, c_init=1.0, step_size=0.01, n_search=args.n_search, n_steps=args.n_steps)
    result = {"metric": "counterfactual", "config": "P19", "n_search": args.n_search, "n_steps": args.n_steps, "runs": []}
    for B in (int(v) for v in args.batches.split(",")):
        b = {k: (v.to(device) if v is not None else None) for k, v in make_batch(cfg, B, seed=3000).items()}
        a = (b["src"], b["static"], b["times"], b["lengths"])
        counterfactual(model, *a, n_search=1, n_steps=2)                                   # warm-up
        t_dev, r = timed(lambda: counterfactual(model, *a, **kw))
        run = {"batch": B, "device_s": t_dev, "device_valid_rate": float(r.valid.float().mean())}
        if B <= args.skip_host_above:
            host_loop(model, *a, 0.1, 1.0, 0.01, 1, 2)                                       # warm-up
            t_host, (hv, _) = timed(lambda: host_loop(model, *a, 0.1, 1.0, 0.01, args.n_search, args.n_steps))
            run.update(host_s=t_host, host_valid_rate=float(hv.float().mean()), speedup=t_host / t_dev)
        result["runs"].append(run)
        print(json.dumps(run), file=sys.stderr)
    result["card"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
