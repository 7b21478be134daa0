#!/usr/bin/env python
"""Throughput of input gradients (the attribution workload: saliency maps, integrated gradients).

    python tools/bench_input_grad.py [--config P19] [--steps 30] [--warmup 5]

One call = eval-mode models_rd.Raindrop_v2.forward with frozen parameters (requires_grad_(False)) on the configuration's
per-GPU batch, then torch.autograd.grad(logits[:, 0].sum(), [src, static, times]).  Timing follows bench.py: an L2 flush
before every call outside the CUDA-event pair, median over calls.  Prints one JSON line with samples/s, ms per call, this
library's kernel launches per call (rd_launch_count; torch's own ops are not counted) and the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import BENCH_CONFIGS, L2_FLUSH_BYTES, build_model, summarize, timed_steps  # noqa: E402
from raindrop_b200.synth import make_batch, model_config  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return "nvidia-smi unavailable (%r)" % (exc,)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="P19", choices=sorted(BENCH_CONFIGS))
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    from raindrop_b200 import lib as L
    lib = L.load()
    device = torch.device("cuda", 0)
    cfg_name, batch, _, opts, _ = BENCH_CONFIGS[args.config]
    cfg = model_config(cfg_name, dropout=0.2)
    model = build_model(cfg, device).eval().requires_grad_(False)
    b = {k: (v.to(device) if v is not None else None) for k, v in make_batch(cfg, batch, seed=2000, **opts).items()}
    src = b["src"].clone().requires_grad_(True)
    times = b["times"].clone().requires_grad_(True)
    static = b["static"].clone().requires_grad_(True) if b["static"] is not None else None
    inputs = [t for t in (src, static, times) if t is not None]

    def call():
        logits, _, _ = model.forward(src, static, times, b["lengths"])
        torch.autograd.grad(logits[:, 0].sum(), inputs)

    for _ in range(max(1, args.warmup)):
        call()
    torch.cuda.synchronize()
    n0 = lib.rd_launch_count()
    call()
    launches = int(lib.rd_launch_count() - n0)
    flush = torch.empty(L2_FLUSH_BYTES // 4, dtype=torch.float32, device=device)
    t = summarize(timed_steps(call, args.steps, flush), 1, device)
    print(json.dumps({"metric": "input gradients, samples/s (%s-shape synthetic)" % cfg_name,
                      "value": round(batch / (t["median"] * 1e-3), 1), "unit": "samples/s", "batch": batch,
                      "ms_per_call": round(t["median"], 4), "ms_p90": round(t["p90"], 4), "launches_per_call": launches,
                      "steps": args.steps, "card": card()}), flush=True)


if __name__ == "__main__":
    main()
