#!/usr/bin/env python
"""DP-SGD step (raindrop_b200.privacy.DPTrainStep) against TrainStep at the same batch size.

    python tools/bench_dp_step.py [--config P19] [--steps 30] [--warmup 3]

Both steps run as captured CUDA graphs on the same synthetic batch, timed in one process, alternating step by step with
an L2 flush outside every CUDA-event pair.  A third graph holds the DP step's norm pass alone (stage 2:
rd_raindrop_v2_per_sample_grad_sqnorms on the step's forward), timed in the same rotation, so the DP step's extra time
splits into the norm pass and the rest (clip, noise, their launches).  Prints one JSON line with the medians, the
spread (p10, p90) and the card's name, power limit and SM clock read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import BENCH_CONFIGS, L2_FLUSH_BYTES, build_model, flush_l2  # noqa: E402
from raindrop_b200.synth import make_batch, model_config  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return "nvidia-smi unavailable (%r)" % (exc,)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="P19", choices=["P12", "P19", "PAM"])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    from raindrop_b200.privacy import DPTrainStep
    from raindrop_b200.train import TrainStep
    device = torch.device("cuda", 0)
    cfg_name, B, _, opts, _ = BENCH_CONFIGS[args.config]
    cfg = model_config(cfg_name, dropout=0.2)
    batch = {k: (v.to(device) if v is not None else None) for k, v in make_batch(cfg, B, seed=2000, **opts).items()}
    runs = {}
    for name in ("train", "dp"):
        model = build_model(cfg, device).train()
        if name == "dp":
            s = DPTrainStep(model, B, max_grad_norm=1.0, noise_multiplier=1.0, expected_batch_size=B, noise_seed=1)
        else:
            s = TrainStep(model, B)
        s.load_batch(batch)
        runs[name] = s
    flush = torch.empty(L2_FLUSH_BYTES // 4, dtype=torch.float32, device=device)
    for s in runs.values():
        s.capture(warmup=args.warmup)
    from raindrop_b200 import lib as L
    dp = runs["dp"]
    dp.step()                      # a forward in the workspace for the norm pass to read
    side = torch.cuda.Stream(device=device)
    side.wait_stream(torch.cuda.current_stream(device))
    with torch.cuda.stream(side):
        dp._norm_pass(L.stream_ptr(device))
    torch.cuda.current_stream(device).wait_stream(side)
    torch.cuda.synchronize()
    norm_graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(norm_graph):
        dp._norm_pass(L.stream_ptr(device))

    class NormPass:
        @staticmethod
        def step():
            norm_graph.replay()
    runs["norm_pass"] = NormPass
    ev = {k: [] for k in runs}
    for _ in range(args.steps):
        for name, s in runs.items():
            flush_l2(flush)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            s.step()
            b.record()
            ev[name].append((a, b))
    torch.cuda.synchronize()
    out = dict(config=args.config, batch=B, steps=args.steps, card=card())
    for name, pairs in ev.items():
        t = np.array([a.elapsed_time(b) for a, b in pairs])
        out[name + "_ms"] = float(np.median(t))
        out[name + "_p10_p90_ms"] = [float(np.percentile(t, 10)), float(np.percentile(t, 90))]
    out["dp_over_train"] = out["dp_ms"] / out["train_ms"]
    out["dp_extra_ms"] = out["dp_ms"] - out["train_ms"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
