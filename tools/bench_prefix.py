#!/usr/bin/env python
"""Early-prediction logits (raindrop_b200.early.prefix_predict) against the loop a user writes without it, on the P19
synthetic configuration:

    python tools/bench_prefix.py [--reps 5]

Two workloads: B = 128 with K = 60 prefixes (every row count 1 .. 60) and B = 3,880 (the size of a P19 test split)
with K = 12 row counts spread over the record.  The loop truncates the batch in torch for each prefix (rows t >= r
written as 0 in src and times, lengths recounted) and runs one eval forward of raindrop_b200.models_rd.Raindrop_v2 per
prefix.  Both are timed with a host clock around work that ends in a device synchronise, alternating call and loop,
median of --reps after one warm-up of each.  The largest absolute difference between the two logits is reported (the
call's forward runs on more rows per launch, so its ob-prop arithmetic may differ in the last bits).  Prints one JSON
line with the medians and the card's name and power limit, read in the same run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import build_model  # noqa: E402
from bench_smoothing import card  # noqa: E402
from raindrop_b200.synth import make_batch, model_config  # noqa: E402


def module_loop(model, src, static, times, lengths, rows):
    """logits [B, K, C] of one module forward per torch-truncated prefix."""
    T = src.shape[0]
    t_idx = torch.arange(T, device=src.device)[:, None]
    out = []
    with torch.no_grad():
        for r in rows:
            keep = t_idx < int(r)
            tm = torch.where(keep, times, 0.0)
            ln = lengths if r >= T else torch.minimum(lengths, (tm > 0).sum(0))
            out.append(model(torch.where(keep[:, :, None], src, 0.0), static, tm, ln)[0])
    return torch.stack(out, 1)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    from raindrop_b200.early import prefix_predict
    device = torch.device("cuda", 0)
    cfg = model_config("P19", dropout=0.2)
    T = cfg["max_len"]
    model = build_model(cfg, device).eval()
    result = {"card": card(), "config": "P19 synthetic, eval logits of K prefixes"}
    for B, rows in ((128, np.arange(1, T + 1)), (3880, np.linspace(T / 12, T, 12).round().astype(np.int64))):
        b = make_batch(cfg, B, seed=3000, device=device)
        a = (b["src"], b["static"], b["times"], b["lengths"])
        call = lambda: prefix_predict(model, *a, rows=rows).logits          # noqa: E731
        loop = lambda: module_loop(model, *a, rows)                         # noqa: E731
        _, got = timed(call)
        _, want = timed(loop)
        tc, tl = [], []
        for _ in range(args.reps):
            tc.append(timed(call)[0])
            tl.append(timed(loop)[0])
        tag = "B%d_K%d" % (B, len(rows))
        result["call_ms_" + tag] = float(np.median(tc))
        result["loop_ms_" + tag] = float(np.median(tl))
        result["speedup_" + tag] = float(np.median(tl) / np.median(tc))
        result["max_abs_diff_" + tag] = float((got - want).abs().max())
    print(json.dumps(result))


if __name__ == "__main__":
    main()
