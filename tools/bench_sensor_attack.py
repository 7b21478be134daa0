#!/usr/bin/env python
"""Worst-case sensor removal (raindrop_b200.sensor_attack.sensor_removal_attack) against the host loop a user writes
without it, on the P19 synthetic configuration:

    python tools/bench_sensor_attack.py [--reps 3]

Workloads: B = 128 and B = 3,880 (the size of a P19 test split), greedy and beam width 4, budget R = 3, every sensor a
player.  The loop runs the same rounds in torch: per round it builds the removed copies of every (beam set, player)
candidate, runs eval forwards of raindrop_b200.models_rd.Raindrop_v2 on them (in pieces of at most 16,384 rows), scores
them and keeps the W lowest scores per sample with torch.topk -- no deduplication and no index tie-break, so it does
less than the call.  Both are timed with a host clock around work that ends in a device synchronise, alternating call
and loop, median of --reps after one warm-up of each.  Prints one JSON line with the medians, the share of samples on
which the two agree on n_removed, and the card's name and power limit, read in the same run.
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

PIECE = 16384


def host_loop(model, src, static, times, lengths, y, R, W):
    """n_removed [B] of the beam search run round by round in torch."""
    T, B, N2 = src.shape
    N = N2 // 2
    dev = src.device
    with torch.no_grad():
        beam = torch.zeros(B, 1, N, dtype=torch.bool, device=dev)           # removed sensors per beam set
        n_removed = torch.full((B,), -1, dtype=torch.int64, device=dev)
        for r in range(R + 1):
            if r == 0:
                cand = beam
            else:
                eye = torch.eye(N, dtype=torch.bool, device=dev)
                cand = (beam[:, :, None, :] | eye[None, None]).flatten(1, 2)    # [B, w*N, N]
                fresh = (~beam[:, :, None, :] & eye[None, None]).any(-1).flatten(1, 2)
            K = cand.shape[1]
            flat = cand.reshape(B * K, N)
            idx = torch.arange(B, device=dev).repeat_interleave(K)
            logits = []
            for i in range(0, B * K, PIECE):
                g = flat[i:i + PIECE][None]
                x = src[:, idx[i:i + PIECE]]
                xs = torch.cat([torch.where(g, 0.0, x[:, :, :N]), torch.where(g, 0.0, x[:, :, N:])], 2)
                st = None if static is None else static[idx[i:i + PIECE]]
                logits.append(model(xs, st, times[:, idx[i:i + PIECE]], lengths[idx[i:i + PIECE]])[0])
            z = torch.cat(logits).view(B, K, -1)
            zy = z.gather(2, y[:, None, None].expand(B, K, 1))[..., 0]
            other = z.scatter(2, y[:, None, None].expand(B, K, 1), float("-inf")).amax(2)
            score = zy - other
            if r > 0:
                score = torch.where(fresh, score, float("inf"))
            succ = (z.argmax(2) != y[:, None]) & torch.isfinite(score)
            first = (n_removed < 0) & succ.any(1)
            n_removed = torch.where(first, r, n_removed)
            keep = torch.topk(score, min(W, K), dim=1, largest=False).indices
            beam = cand.gather(1, keep[:, :, None].expand(-1, -1, N))
    torch.cuda.synchronize()
    return n_removed


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from raindrop_b200.sensor_attack import sensor_removal_attack
    device = torch.device("cuda", 0)
    cfg = model_config("P19", dropout=0.2)
    model = build_model(cfg, device).eval()
    R = 3
    result = {"card": card(), "config": "P19 synthetic, %d players, max_removed %d" % (cfg["d_inp"], R)}
    for B in (128, 3880):
        b = make_batch(cfg, B, seed=3000, device=device)
        a = (b["src"], b["static"], b["times"], b["lengths"])
        for W in (1, 4):
            call = lambda: sensor_removal_attack(model, *a, b["y"], max_removed=R, beam_width=W).n_removed   # noqa: E731
            loop = lambda: host_loop(model, *a, b["y"], R, W)                                              # noqa: E731
            _, got = timed(call)
            _, want = timed(loop)
            tc, tl = [], []
            for _ in range(args.reps):
                tc.append(timed(call)[0])
                tl.append(timed(loop)[0])
            tag = "B%d_W%d" % (B, W)
            result["call_ms_" + tag] = float(np.median(tc))
            result["loop_ms_" + tag] = float(np.median(tl))
            result["speedup_" + tag] = float(np.median(tl) / np.median(tc))
            result["n_removed_agree_" + tag] = float((got == want).double().mean())
    print(json.dumps(result))


if __name__ == "__main__":
    main()
