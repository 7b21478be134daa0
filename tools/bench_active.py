#!/usr/bin/env python
"""Batch active learning: batch_bald and badge_from_features against a torch restatement of the same greedy loops.

    python tools/bench_active.py [--shapes P19 PAM] [--k 100] [--steps 3]

Shapes (synthetic replicates' logits [M, N, C] and hidden features [N, F] from a fixed seed):
  P19  N = 31,000, C = 2, M = 100          PAM  N = 5,333, C = 8, M = 100
torch: per greedy step of BatchBALD, the chunked product P_A^T p (torch.matmul in fp32, TF32 off as torch's default)
and -sum xlogy over the configurations, with the same scaled rows, exact / sampled switch and fp64 bookkeeping; its
BADGE materialises the embeddings [N, C (F + 1)], updates D^2 from their squared norms and a matrix-vector product and
draws with torch.multinomial.  Both sides run to completion before the clock stops (host clock around a device synchronise,
median of --steps calls after one warm-up call).  Prints one JSON line per shape, with the card's name and power limit
read in the same run.  The torch loop is a timing yardstick, not a reference: the tests compare against
oracle/active_oracle.py.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from raindrop_b200 import active as AC  # noqa: E402

SHAPES = {"P19": (31_000, 2, 100), "PAM": (5_333, 8, 100)}


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return "nvidia-smi unavailable (%r)" % (exc,)


def torch_batch_bald(logits, k, n_configs, seed, chunk=4096):
    """The greedy loop with torch ops: exact rows while C^i <= n_configs, then sampled rows (torch's own generator)."""
    M, N, C = logits.shape
    p = torch.softmax(logits.double(), dim=2).float()                     # [M, N, C]
    ce = -(torch.special.xlogy(p.double(), p.double())).sum(2).mean(0)     # [N]
    pf = p.reshape(M, N * C)
    rows = torch.ones(1, M, device=logits.device)
    ls = torch.zeros(1, dtype=torch.float64, device=logits.device)
    w = torch.full((1,), 1.0 / M, dtype=torch.float64, device=logits.device)
    chosen = torch.zeros(N, dtype=torch.bool, device=logits.device)
    condA = torch.zeros((), dtype=torch.float64, device=logits.device)
    g = torch.Generator(device=logits.device).manual_seed(seed)
    ms, picks, exact, R = None, [], True, 1
    for i in range(k):
        H = torch.empty(N, dtype=torch.float64, device=logits.device)
        Lr = (ls - math.log(M))[:, None]
        for n0 in range(0, N, chunk):
            n1 = min(N, n0 + chunk)
            Q = torch.matmul(rows, pf[:, n0 * C:n1 * C]).double()          # [R, nc C]
            v = (torch.special.xlogy(Q, Q) + Q * Lr).reshape(R, n1 - n0, C).sum(2)
            H[n0:n1] = -(w[:, None] * v).sum(0)
        sc = torch.where(chosen, torch.full_like(H, -math.inf), H - condA - ce)
        best = torch.argmax(sc)
        picks.append(best)
        chosen[best] = True
        condA = condA + ce[best]
        if i + 1 == k:
            break
        if exact and R * C <= n_configs:
            new = (rows[:, None, :] * p[:, best, :].t()[None]).reshape(R * C, M)
            mx = new.max(1).values.clamp_min(1e-38)
            rows, ls = new / mx[:, None], ls.repeat_interleave(C) + mx.double().log()
            w = ls.exp() / M
            R *= C
            continue
        todo = [best]
        if exact:
            exact, R = False, n_configs
            ms = torch.randint(0, M, (R,), generator=g, device=logits.device)
            rows = torch.ones(R, M, device=logits.device)
            ls = torch.zeros(R, dtype=torch.float64, device=logits.device)
            todo = picks
        for a in todo:
            y = torch.multinomial(p[ms, a, :], 1, generator=g)[:, 0]
            new = rows * p[:, a, :].t()[y]
            mx = new.max(1).values.clamp_min(1e-38)
            rows, ls = new / mx[:, None], ls + mx.double().log()
        w = 1.0 / (R * rows.double().sum(1))
    return torch.stack(picks)


def torch_badge(hidden, logits, k, seed):
    N, F = hidden.shape
    p = torch.softmax(logits.double(), 1)
    a = p.clone()
    a[torch.arange(N, device=p.device), logits.argmax(1)] -= 1.0
    ht = torch.cat([hidden.double(), torch.ones(N, 1, dtype=torch.float64, device=p.device)], 1)
    g = (a[:, :, None] * ht[:, None, :]).reshape(N, -1)                   # the materialised embeddings
    gn = (g * g).sum(1)
    pick = torch.argmax(gn)
    picks = [pick]
    d2 = torch.full((N,), math.inf, dtype=torch.float64, device=p.device)
    gen = torch.Generator(device=p.device).manual_seed(seed)
    for _ in range(1, k):
        d2 = torch.minimum(d2, (gn + gn[pick] - 2.0 * (g @ g[pick])).clamp_min(0.0))
        d2[torch.stack(picks)] = 0.0
        pick = torch.multinomial(d2, 1, generator=gen)[0]
        picks.append(pick)
    return torch.stack(picks)


def timed(fn, steps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--shapes", nargs="*", default=list(SHAPES))
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--n-configs", type=int, default=10_000)
    ap.add_argument("--features", type=int, default=64, help="F of the hidden features")
    ap.add_argument("--steps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_active.py measures on the GPU: no CUDA device")
    dev = torch.device("cuda")
    for name in args.shapes:
        N, C, M = SHAPES[name]
        gen = torch.Generator(device=dev).manual_seed(0)
        centre = torch.randn(1, N, C, device=dev, generator=gen) * 1.5
        logits = (centre + torch.randn(M, N, C, device=dev, generator=gen) * 1.5).contiguous()
        hidden = torch.relu(torch.randn(N, args.features, device=dev, generator=gen))
        out = dict(shape=name, N=N, C=C, M=M, k=args.k, n_configs=args.n_configs, F=args.features, card=card())
        out["batch_bald_s"] = timed(lambda: AC.batch_bald(logits, args.k, n_configs=args.n_configs), args.steps)
        out["torch_batch_bald_s"] = timed(lambda: torch_batch_bald(logits, args.k, args.n_configs, 0), args.steps)
        out["badge_s"] = timed(lambda: AC.badge_from_features(hidden, logits[0], args.k), args.steps)
        out["torch_badge_s"] = timed(lambda: torch_badge(hidden, logits[0], args.k, 0), args.steps)
        ours = AC.batch_bald(logits, args.k, n_configs=args.n_configs)
        ref = torch_batch_bald(logits, args.k, args.n_configs, 0)
        ex = int(ours.exact.sum())
        out["exact_picks"] = ex
        out["exact_picks_agree"] = int((ours.indices[:ex] == ref[:ex]).sum())
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
