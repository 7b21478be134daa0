#!/usr/bin/env python
"""Times raindrop_b200.valuation.knn_shapley_from_features (rd_knn_shapley) against a torch restatement of the same
values (fp64 torch.mm of the normalised rows, stable torch.sort, cumsum, scatter), at the record counts of the data sets'
training and validation splits, with random ReLU features of the "hidden" width:

    python tools/bench_valuation.py                   # P19 (against 3,880 queries and leave-one-out), P12, PAM

Both sides start from the same device-normalised rows, so they rank the same similarities up to the last bits of the
dot; the maximal differences of values and utility are printed.  Times are CUDA-event medians over --reps calls after
--warmup.  Prints one JSON line per shape and the card's name and power limit, read in the same run.
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

from raindrop_b200 import lib as L  # noqa: E402
from raindrop_b200 import valuation as VA  # noqa: E402

# (name, n_train, n_query or None for leave-one-out, feature width of the "hidden" layer, classes)
SHAPES = [("P19", 31_000, 3_880, 186, 2), ("P19-loo", 31_000, None, 186, 2), ("P12", 9_590, 1_199, 196, 2),
          ("P12-loo", 9_590, None, 196, 2), ("PAM", 4_266, 533, 84, 8), ("PAM-loo", 4_266, None, 84, 8)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def torch_knn_shapley(bank, n, queries, nq, yt, yq, k, loo, chunk=256):
    """The restatement: (values [n] = mean over queries, utility [nq])."""
    B = bank[:n].double()
    values = torch.zeros(n, dtype=torch.float64, device=bank.device)
    util = torch.empty(nq, dtype=torch.float64, device=bank.device)
    N = n - 1 if loo else n
    j = torch.arange(1, N + 1, dtype=torch.float64, device=bank.device)
    c = torch.minimum(j, torch.tensor(float(k), dtype=torch.float64, device=bank.device)) / (j * k)
    w = torch.where(j > k, 1.0 / (j * (j - 1)).clamp_min(1), torch.zeros_like(j))
    for q0 in range(0, nq, chunk):
        q1 = min(nq, q0 + chunk)
        S = queries[q0:q1].double() @ B.T
        if loo:
            S[torch.arange(q1 - q0), torch.arange(q0, q1)] = -float("inf")      # the query's own record last
        order = torch.sort(S, dim=1, descending=True, stable=True).indices[:, :N]
        m = (yt[order] == yq[q0:q1, None]).double()
        t = m * w
        tail = torch.flip(torch.cumsum(torch.flip(t, [1]), 1), [1]) - t       # sum over j > r
        s = m * c - tail
        per = torch.zeros(q1 - q0, n, dtype=torch.float64, device=bank.device).scatter_(1, order, s)
        values += per.sum(0)
        util[q0:q1] = m[:, :min(k, N)].sum(1) / k
    return values / nq, util


def timed(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), fn()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default=",".join(s[0] for s in SHAPES))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_valuation.py measures on the GPU and needs CUDA")
    dev_card = card()
    lib = L.load()
    for name, n, nq, F, C in SHAPES:
        if name not in a.shapes.split(","):
            continue
        g = torch.Generator(device="cuda").manual_seed(n + F)
        ft = torch.relu(torch.randn(n, F, device="cuda", generator=g))
        yt = torch.randint(0, C, (n,), device="cuda", generator=g)
        loo = nq is None
        fq = None if loo else torch.relu(torch.randn(nq, F, device="cuda", generator=g))
        yq = None if loo else torch.randint(0, C, (nq,), device="cuda", generator=g)
        Fp = (F + 3) // 4 * 4
        bank = VA._bank(lib, ft, n, F, Fp)
        queries, m = (bank, n) if loo else (VA._bank(lib, fq, nq, F, Fp), nq)
        t_dev, res = timed(lambda: VA.knn_shapley_from_features(ft, yt, fq, yq, k=a.k), a.warmup, a.reps)
        t_ref, (v_ref, u_ref) = timed(lambda: torch_knn_shapley(bank, n, queries, m, yt, yt if loo else yq, a.k, loo),
                                      a.warmup, a.reps)
        print(json.dumps(dict(shape=name, n_train=n, n_query=m, F=F, classes=C, k=a.k, device_ms=round(t_dev, 3),
                              torch_ms=round(t_ref, 3),
                              values_max_diff=float((res.values - v_ref).abs().max()),
                              utility_max_diff=float((res.utility - u_ref).abs().max()),
                              chunk=VA._chunk(lib, n, Fp, m, None), card=dev_card)), flush=True)


if __name__ == "__main__":
    main()
