#!/usr/bin/env python
"""Accuracy of KernelSHAP against permutation sampling at equal coalition budgets.

    python tools/kernel_shap_accuracy.py --cpu                  # TINY fixture values against exact Shapley values
    python tools/kernel_shap_accuracy.py [--config P19] [--batch 128] [--repeats 3] [--ref-permutations 200]

Budgets are counts of coalition forwards (the two endpoints not counted).  Permutation sampling with m permutations
costs m*(P-1) coalitions, so each budget is rounded to m = max(1, round(budget / (P-1))) permutations and KernelSHAP gets
exactly m*(P-1) coalitions too.  The error is the MSE over (sample, player) against a reference, averaged over
--repeats seeds, and is printed as one JSON line per (players, budget).

GPU half: the P19-shape synthetic model and batch of bench.py (eval mode, zero baselines, target = the labels, the
static vector one more player), over (a) one player per sensor and (b) (sensor, 6-unit time window) players
(time_window_mask, 6 windows).  There are no exact values at these P, so the reference is shapley_value_sampling with
--ref-permutations permutations, run as two independent halves: ref = their mean, and MSE(half1 - half2) / 4 estimates
the reference's own MSE (reported as ref_mse_estimate; an estimator's MSE below it is not resolved).

CPU half (--cpu): the reference coalition values of tests/golden/kernel_shap.npz (every coalition of the TINY cases,
P = 6), exact Shapley values from all_coalitions, and both estimators evaluated on the stored values in fp64.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from raindrop_b200 import attribution as A  # noqa: E402

BUDGETS = (340, 850, 1700, 5100)
CPU_BUDGETS = (10, 25, 50, 100)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return "nvidia-smi unavailable (%r)" % (exc,)


def permutation_estimate(values, orders):
    """Permutation sampling on a value table [2^P, B] (rows in itertools.product order: player 0 is the top bit)."""
    P = orders.shape[1]
    phi = np.zeros((values.shape[1], P))
    for p in orders:
        row, prev = 0, values[0]
        for g in p:
            row |= 1 << (P - 1 - g)
            cur = values[row]
            phi[:, g] += cur - prev
            prev = cur
    return phi / len(orders)


def cpu_half(args):
    z = np.load(os.path.join(ROOT, "tests", "golden", "kernel_shap.npz"))
    for name in ("tiny_dense", "tiny_t0", "tiny_sparse", "tiny8_nostatic"):
        vals = z[name + ".values"]
        P = vals.shape[0].bit_length() - 1

        def rows(Z):
            return (Z.astype(np.int64) << np.arange(P - 1, -1, -1)).sum(axis=1)

        def kshap(Z, w):
            return A.kernel_shap_from_values(vals[rows(Z)], vals[0], vals[-1], Z, w)
        exact = kshap(*A.all_coalitions(P))
        for budget in CPU_BUDGETS:
            m = max(1, round(budget / (P - 1)))
            e_ks, e_pm = [], []
            for r in range(args.cpu_repeats):
                e_ks.append(np.mean((kshap(*A.sample_coalitions(P, m * (P - 1), seed=r)) - exact) ** 2))
                e_pm.append(np.mean((permutation_estimate(vals, A.sample_permutations(P, m, seed=r)) - exact) ** 2))
            print(json.dumps({"half": "cpu", "case": name, "players": P, "coalitions": m * (P - 1), "permutations": m,
                              "repeats": args.cpu_repeats, "reference": "exact (all_coalitions on the reference values)",
                              "mse_kernel_shap": float(np.mean(e_ks)), "mse_permutation": float(np.mean(e_pm)),
                              "ratio": float(np.mean(e_ks) / np.mean(e_pm))}), flush=True)


def gpu_half(args):
    import torch
    from bench import BENCH_CONFIGS, build_model
    from raindrop_b200.synth import make_batch, model_config
    device = torch.device("cuda", 0)
    cfg_name, batch, _, opts, _ = BENCH_CONFIGS[args.config]
    cfg = model_config(cfg_name, dropout=0.2)
    model = build_model(cfg, device).eval().requires_grad_(False)
    B = args.batch or batch
    b = {k: (v.to(device) if v is not None else None) for k, v in make_batch(cfg, B, seed=2000, **opts).items()}
    call = (model, b["src"], b["static"], b["times"], b["lengths"])
    N = cfg["d_inp"]
    mask, n_win = A.time_window_mask(b["times"], args.window, n_windows=args.n_windows, sensor_groups=N)
    info = card()
    for what, kw in (("sensors", {}), ("(sensor, %g-unit window)" % args.window, dict(feature_mask=mask))):
        half = args.ref_permutations // 2
        h = [_cat(*A.shapley_value_sampling(*call, target=b["y"], n_samples=half, seed=10_000 + i, **kw))
             for i in range(2)]
        ref = (h[0].double() + h[1].double()) / 2
        ref_mse = float(((h[0].double() - h[1].double()) ** 2).mean()) / 4
        P = ref.shape[1]
        for budget in BUDGETS:
            m = max(1, round(budget / (P - 1)))
            e_ks, e_pm = [], []
            for r in range(args.repeats):
                ks = _cat(*A.kernel_shap(*call, target=b["y"], n_samples=m * (P - 1), seed=r, **kw))
                pm = _cat(*A.shapley_value_sampling(*call, target=b["y"], n_samples=m, seed=r, **kw))
                e_ks.append(float(((ks.double() - ref) ** 2).mean()))
                e_pm.append(float(((pm.double() - ref) ** 2).mean()))
            print(json.dumps({"half": "gpu", "config": cfg_name, "batch": B, "players": what, "n_players": P,
                              "coalitions": m * (P - 1), "permutations": m, "repeats": args.repeats,
                              "reference": "shapley_value_sampling, %d permutations (two halves of %d)"
                                           % (2 * half, half),
                              "ref_mse_estimate": ref_mse, "mse_kernel_shap": float(np.mean(e_ks)),
                              "mse_permutation": float(np.mean(e_pm)), "ratio": float(np.mean(e_ks) / np.mean(e_pm)),
                              "card": info}), flush=True)


def _cat(a_players, a_static):
    import torch
    return a_players if a_static is None else torch.cat([a_players, a_static[:, None]], dim=1)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--cpu", action="store_true", help="the CPU half on the TINY fixture values")
    ap.add_argument("--cpu-repeats", type=int, default=200)
    ap.add_argument("--config", default="P19")
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--ref-permutations", type=int, default=200)
    ap.add_argument("--window", type=float, default=6.0)
    ap.add_argument("--n-windows", type=int, default=6)
    args = ap.parse_args()
    if args.cpu:
        cpu_half(args)
    else:
        gpu_half(args)


if __name__ == "__main__":
    main()
