#!/usr/bin/env python
"""Accuracy of TracIn-RP (influence.project / tracin_sketch) against exact TracIn (influence.tracin) on a P19-shaped
synthetic set, for several projection dims.  Prints one JSON line per dim:
  err_normalised      |sketch - exact| / (||g_q|| ||g_t||): median, 99th percentile and max over every score
  spearman            the Spearman correlation of each query's row of scores: median and min over the queries
  top10_overlap       |top-10 proponents (largest scores) of sketch and exact| / 10, the same for the opponents (most
                      negative): mean over the queries
The gradient norms come from self_influence.  One checkpoint (the synthetic weights), each query scored with its
predicted class.

    python tools/tracin_rp_accuracy.py --n-query 64 --n-train 2048 --dims 1024 4096 16384
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
from scipy.stats import spearmanr

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

from helpers import build_dropin, to_dev  # noqa: E402
from raindrop_b200 import influence as IF  # noqa: E402
from raindrop_b200.synth import make_batch, model_config  # noqa: E402


def top_overlap(a, b, k):
    """Mean over rows of |top-k(a) & top-k(b)| / k (largest values)."""
    ia, ib = np.argsort(-a, axis=1)[:, :k], np.argsort(-b, axis=1)[:, :k]
    return float(np.mean([len(set(x) & set(y)) / k for x, y in zip(ia, ib)]))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--shape", default="P19")
    ap.add_argument("--n-query", type=int, default=64)
    ap.add_argument("--n-train", type=int, default=2048)
    ap.add_argument("--dims", type=int, nargs="+", default=[1024, 4096, 16384])
    ap.add_argument("--seed", type=int, default=0, help="projection seed")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tracin_rp_accuracy runs on a CUDA device")
    cfg = model_config(args.shape, dropout=0.2)
    model = build_dropin(cfg, 21)
    model.eval()
    dq = to_dev(make_batch(cfg, args.n_query, seed=71))
    dt = to_dev(make_batch(cfg, args.n_train, seed=72))
    q = dict(src=dq["src"], static=dq["static"], times=dq["times"], lengths=dq["lengths"], y=None)
    t = dict(src=dt["src"], static=dt["static"], times=dt["times"], lengths=dt["lengths"], y=dt["y"])
    exact = IF.tracin(model, q, t).cpu().numpy()
    with torch.no_grad():                  # the queries' norms are those of their predicted class
        logits, _, _ = model.forward(dq["src"], dq["static"], dq["times"], dq["lengths"])
    nq = IF.self_influence(model, dict(q, y=logits.argmax(1))).sqrt().cpu().numpy()
    nt = IF.self_influence(model, t).sqrt().cpu().numpy()
    norm = nq[:, None] * nt[None, :]
    for dim in args.dims:
        sk = IF.tracin_sketch(IF.project(model, q, dim=dim, seed=args.seed),
                              IF.project(model, t, dim=dim, seed=args.seed)).cpu().numpy()
        err = np.abs(sk - exact) / norm
        rho = np.array([spearmanr(sk[i], exact[i])[0] for i in range(len(sk))])
        print(json.dumps(dict(shape=args.shape, dim=dim, n_query=args.n_query, n_train=args.n_train, seed=args.seed,
                              err_normalised=dict(median=float(np.median(err)), p99=float(np.quantile(err, 0.99)),
                                                  max=float(err.max()), sigma_1_over_sqrt_dim=float(dim ** -0.5)),
                              spearman=dict(median=float(np.median(rho)), min=float(rho.min())),
                              top10_overlap=dict(proponents=top_overlap(sk, exact, 10),
                                                 opponents=top_overlap(-sk, -exact, 10)))), flush=True)


if __name__ == "__main__":
    main()
