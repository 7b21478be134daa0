#!/usr/bin/env python
"""How close EK-FAC influence (raindrop_b200.influence.ekfac_*) comes to the exact damped inverse of the empirical Fisher,
on one small field group at TINY.  The exact reference is built densely in float64 from per_sample_grads rows:
F = (1/n) sum_t g_t g_t^T over the group's columns, score = g_q^T (F + lambda I)^-1 g_t, with lambda = 0.1 mean eig(F).
EK-FAC (empirical Fisher, its default damping) and TracIn are scored on the same pairs; prints one JSON line with their
Spearman correlations against the exact scores, overall and per query (mean).

    python tools/ekfac_accuracy.py --n-train 400 --n-query 16
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="TINY")
    ap.add_argument("--n-train", type=int, default=400)
    ap.add_argument("--n-query", type=int, default=16)
    ap.add_argument("--block", type=int, default=1, help="index into influence.kfac_blocks (default: out_proj of layer 0)")
    a = ap.parse_args()
    cfg = model_config(a.shape, dropout=0.2)
    model = build_dropin(cfg, 21)
    model.eval()
    dt, dq = to_dev(make_batch(cfg, a.n_train, seed=2)), to_dev(make_batch(cfg, a.n_query, seed=3))
    w, b, nout, kin = IF.kfac_blocks(model)[a.block]
    fields = [w, b]
    q = lambda d: dict(src=d["src"], static=d["static"], times=d["times"], lengths=d["lengths"], y=d["y"])
    f = IF.ekfac_factors(model, q(dt), fisher="empirical", fields=fields)
    ek = IF.ekfac_influence(model, q(dq), q(dt), f).cpu().numpy()
    tr = IF.tracin(model, q(dq), q(dt), fields=fields).cpu().numpy()
    off = {k: o for k, o, _ in IF.grad_layout(model)}
    cols = np.r_[off[w]:off[w] + nout * kin, off[b]:off[b] + nout]

    def rows(d):
        R = IF._row_batch(IF.L.load(), model._plan, IF._bucket_length(IF.grad_layout(model)))
        out = [IF.per_sample_grads(model, d["src"][:, i:i + R], None if d["static"] is None else d["static"][i:i + R],
                                   d["times"][:, i:i + R], d["lengths"][i:i + R], d["y"][i:i + R])
               for i in range(0, d["src"].shape[1], R)]
        return torch.cat(out).double().cpu().numpy()[:, cols]
    Gt, Gq = rows(dt), rows(dq)
    Fm = Gt.T @ Gt / len(Gt)
    lam = 0.1 * np.linalg.eigvalsh(Fm).mean()
    exact = Gq @ np.linalg.solve(Fm + lam * np.eye(len(Fm)), Gt.T)
    per_q = lambda s: float(np.mean([spearmanr(s[i], exact[i])[0] for i in range(len(s))]))
    print(json.dumps(dict(shape=a.shape, block=w, columns=len(cols), n_train=a.n_train, n_query=a.n_query,
                          spearman_ekfac=float(spearmanr(ek.ravel(), exact.ravel())[0]),
                          spearman_tracin=float(spearmanr(tr.ravel(), exact.ravel())[0]),
                          spearman_per_query_ekfac=per_q(ek), spearman_per_query_tracin=per_q(tr))), flush=True)


if __name__ == "__main__":
    main()
