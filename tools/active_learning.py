#!/usr/bin/env python
"""Simulated active learning for Raindrop_v2: how fast do the acquisition functions of raindrop_b200.active buy test
accuracy, label by label?

    python tools/active_learning.py --shape P19 --n-pool 4000 --n-test 1000 --seed-labels 100 --k 100 --rounds 5

Data: the planted-label synthetic data of tools/attribution_lds.py (make_batch samples of --shape, labelled by the sign
of the observed-value mean of sensors 0 and 1, --label-noise of them flipped); the first --n-pool records are the pool,
the next --n-test the test set.
Loop, per method: start from the same --seed-labels random labelled records; then --rounds times: train a fresh model
(same initial weights for every method) with TrainStep for --epochs epochs on the labelled set, record test AUROC and
AUPRC, and acquire --k more labels from the unlabelled rest with
  random     uniformly at random;
  bald       the k largest single-point mutual informations (batch_bald's `bald` over pool_logits, M = --mc);
  batchbald  batch_bald over the same logits (--n-configs);
  badge      badge on the model's eval forward.
Prints one JSON line per (method, round) and writes labelled-set sizes, AUROC and AUPRC per method to --out (.npz).
An evaluation, not a test: whichever way the curves come out, they are what was measured.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

METHODS = ("random", "bald", "batchbald", "badge")


def _load(args):
    """(cfg, DeviceDataset over pool + test, pool indices, test indices, labels [n] numpy)."""
    from attribution_lds import planted_data
    from raindrop_b200.data import DeviceDataset
    from raindrop_b200.synth import model_config
    cfg = model_config(args.shape, dropout=args.dropout)
    cfg["n_classes"] = 2
    n = args.n_pool + args.n_test
    b = planted_data(cfg, n, args.seed, args.label_noise)
    ds = DeviceDataset(b["src"], b["static"], b["times"], b["y"])
    return cfg, ds, np.arange(args.n_pool), np.arange(args.n_pool, n), b["y"].numpy()


def _evaluate(model, ds, test, labels):
    from raindrop_b200.ood import _auroc, _average_precision, features
    from raindrop_b200.influence import _source
    _, fetch = _source((ds, torch.from_numpy(test)), "test")
    src, static, times, lengths, _ = fetch(0, len(test))
    _, z = features(model, src, static, times, lengths)
    s = torch.softmax(z.double(), 1)[:, 1].cpu().numpy()
    y = labels[test]
    return _auroc(s[y == 1], s[y == 0]), _average_precision(s[y == 1], s[y == 0])


def _acquire(method, model, ds, unl, k, args, rng):
    from raindrop_b200 import active as AC
    if method == "random":
        return rng.choice(unl, size=k, replace=False)
    if method == "badge":
        return unl[AC.badge(model, (ds, torch.from_numpy(unl)), k, seed=args.seed).indices.cpu().numpy()]
    logits = AC.pool_logits(model, (ds, torch.from_numpy(unl)), n_samples=args.mc, seed=args.seed)
    res = AC.batch_bald(logits, k, n_configs=args.n_configs, seed=args.seed)
    if method == "bald":
        return unl[torch.topk(res.bald, k).indices.cpu().numpy()]
    return unl[res.indices.cpu().numpy()]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--shape", default="P19")
    ap.add_argument("--n-pool", type=int, default=4000)
    ap.add_argument("--n-test", type=int, default=1000)
    ap.add_argument("--seed-labels", type=int, default=100)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--batch-size", type=int, default=32)
    ap.add_argument("--lr", type=float, default=1e-3)
    ap.add_argument("--dropout", type=float, default=0.2)
    ap.add_argument("--label-noise", type=float, default=0.1)
    ap.add_argument("--mc", type=int, default=30, help="Monte Carlo dropout replicates")
    ap.add_argument("--n-configs", type=int, default=10_000)
    ap.add_argument("--methods", nargs="*", default=list(METHODS), choices=METHODS)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default="active_learning.npz")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("active_learning.py trains on the GPU: no CUDA device")
    from attribution_lds import card, train_model
    cfg, ds, pool, test, labels = _load(args)
    first = np.random.default_rng(args.seed).choice(pool, size=args.seed_labels, replace=False)
    curves = {}
    for method in args.methods:
        rng = np.random.default_rng(args.seed + 1)
        lab = first.copy()
        sizes, aurocs, auprcs = [], [], []
        for r in range(args.rounds + 1):
            bs = min(args.batch_size, len(lab))
            model = train_model(cfg, ds, torch.from_numpy(lab), 21, args.epochs, bs, args.lr, args.seed + r)
            model._plan.obprop_mode = 2
            auroc, auprc = _evaluate(model, ds, test, labels)
            sizes.append(len(lab))
            aurocs.append(auroc)
            auprcs.append(auprc)
            print(json.dumps(dict(method=method, round=r, labelled=len(lab), auroc=auroc, auprc=auprc)), flush=True)
            if r == args.rounds:
                break
            unl = np.setdiff1d(pool, lab)
            lab = np.concatenate([lab, _acquire(method, model, ds, unl, args.k, args, rng)])
        curves[method] = (sizes, aurocs, auprcs)
    np.savez(args.out, methods=np.array(list(curves)), **{"%s_%s" % (m, f): np.array(v[i]) for m, v in curves.items()
                                                           for i, f in enumerate(("labelled", "auroc", "auprc"))})
    print(json.dumps(dict(summary={m: dict(labelled=v[0], auroc=v[1], auprc=v[2]) for m, v in curves.items()},
                          card=card())), flush=True)


if __name__ == "__main__":
    main()
