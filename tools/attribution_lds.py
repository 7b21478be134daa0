#!/usr/bin/env python
"""Linear datamodeling score (LDS; Park et al. 2023) of the training-data attribution methods of raindrop_b200.influence
on synthetic data with a planted learnable label: how well does each method's sum of scores over a training subset rank
what training on that subset actually does to a query's prediction?

    python tools/attribution_lds.py --shape P19 --n-train 1000 --n-query 100 --subsets 50

Data: raindrop_b200.synth.make_batch samples of --shape (2 classes), labelled by the sign of the observed-value mean of
sensors 0 and 1 (their sum against its median over all samples), with a share --label-noise of the labels flipped.
Then:
  - J = --subsets models are trained with TrainStep on random half subsets S_j of the training set (each from its own
    initial weights), and the true-label margin m_j(q) = z_y - log sum_{c != y} exp(z_c) of every query is recorded;
  - the methods score every query against the whole training set at models trained on all of it (--members of them for
    TRAK with M = --members): TracIn (one checkpoint, lr 1), TracIn-RP (--projection dims), EK-FAC (default damping) and
    TRAK with M = 1 and M = --members, its damping swept over --damping factors of the mean largest eigenvalue;
  - per query, the Spearman correlation over j between m_j(q) and the predicted sum_{i in S_j} tau(q, i).
Prints one JSON line: the mean +- standard error over queries of each method's correlation, the models' query accuracy
and the card's name and power limit.  An evaluation, not a test: there is no threshold.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def planted_data(cfg, n, seed, noise):
    """make_batch samples whose label is the sign of the mean observed value of sensors 0 and 1 (against its median),
    a share `noise` of them flipped."""
    from raindrop_b200.synth import make_batch
    b = make_batch(cfg, n, seed=seed)
    N = cfg["d_inp"]
    v, m = b["src"][:, :, :N], b["src"][:, :, N:]
    mean = (v[:, :, :2] * m[:, :, :2]).sum((0, 2)) / m[:, :, :2].sum((0, 2)).clamp_min(1.0)
    y = (mean > mean.median()).long()
    g = torch.Generator().manual_seed(seed + 1)
    flip = torch.rand(n, generator=g) < noise
    b["y"] = torch.where(flip, 1 - y, y)
    return b


def train_model(cfg, ds, idx, init_seed, epochs, batch, lr, seed):
    from helpers import build_dropin
    from raindrop_b200.train import TrainStep
    model = build_dropin(cfg, init_seed).train()
    step = TrainStep(model, batch, lr=lr)
    g = torch.Generator().manual_seed(seed)
    n = len(idx)
    for _ in range(epochs):
        perm = idx[torch.randperm(n, generator=g)]
        for i in range(n // batch):
            ds.fill(step, perm[i * batch:(i + 1) * batch])
            step.step()
    return model.eval()


def margins(model, q):
    with torch.no_grad():
        z, _, _ = model.forward(q["src"], q["static"], q["times"], q["lengths"])
    z = z.double()
    rest = z.clone()
    rest[torch.arange(len(q["y"])), q["y"]] = float("-inf")
    return (z.gather(1, q["y"][:, None])[:, 0] - torch.logsumexp(rest, dim=1)).cpu().numpy(), \
        (z.argmax(1) == q["y"]).double().mean().item()


def lds(actual, masks, scores):
    """Per query: Spearman correlation over subsets between actual [J, nq] and masks [J, nt] @ scores[q]."""
    from scipy.stats import spearmanr
    pred = masks @ scores.T                                       # [J, nq]
    rho = np.array([spearmanr(actual[:, q], pred[:, q]).statistic for q in range(actual.shape[1])])
    rho = rho[np.isfinite(rho)]
    return dict(mean=float(rho.mean()), se=float(rho.std(ddof=1) / np.sqrt(len(rho))), n=int(len(rho)))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--shape", default="P19")
    ap.add_argument("--n-train", type=int, default=1000)
    ap.add_argument("--n-query", type=int, default=100)
    ap.add_argument("--subsets", type=int, default=50, help="J: models trained on random half subsets")
    ap.add_argument("--members", type=int, default=5, help="M of the TRAK ensemble")
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--lr", type=float, default=1e-3)
    ap.add_argument("--dropout", type=float, default=0.2)
    ap.add_argument("--label-noise", type=float, default=0.1)
    ap.add_argument("--projection", type=int, default=4096, help="dims of TracIn-RP and TRAK")
    ap.add_argument("--damping", type=float, nargs="*", default=[0.0, 1e-4, 1e-3, 1e-2, 1e-1],
                    help="TRAK damping, as factors of the mean largest eigenvalue over the members")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()

    from raindrop_b200 import influence as IF
    from raindrop_b200.data import DeviceDataset
    from raindrop_b200.synth import model_config
    if not torch.cuda.is_available():
        raise SystemExit("attribution_lds runs on a CUDA device")
    cfg = model_config(a.shape, dropout=a.dropout)
    if cfg["n_classes"] != 2:
        raise SystemExit("the planted label has 2 classes; --shape %s has %d" % (a.shape, cfg["n_classes"]))
    t_start = time.perf_counter()
    tr = planted_data(cfg, a.n_train, a.seed, a.label_noise)
    te = planted_data(cfg, a.n_query, a.seed + 1000, 0.0)
    ds = DeviceDataset(tr["src"], tr["static"], tr["times"], tr["y"])
    q = {k: (v.cuda() if v is not None else None) for k, v in te.items()}
    train = {k: (v.cuda() if v is not None else None) for k, v in tr.items()}

    # J models on random half subsets
    rng = np.random.default_rng(a.seed)
    masks = np.zeros((a.subsets, a.n_train))
    actual = np.zeros((a.subsets, a.n_query))
    accs = []
    for j in range(a.subsets):
        idx = np.sort(rng.choice(a.n_train, a.n_train // 2, replace=False))
        masks[j, idx] = 1.0
        m = train_model(cfg, ds, torch.from_numpy(idx), 1000 + j, a.epochs, a.batch_size, a.lr, a.seed + j)
        actual[j], acc = margins(m, q)
        accs.append(acc)
        del m
    t_subsets = time.perf_counter() - t_start

    # the attributions, at models trained on the whole training set
    full_idx = torch.arange(a.n_train)
    members = [train_model(cfg, ds, full_idx, 2000 + k, a.epochs, a.batch_size, a.lr, a.seed + 500 + k)
               for k in range(a.members)]
    full_acc = [margins(m, q)[1] for m in members]
    model = members[0]
    sds = [{k: v.detach().clone() for k, v in m.state_dict().items()} for m in members]
    qn = dict(q, y=q["y"])
    res = {}
    t0 = time.perf_counter()
    res["tracin"] = lds(actual, masks, IF.tracin(model, qn, train).cpu().numpy())
    sk = dict(dim=a.projection, seed=a.seed)
    res["tracin_rp"] = lds(actual, masks, IF.tracin_sketch(IF.project(model, qn, **sk), IF.project(model, train, **sk))
                           .cpu().numpy())
    res["ekfac"] = lds(actual, masks, IF.ekfac_influence(model, qn, train, IF.ekfac_factors(model, train)).cpu().numpy())
    for M in sorted({1, a.members}):
        feats = IF.trak_features(model, train, checkpoints=sds[:M], dim=a.projection, seed=a.seed)
        scale = feats.eigenvalues.max(dim=1).values.mean().item()
        for f in a.damping:
            S = IF.trak(model, qn, feats, damping=f * scale, checkpoints=sds[:M]).cpu().numpy()
            res["trak_M%d_damping%g" % (M, f)] = lds(actual, masks, S)
        del feats
    t_methods = time.perf_counter() - t0
    print(json.dumps(dict(card=card(), shape=a.shape, n_train=a.n_train, n_query=a.n_query, subsets=a.subsets,
                          members=a.members, epochs=a.epochs, projection=a.projection, label_noise=a.label_noise,
                          subset_model_query_accuracy=float(np.mean(accs)), full_model_query_accuracy=full_acc,
                          damping_scale="factor of the mean largest eigenvalue", lds=res,
                          subset_training_s=t_subsets, methods_s=t_methods)), flush=True)


if __name__ == "__main__":
    main()
