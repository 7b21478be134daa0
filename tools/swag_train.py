#!/usr/bin/env python
"""Trains a Raindrop_v2 checkpoint, then runs an SWA phase that collects an SWAG posterior (raindrop_b200.swag), and
writes the checkpoint, the SWA weights and the posterior:

    python tools/swag_train.py --data P19data/processed_data/PTdict_list.npy \\
        --outcomes P19data/processed_data/arr_outcomes.npy --split P19data/splits/phy19_split1_new.npy \\
        --epochs 20 --swa-epochs 10 --swa-lr 5e-4 --collect-every 0 --rank 20 --out p19
    python tools/swag_train.py --synthetic P19 --n-samples 4096 --epochs 3 --swa-epochs 5 --out p19

The training part of the split is resident on the device (DeviceDataset); every epoch is a fresh permutation in batches
of --batch-size (the last partial batch is dropped) through one CUDA-graph TrainStep at --lr.  The SWA phase continues
at the constant learning rate --swa-lr (TrainStep.set_lr) and collects one snapshot every --collect-every steps, or once
per epoch with 0 (Maddox et al.'s schedule).  Files: <out>.pt (state dict at the end of training), <out>_swa.pt (the
state dict with the SWA weights) and <out>_swag.pt (SWAG.save; tools/laplace_uncertainty.py --swag reads it).  The model
has the shape of tools/dp_train.py (d_model = 4 d_inp, nhid = 2 d_model, two layers, two heads).
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from dp_train import build_model  # noqa: E402
from raindrop_b200 import data as RD  # noqa: E402
from raindrop_b200.swag import SWAG  # noqa: E402
from raindrop_b200.synth import make_batch, model_config  # noqa: E402
from raindrop_b200.train import TrainStep  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--data", help="PTdict_list.npy (P12 / P19 / eICU: list of dicts; PAM: plain array)")
    src.add_argument("--synthetic", help="synthetic samples of a raindrop_b200.synth configuration (P12, P19, PAM, ...)")
    ap.add_argument("--outcomes", help="arr_outcomes.npy (--data): labels in column --label-col")
    ap.add_argument("--label-col", type=int, default=-1)
    ap.add_argument("--split", help="split file (idx_train, idx_val, idx_test); without it every sample trains")
    ap.add_argument("--n-samples", type=int, default=4096, help="--synthetic: training samples")
    ap.add_argument("--n-classes", type=int, default=2, help="--data: number of classes")
    ap.add_argument("--batch-size", type=int, default=128)
    ap.add_argument("--epochs", type=int, default=10, help="training epochs before the SWA phase")
    ap.add_argument("--lr", type=float, default=1e-3)
    ap.add_argument("--swa-epochs", type=int, default=10)
    ap.add_argument("--swa-lr", type=float, default=5e-4, help="constant learning rate of the SWA phase")
    ap.add_argument("--collect-every", type=int, default=0, help="steps between snapshots (0: one per epoch)")
    ap.add_argument("--rank", type=int, default=20, help="deviation columns of the posterior")
    ap.add_argument("--dropout", type=float, default=0.2)
    ap.add_argument("--seed", type=int, default=0, help="model initialisation and permutation seed")
    ap.add_argument("--out", default="swag_model", help="prefix of the three output files")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("swag_train runs on a CUDA device")
    device = torch.device("cuda", torch.cuda.current_device())

    if args.synthetic:
        cfg = model_config(args.synthetic)
        b = make_batch(cfg, args.n_samples, seed=args.seed, device=device)
        P, Pstatic, Ptime, y = b["src"], b["static"], b["times"], b["y"]
        d_static, n_classes = (cfg["d_static"] if cfg["static"] else 0), cfg["n_classes"]
    else:
        if not args.outcomes:
            raise SystemExit("--data needs --outcomes (the labels)")
        raw = np.load(args.data, allow_pickle=True)
        is_list = raw.dtype == object and isinstance(raw.flat[0], dict)
        P_raw, minutes, static = RD.load_ptdict_list(args.data) if is_list else RD.load_array_dataset(args.data)
        n = len(P_raw)
        idx = RD.load_split(args.split)[0] if args.split else np.arange(n)
        labels = np.asarray(np.load(args.outcomes, allow_pickle=True)).reshape(n, -1)[idx, args.label_col].astype(np.int64)
        mf, stdf = RD.feature_stats(torch.as_tensor(P_raw[idx]).to(device))
        st = None if static is None else static[idx]
        P, Pstatic, Ptime, y = RD.tensorize_normalize(P_raw[idx], minutes[idx], st, labels, mf, stdf, device=device)
        d_static, n_classes = (0 if Pstatic is None else Pstatic.shape[1]), args.n_classes
    T, n, width = P.shape
    if n < args.batch_size:
        raise SystemExit("%d training samples, fewer than --batch-size %d" % (n, args.batch_size))
    model = build_model(width // 2, T, d_static, n_classes, args.dropout, args.seed, device).train()
    ds = RD.DeviceDataset(P, Pstatic, Ptime, y, device=device)
    step = TrainStep(model, args.batch_size, lr=args.lr)
    rng = np.random.default_rng(args.seed)
    steps_per_epoch = n // args.batch_size

    def epoch(post=None):
        perm = torch.from_numpy(rng.permutation(n))
        loss = torch.zeros((), dtype=torch.float64, device=device)
        for i in range(steps_per_epoch):
            ds.fill(step, perm[i * args.batch_size:(i + 1) * args.batch_size])
            loss += step.step()[0]
            if post is not None and args.collect_every > 0 and (i + 1) % args.collect_every == 0:
                post.collect(step)
        if post is not None and args.collect_every == 0:
            post.collect(step)
        return loss.item() / steps_per_epoch

    for ep in range(args.epochs):
        print("epoch %d: mean loss %.4f" % (ep + 1, epoch()), flush=True)
    torch.save(model.state_dict(), args.out + ".pt")
    post = SWAG(model, rank=args.rank)
    step.set_lr(args.swa_lr)
    for ep in range(args.swa_epochs):
        loss = epoch(post)
        print("SWA epoch %d (lr %g): mean loss %.4f, %d snapshots" % (ep + 1, args.swa_lr, loss, post.n_collected),
              flush=True)
    post.save(args.out + "_swag.pt")
    post.load_mean(model)
    torch.save(model.state_dict(), args.out + "_swa.pt")
    print("wrote %s.pt, %s_swa.pt, %s_swag.pt (%d snapshots, rank %d)" % (args.out, args.out, args.out, post.n_collected,
                                                                          args.rank))


if __name__ == "__main__":
    main()
