#!/usr/bin/env python
"""Trains a Raindrop_v2 checkpoint with differential privacy (DP-SGD, raindrop_b200.privacy.DPTrainStep) and prints the
privacy spent, epsilon at --delta, after every epoch:

    python tools/dp_train.py --data P19data/processed_data/PTdict_list.npy \\
        --outcomes P19data/processed_data/arr_outcomes.npy --split P19data/splits/phy19_split1_new.npy \\
        --q 0.01 --max-grad-norm 1.0 --noise-multiplier 1.1 --epochs 10 --out dp_model.pt
    python tools/dp_train.py --synthetic P19 --n-samples 4096 --target-epsilon 8 --epochs 5 --out dp_model.pt

The training part of the split is resident on the device (DeviceDataset); each step draws a Poisson batch of rate --q
(PoissonSampler, fixed capacity, weight 0 in the empty slots), so the RDP accountant of the subsampled Gaussian
mechanism applies; an epoch is round(1 / q) steps.  --target-epsilon picks the noise multiplier that spends exactly that
budget over all epochs (noise_multiplier_for).  The normalisation statistics are computed from the training part and are
not private.  The model has the shape of raindrop_b200.synth.model_config (d_model = 4 d_inp, nhid = 2 d_model, two
layers, two heads); the noise seed comes from os.urandom, and (seed, step) of the noise stream is saved with the
checkpoint so that a resumed run never replays it.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from raindrop_b200 import data as RD  # noqa: E402
from raindrop_b200.privacy import DPTrainStep, PoissonSampler, epsilon, noise_multiplier_for  # noqa: E402
from raindrop_b200.synth import make_batch, model_config  # noqa: E402


def build_model(d_inp, max_len, d_static, n_classes, dropout, seed, device):
    from raindrop_b200.models_rd import Raindrop_v2
    torch.manual_seed(seed)
    d_model = 4 * d_inp
    kw = {} if d_static > 0 else {"static": False}
    m = Raindrop_v2(d_inp, d_model, 2, 2 * d_model, 2, dropout, max_len, d_static, 100, 0.5, "mean", n_classes,
                    torch.ones(d_inp, d_inp), **kw)
    return m.to(device)


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
    ap.add_argument("--q", type=float, default=0.01, help="Poisson sampling rate")
    ap.add_argument("--max-grad-norm", type=float, default=1.0)
    noise = ap.add_mutually_exclusive_group()
    noise.add_argument("--noise-multiplier", type=float, default=None)
    noise.add_argument("--target-epsilon", type=float, default=None)
    ap.add_argument("--delta", type=float, default=1e-5)
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--lr", type=float, default=1e-3)
    ap.add_argument("--dropout", type=float, default=0.2)
    ap.add_argument("--seed", type=int, default=0, help="model initialisation and sampler seed")
    ap.add_argument("--out", default=None, help="checkpoint file (state dict + DP metadata, torch.save)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("DP training runs on a CUDA device")
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
    model = build_model(width // 2, T, d_static, n_classes, args.dropout, args.seed, device).train()
    ds = RD.DeviceDataset(P, Pstatic, Ptime, y, device=device)

    sampler = PoissonSampler(n, args.q, seed=args.seed)
    steps_per_epoch = max(1, int(round(1.0 / args.q)))
    total = steps_per_epoch * args.epochs
    if args.target_epsilon is not None:
        sigma = noise_multiplier_for(args.target_epsilon, args.delta, args.q, total)
    else:
        sigma = 1.0 if args.noise_multiplier is None else args.noise_multiplier
    L_ = args.q * n
    step = DPTrainStep(model, sampler.capacity, args.max_grad_norm, sigma, L_, lr=args.lr)
    print("n_train %d, q %g, capacity %d, expected batch %.1f, sigma %.4f, C %g, %d steps per epoch"
          % (n, args.q, sampler.capacity, L_, sigma, args.max_grad_norm, steps_per_epoch))
    done = 0
    for ep in range(args.epochs):
        loss_sum = torch.zeros((), dtype=torch.float64, device=device)
        clipped = torch.zeros((), dtype=torch.float64, device=device)
        for _ in range(steps_per_epoch):
            idx, weight = sampler.sample()
            ds.fill(step, torch.from_numpy(idx))
            step.weight.copy_(torch.from_numpy(weight))
            loss_sum += step.step()[0]
            clipped += step.clipped_fraction()
            done += 1
        print("epoch %d: mean loss %.4f, clipped %.1f %%, epsilon %.4f at delta %g"
              % (ep + 1, loss_sum.item() / steps_per_epoch, 100.0 * clipped.item() / steps_per_epoch,
                 epsilon(args.q, sigma, done, args.delta), args.delta), flush=True)
    if args.out:
        seed, nstep = step.noise_key_state()
        torch.save(dict(state_dict=model.state_dict(), q=args.q, noise_multiplier=sigma, max_grad_norm=args.max_grad_norm,
                        steps=done, delta=args.delta, epsilon=epsilon(args.q, sigma, done, args.delta),
                        noise_key=(seed, nstep)), args.out)
        print("wrote", args.out)


if __name__ == "__main__":
    main()
