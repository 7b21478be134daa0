#!/usr/bin/env python
"""Certified L2 robustness of a trained Raindrop_v2 by randomized smoothing (raindrop_b200.smoothing.certify, Cohen,
Rosenfeld & Kolter 2019):

    python tools/certify.py --checkpoint model.pt --data P19data/processed_data/PTdict_list.npy \\
        --outcomes P19data/processed_data/arr_outcomes.npy --split P19data/splits/phy19_split1_new.npy --part test \\
        --sigma 0.25 --out certify.tsv
    python tools/certify.py --synthetic P19 --n-samples 256 --sigma 0.25 --n 10000
    python tools/certify.py --synthetic P19 --n-samples 256 --ablate 5 --n 10000        # randomized ablation
    python tools/certify.py --synthetic P19 --n-samples 256 --ablate 3 --exhaustive     # all C(P, 3) subsets

The data arguments are those of tools/adv_robustness.py; without --checkpoint the model has the synthetic weights of
raindrop_b200.synth (a smoke run, not a trained model).  sigma and the radii are in normalised units (per-feature
standard deviations); the noise and the certificate cover the observed values (the statics too with --perturb-static),
the threat model of pgd(norm="l2").  Writes one row per sample (index, label, prediction, radius, correct, time; -1 =
abstain) to --out as Cohen's certify.py does, prints the certified accuracy at each --radii and the abstain rate, then
one JSON line.

--ablate K certifies by randomized ablation instead (raindrop_b200.ablation.certify, Levine & Feizi 2020): each
replicate keeps K sensors (players: every sensor, plus the statics with --ablate-static) and zeroes the values and masks
of the others (--keep-mask: the values only).  The radius is a number of sensors whose data may change arbitrarily;
the rows and the printed certified accuracy are per rho = 0, 1, 2, ... up to P - K.  --exhaustive enumerates all
C(P, K) subsets once and certifies deterministically (no alpha, --n0 and --n unused).
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

from adv_robustness import load_split  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--checkpoint", help="state dict of a trained Raindrop_v2 (torch.save); default: synthetic weights")
    ap.add_argument("--nhead", type=int, default=2)
    ap.add_argument("--dropout", type=float, default=0.2)
    ap.add_argument("--seed", type=int, default=0, help="torch.manual_seed before building the model (R_u); noise seed")
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--data", help="PTdict_list.npy (P12 / P19 / eICU: list of dicts; PAM: plain array)")
    src.add_argument("--synthetic", help="synthetic batches of a raindrop_b200.synth configuration (P12, P19, PAM, ...)")
    ap.add_argument("--outcomes", help="arr_outcomes.npy: labels in column --label-col")
    ap.add_argument("--label-col", type=int, default=-1)
    ap.add_argument("--split", help="split file (idx_train, idx_val, idx_test); without it every sample is used")
    ap.add_argument("--part", default="test", choices=["train", "val", "test"])
    ap.add_argument("--n-samples", type=int, default=512, help="--synthetic: number of samples")
    ap.add_argument("--batch-size", type=int, default=128)
    ap.add_argument("--sigma", type=float, default=0.25)
    ap.add_argument("--n0", type=int, default=100, help="selection draws per sample")
    ap.add_argument("--n", type=int, default=100_000, help="estimation draws per sample")
    ap.add_argument("--alpha", type=float, default=0.001)
    ap.add_argument("--radii", type=float, nargs="+", default=[0.0, 0.25, 0.5, 0.75, 1.0])
    ap.add_argument("--perturb-static", action="store_true")
    ap.add_argument("--ablate", type=int, metavar="K", help="randomized ablation keeping K players (instead of --sigma)")
    ap.add_argument("--exhaustive", action="store_true", help="--ablate: every C(P, K) subset once (deterministic)")
    ap.add_argument("--ablate-static", action="store_true", help="--ablate: the static vector is a player too")
    ap.add_argument("--keep-mask", action="store_true", help="--ablate: zero an ablated sensor's values, keep its mask")
    ap.add_argument("--out", help="per-sample rows (tab-separated); default: not written")
    args = ap.parse_args()

    from raindrop_b200 import ablation
    from raindrop_b200.smoothing import certify
    if args.ablate is None and (args.exhaustive or args.ablate_static or args.keep_mask):
        raise SystemExit("--exhaustive, --ablate-static and --keep-mask need --ablate")
    if not torch.cuda.is_available():
        raise SystemExit("certify runs on a CUDA device")
    device = torch.device("cuda", torch.cuda.current_device())
    if args.checkpoint:
        from ig_sensor_ranking import model_from_state_dict
        model = model_from_state_dict(torch.load(args.checkpoint, map_location="cpu"), args.nhead, args.seed, device,
                                      dropout=args.dropout).eval()
    else:
        if not args.synthetic:
            raise SystemExit("--data needs --checkpoint")
        from bench import build_model
        from raindrop_b200.synth import model_config
        model = build_model(model_config(args.synthetic, dropout=args.dropout), device).eval()
    P, Pstatic, Ptime, labels = load_split(args, model, device)
    n = P.shape[1]
    rows = []
    pred, radius = np.empty(n, np.int64), np.empty(n)
    t_all = time.perf_counter()
    for s in range(0, n, args.batch_size):
        e = min(n, s + args.batch_size)
        times = Ptime[:, s:e]
        lengths = torch.sum(times > 0, dim=0)
        static = None if Pstatic is None else Pstatic[s:e]
        t0 = time.perf_counter()
        # each batch draws from its own replicate range, so no two samples of the run share noise
        if args.ablate is not None:
            r = ablation.certify(model, P[:, s:e], static, times, lengths, keep=args.ablate, n0=args.n0,
                                 n_samples=args.n, alpha=args.alpha, exhaustive=args.exhaustive, seed=args.seed,
                                 step=s * (args.n0 + args.n), ablate_static=args.ablate_static,
                                 ablate_mask=not args.keep_mask)
            n_players = r.n_players
        else:
            r = certify(model, P[:, s:e], static, times, lengths, sigma=args.sigma, n0=args.n0, n_samples=args.n,
                        alpha=args.alpha, seed=args.seed, step=s * (args.n0 + args.n), perturb_static=args.perturb_static)
        dt = (time.perf_counter() - t0) / (e - s)
        pred[s:e], radius[s:e] = r.prediction, r.radius
        y = labels[s:e].cpu().numpy()
        for i in range(e - s):
            rows.append((s + i, int(y[i]), int(r.prediction[i]), float(r.radius[i]), int(r.prediction[i] == y[i]), dt))
    elapsed = time.perf_counter() - t_all
    if args.out:
        with open(args.out, "w") as f:
            f.write("idx\tlabel\tpredict\tradius\tcorrect\ttime\n")
            for row in rows:
                f.write("%d\t%d\t%d\t%.6g\t%d\t%.6g\n" % row)
    y = labels.cpu().numpy()
    correct = pred == y
    radii = args.radii if args.ablate is None else list(range(n_players - args.ablate + 1))
    acc = {"%g" % r: float(np.mean(correct & (radius >= r))) for r in radii}
    abstain = float(np.mean(pred < 0))
    if args.ablate is None:
        print("sigma %g, n0 %d, n %d, alpha %g: %d samples in %.2f s (%.1f samples/s)"
              % (args.sigma, args.n0, args.n, args.alpha, n, elapsed, n / elapsed))
        head = dict(sigma=args.sigma, n0=args.n0, n=args.n, alpha=args.alpha)
    else:
        mode = "exhaustive" if args.exhaustive else "n0 %d, n %d, alpha %g" % (args.n0, args.n, args.alpha)
        print("ablation keeping %d of %d players, %s: %d samples in %.2f s (%.1f samples/s)"
              % (args.ablate, n_players, mode, n, elapsed, n / elapsed))
        head = dict(keep=args.ablate, players=n_players, exhaustive=args.exhaustive, ablate_static=args.ablate_static,
                    ablate_mask=not args.keep_mask)
        if not args.exhaustive:
            head.update(n0=args.n0, n=args.n, alpha=args.alpha)
    for r in radii:
        print("certified accuracy at radius %-6g %.4f" % (r, acc["%g" % r]))
    print("abstain rate %.4f" % abstain)
    print(json.dumps(dict(head, samples=n, seconds=elapsed, certified_accuracy=acc, abstain=abstain)))


if __name__ == "__main__":
    main()
