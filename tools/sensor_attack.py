#!/usr/bin/env python
"""Worst-case sensor removal of a trained Raindrop_v2 (raindrop_b200.sensor_attack): the fewest missing sensors that
flip each prediction, and the robust accuracy under r adversarially missing sensors.

    python tools/sensor_attack.py --checkpoint model.pt --data P19data/processed_data/PTdict_list.npy \\
        --outcomes P19data/processed_data/arr_outcomes.npy --split P19data/splits/phy19_split1_new.npy --part test \\
        --max-removed 3 --beam 4 --out attack.tsv
    python tools/sensor_attack.py --synthetic P19 --n-samples 256 --max-removed 3              # greedy
    python tools/sensor_attack.py --synthetic P19 --n-samples 256 --max-removed 2 --exhaustive

The data arguments are those of tools/certify.py; without --checkpoint the model has the synthetic weights of
raindrop_b200.synth (a smoke run, not a trained model).  The reference class is the label (untargeted).  Players are
every sensor, plus the statics with --remove-static; a removed sensor has its values and mask zeroed (--keep-mask: the
values only).  Prints the robust accuracy for r = 0 .. max_removed (an upper bound for greedy and beam search, exact
with --exhaustive) and the sensors that appear most often in the found sets, then one JSON line.  --out writes one row
per sample: index, label, clean prediction, n_removed (-1: no flip within the budget), the removed sensors (names
from --names or indices; "static" for the static player) and the final score.
"""
import argparse
import json
import os
import sys
import time
from types import SimpleNamespace

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
    ap.add_argument("--seed", type=int, default=0, help="torch.manual_seed before building the model (R_u)")
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--data", help="PTdict_list.npy (P12 / P19 / eICU: list of dicts; PAM: plain array)")
    src.add_argument("--synthetic", help="synthetic batches of a raindrop_b200.synth configuration (P12, P19, PAM, ...)")
    ap.add_argument("--outcomes", help="arr_outcomes.npy: labels in column --label-col")
    ap.add_argument("--label-col", type=int, default=-1)
    ap.add_argument("--split", help="split file (idx_train, idx_val, idx_test); without it every sample is used")
    ap.add_argument("--part", default="test", choices=["train", "val", "test"])
    ap.add_argument("--n-samples", type=int, default=512, help="--synthetic: number of samples")
    ap.add_argument("--batch-size", type=int, default=128)
    ap.add_argument("--max-removed", type=int, default=3)
    ap.add_argument("--beam", type=int, default=1, metavar="W", help="beam width (1: greedy)")
    ap.add_argument("--exhaustive", action="store_true", help="every set of at most --max-removed players")
    ap.add_argument("--remove-static", action="store_true", help="the static vector is a player too")
    ap.add_argument("--keep-mask", action="store_true", help="zero a removed sensor's values, keep its mask")
    ap.add_argument("--names", help="a text file with one sensor name per line (default: indices)")
    ap.add_argument("--top", type=int, default=10, help="print the sensors most often removed")
    ap.add_argument("--out", help="per-sample rows (tab-separated); default: not written")
    args = ap.parse_args()

    from raindrop_b200.sensor_attack import robust_accuracy, sensor_removal_attack
    if not torch.cuda.is_available():
        raise SystemExit("sensor_attack runs on a CUDA device")
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
    names = None
    if args.names:
        with open(args.names) as f:
            names = [line.strip() for line in f if line.strip()]
    n = P.shape[1]
    nr, clean_pred, scores, sets = [], [], [], []
    t_all = time.perf_counter()
    for s in range(0, n, args.batch_size):
        e = min(n, s + args.batch_size)
        times = Ptime[:, s:e]
        lengths = torch.sum(times > 0, dim=0)
        static = None if Pstatic is None else Pstatic[s:e]
        r = sensor_removal_attack(model, P[:, s:e], static, times, lengths, labels[s:e], max_removed=args.max_removed,
                                  beam_width=args.beam, exhaustive=args.exhaustive, remove_static=args.remove_static,
                                  remove_mask=not args.keep_mask)
        players = r.players.tolist()
        nr.append(r.n_removed.cpu())
        clean_pred.append(r.clean_logits.argmax(1).cpu())
        scores.append(r.score.cpu())
        sets.append(r.removed.cpu())
    torch.cuda.synchronize()
    elapsed = time.perf_counter() - t_all
    nr, clean_pred = torch.cat(nr).numpy(), torch.cat(clean_pred).numpy()
    scores, sets = torch.cat(scores).numpy(), torch.cat(sets).numpy()
    y = labels.cpu().numpy()
    acc = robust_accuracy(SimpleNamespace(n_removed=nr, max_removed=args.max_removed))

    def name(p):
        sensor = players[p]
        return "static" if sensor < 0 else (names[sensor] if names else str(sensor))
    flipped = nr > 0
    counts = sets[flipped].sum(0) if flipped.any() else np.zeros(len(players), np.int64)
    order = [p for p in np.argsort(-counts, kind="stable") if counts[p] > 0][:args.top]
    if args.out:
        with open(args.out, "w") as f:
            f.write("idx\tlabel\tclean_pred\tn_removed\tremoved\tscore\n")
            for i in range(n):
                rem = ",".join(name(p) for p in np.flatnonzero(sets[i]))
                f.write("%d\t%d\t%d\t%d\t%s\t%.6g\n" % (i, y[i], clean_pred[i], nr[i], rem, scores[i]))
    mode = "exhaustive" if args.exhaustive else ("greedy" if args.beam == 1 else "beam %d" % args.beam)
    print("%s search over %d players, up to %d removed: %d samples in %.2f s (%.1f samples/s)"
          % (mode, len(players), args.max_removed, n, elapsed, n / elapsed))
    for r, a in enumerate(acc):
        print("robust accuracy with %d removed  %.4f" % (r, a))
    print("most often removed in the sets that flip a correct prediction:")
    for p in order:
        print("  %-12s %d" % (name(p), counts[p]))
    print(json.dumps(dict(mode=mode, players=len(players), max_removed=args.max_removed, samples=n, seconds=elapsed,
                          robust_accuracy=acc.tolist(), most_removed={name(p): int(counts[p]) for p in order})))


if __name__ == "__main__":
    main()
