#!/usr/bin/env python
"""Clean and robust accuracy of a trained Raindrop_v2 under FGSM and PGD-K attacks (raindrop_b200.adversarial.pgd) over
a list of budgets eps:

    python tools/adv_robustness.py --checkpoint model.pt --data P19data/processed_data/PTdict_list.npy \\
        --outcomes P19data/processed_data/arr_outcomes.npy --split P19data/splits/phy19_split1_new.npy --part test \\
        --eps 0.05 0.1 0.2
    python tools/adv_robustness.py --checkpoint model.pt --synthetic P19 --n-samples 512 --norm l2 --eps 0.5 1 2

The data arguments are those of tools/mc_uncertainty.py.  eps is in normalised units (per-feature standard deviations);
only observed values are perturbed (the mask, times and lengths never change), and the statics too with
--perturb-static.  FGSM is one step of size eps from x; PGD-K takes --pgd-steps steps of 2.5 eps / K from a random start.
Prints one line per eps and one JSON line with every accuracy.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from ig_sensor_ranking import model_from_state_dict  # noqa: E402


def load_split(args, model, device):
    """(P, Pstatic, Ptime, labels) on the device, as tools/mc_uncertainty.py reads them."""
    from raindrop_b200 import data as RD
    from raindrop_b200.synth import make_batch, model_config
    N, T = model.d_inp, model.max_len
    if args.synthetic:
        cfg = model_config(args.synthetic)
        if cfg["d_inp"] != N or cfg["max_len"] != T or cfg["static"] != model.static:
            raise SystemExit("--synthetic %s does not match the checkpoint (d_inp %d, max_len %d)" % (args.synthetic, N, T))
        b = make_batch(cfg, args.n_samples, seed=args.seed, device=device)
        return b["src"], b["static"], b["times"], b["y"]
    if not args.outcomes:
        raise SystemExit("robust accuracy needs labels: give --outcomes")
    raw = np.load(args.data, allow_pickle=True)
    is_list = raw.dtype == object and isinstance(raw.flat[0], dict)
    P_raw, minutes, static = RD.load_ptdict_list(args.data) if is_list else RD.load_array_dataset(args.data)
    if P_raw.shape[1] != T or P_raw.shape[2] != N:
        raise SystemExit("data [n, T=%d, F=%d] does not match the checkpoint (max_len %d, d_inp %d)"
                         % (P_raw.shape[1], P_raw.shape[2], T, N))
    n = len(P_raw)
    idx_train, idx = np.arange(n), np.arange(n)
    if args.split:
        parts = RD.load_split(args.split)
        idx_train, idx = parts[0], parts[("train", "val", "test").index(args.part)]
    labels = np.asarray(np.load(args.outcomes, allow_pickle=True)).reshape(n, -1)[idx, args.label_col].astype(np.int64)
    mf, stdf = RD.feature_stats(torch.as_tensor(P_raw[idx_train]).to(device))
    st = None if (static is None or not model.static) else static[idx]
    P, Pstatic, Ptime, _ = RD.tensorize_normalize(P_raw[idx], minutes[idx], st, labels, mf, stdf, device=device)
    return P, Pstatic, Ptime, torch.as_tensor(labels, device=device)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--checkpoint", required=True, help="state dict of a trained Raindrop_v2 (torch.save)")
    ap.add_argument("--nhead", type=int, default=2)
    ap.add_argument("--dropout", type=float, default=0.2)
    ap.add_argument("--seed", type=int, default=0, help="torch.manual_seed before building the model (R_u); attack seed")
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--data", help="PTdict_list.npy (P12 / P19 / eICU: list of dicts; PAM: plain array)")
    src.add_argument("--synthetic", help="synthetic batches of a raindrop_b200.synth configuration (P12, P19, PAM, ...)")
    ap.add_argument("--outcomes", help="arr_outcomes.npy: labels in column --label-col")
    ap.add_argument("--label-col", type=int, default=-1)
    ap.add_argument("--split", help="split file (idx_train, idx_val, idx_test); without it every sample is used")
    ap.add_argument("--part", default="test", choices=["train", "val", "test"])
    ap.add_argument("--n-samples", type=int, default=512, help="--synthetic: number of samples")
    ap.add_argument("--batch-size", type=int, default=512)
    ap.add_argument("--eps", type=float, nargs="+", default=[0.05, 0.1, 0.2])
    ap.add_argument("--norm", default="linf", choices=["linf", "l2"])
    ap.add_argument("--pgd-steps", type=int, default=10)
    ap.add_argument("--perturb-static", action="store_true")
    args = ap.parse_args()

    from raindrop_b200.adversarial import pgd
    if not torch.cuda.is_available():
        raise SystemExit("pgd runs on a CUDA device")
    device = torch.device("cuda", torch.cuda.current_device())
    model = model_from_state_dict(torch.load(args.checkpoint, map_location="cpu"), args.nhead, args.seed, device,
                                  dropout=args.dropout).eval()
    P, Pstatic, Ptime, labels = load_split(args, model, device)
    n = P.shape[1]
    attacks = {"fgsm": dict(n_steps=1, random_start=False), "pgd%d" % args.pgd_steps: dict(n_steps=args.pgd_steps)}
    correct = {"clean": 0}
    for eps in args.eps:
        for a in attacks:
            correct["%s@%g" % (a, eps)] = 0
    for s in range(0, n, args.batch_size):
        e = min(n, s + args.batch_size)
        src, times, y = P[:, s:e], Ptime[:, s:e], labels[s:e]
        lengths = torch.sum(times > 0, dim=0)
        static = None if Pstatic is None else Pstatic[s:e]
        for eps in args.eps:
            for a, kw in attacks.items():
                step_size = eps if a == "fgsm" else None
                r = pgd(model, src, static, times, lengths, y, eps=eps, norm=args.norm, step_size=step_size,
                        seed=args.seed, step=s, perturb_static=args.perturb_static, **kw)
                correct["%s@%g" % (a, eps)] += int((~r.success).sum())
        correct["clean"] += int((r.clean_logits.argmax(1) == y).sum())
    acc = {k: v / n for k, v in correct.items()}
    print("clean accuracy %.4f over %d samples (%s)" % (acc["clean"], n, args.norm))
    for eps in args.eps:
        print("eps %-8g " % eps + "  ".join("%s %.4f" % (a, acc["%s@%g" % (a, eps)]) for a in attacks))
    print(json.dumps(dict(acc, norm=args.norm, n=n)))


if __name__ == "__main__":
    main()
