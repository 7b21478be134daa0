#!/usr/bin/env python
"""Writes MC_uncertainty_<name>.npz, the Monte Carlo dropout uncertainty of every sample of a data split, from a trained
Raindrop_v2 (raindrop_b200.uncertainty.mc_dropout), and prints how accuracy changes when the least certain samples are
set aside:

    python tools/mc_uncertainty.py --checkpoint model.pt --data P19data/processed_data/PTdict_list.npy \\
        --outcomes P19data/processed_data/arr_outcomes.npy --split P19data/splits/phy19_split1_new.npy --part test \\
        --name P19
    python tools/mc_uncertainty.py --checkpoint model.pt --synthetic P19 --n-samples 512

The checkpoint, data, split and normalisation are read as tools/ig_sensor_ranking.py reads them.  The dropout
probability is not in a state dict: --dropout (default 0.2) must be the one the model was trained with.  Per batch, one
mc_dropout call with --mc-samples replicates (seed --seed, steps 0 ..) and one deterministic eval forward.

The file holds float32 arrays over the samples: mean_probs [n, C], variance [n, C], predictive_entropy,
expected_entropy, mutual_information and eval_probs [n, C] (softmax of the eval forward), plus labels [n] (int64; -1
without --outcomes).  With labels it prints the accuracy of argmax mean_probs and of the eval forward, and the accuracy of
argmax mean_probs over the 100 / 90 / 80 / 70 % of samples with the lowest mutual information.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from ig_sensor_ranking import model_from_state_dict  # noqa: E402

COVERAGES = (1.0, 0.9, 0.8, 0.7)


def coverage_accuracy(pred, labels, score, coverages=COVERAGES):
    """{coverage: accuracy of pred over the ceil(coverage * n) samples of lowest score} (stable order on ties)."""
    order = np.argsort(score, kind="stable")
    out = {}
    for c in coverages:
        k = max(1, int(np.ceil(c * len(order))))
        keep = order[:k]
        out[c] = float(np.mean(pred[keep] == labels[keep]))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--checkpoint", required=True, help="state dict of a trained Raindrop_v2 (torch.save)")
    ap.add_argument("--nhead", type=int, default=2)
    ap.add_argument("--dropout", type=float, default=0.2, help="the dropout probability the model was trained with")
    ap.add_argument("--seed", type=int, default=0, help="torch.manual_seed before building the model (R_u); MC seed")
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--data", help="PTdict_list.npy (P12 / P19 / eICU: list of dicts; PAM: plain array)")
    src.add_argument("--synthetic", help="synthetic batches of a raindrop_b200.synth configuration (P12, P19, PAM, ...)")
    ap.add_argument("--outcomes", help="arr_outcomes.npy: labels in column --label-col")
    ap.add_argument("--label-col", type=int, default=-1)
    ap.add_argument("--split", help="split file (idx_train, idx_val, idx_test); without it every sample is used")
    ap.add_argument("--part", default="test", choices=["train", "val", "test"])
    ap.add_argument("--n-samples", type=int, default=512, help="--synthetic: number of samples")
    ap.add_argument("--mc-samples", type=int, default=30, help="Monte Carlo replicates per sample")
    ap.add_argument("--batch-size", type=int, default=128)
    ap.add_argument("--name", help="file name suffix (default: the synthetic configuration or 'dataset')")
    ap.add_argument("--out-dir", default=".")
    args = ap.parse_args()

    from raindrop_b200 import data as RD
    from raindrop_b200.synth import make_batch, model_config
    from raindrop_b200.uncertainty import mc_dropout
    if not torch.cuda.is_available():
        raise SystemExit("mc_dropout runs on a CUDA device")
    device = torch.device("cuda", torch.cuda.current_device())
    model = model_from_state_dict(torch.load(args.checkpoint, map_location="cpu"), args.nhead, args.seed, device,
                                  dropout=args.dropout)
    N, T = model.d_inp, model.max_len
    labels = None
    if args.synthetic:
        cfg = model_config(args.synthetic)
        if cfg["d_inp"] != N or cfg["max_len"] != T or cfg["static"] != model.static:
            raise SystemExit("--synthetic %s does not match the checkpoint (d_inp %d, max_len %d)" % (args.synthetic, N, T))
        b = make_batch(cfg, args.n_samples, seed=args.seed, device=device)
        P, Pstatic, Ptime = b["src"], b["static"], b["times"]
        labels = b["y"].cpu().numpy()
        name = args.name or args.synthetic
    else:
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
        if args.outcomes:
            labels = np.asarray(np.load(args.outcomes, allow_pickle=True)).reshape(n, -1)[idx, args.label_col]
            labels = labels.astype(np.int64)
        mf, stdf = RD.feature_stats(torch.as_tensor(P_raw[idx_train]).to(device))
        st = None if (static is None or not model.static) else static[idx]
        y0 = labels if labels is not None else np.zeros(len(idx), dtype=np.int64)
        P, Pstatic, Ptime, _ = RD.tensorize_normalize(P_raw[idx], minutes[idx], st, y0, mf, stdf, device=device)
        name = args.name or "dataset"

    keys = ("mean_probs", "variance", "predictive_entropy", "expected_entropy", "mutual_information")
    parts = {k: [] for k in keys + ("eval_probs",)}
    n = P.shape[1]
    for s in range(0, n, args.batch_size):
        e = min(n, s + args.batch_size)
        src, times = P[:, s:e], Ptime[:, s:e]
        lengths = torch.sum(times > 0, dim=0)
        static = None if Pstatic is None else Pstatic[s:e]
        res = mc_dropout(model, src, static, times, lengths, n_samples=args.mc_samples, seed=args.seed, step=0)
        with torch.no_grad():
            logits = model(src, static, times, lengths)[0]
        for k in keys:
            parts[k].append(getattr(res, k).cpu().numpy())
        parts["eval_probs"].append(torch.softmax(logits.double(), dim=1).float().cpu().numpy())
    out = {k: np.concatenate(v) for k, v in parts.items()}
    out["labels"] = labels if labels is not None else np.full(n, -1, dtype=np.int64)
    path = os.path.join(args.out_dir, "MC_uncertainty_%s.npz" % name)
    np.savez(path, **out)
    print("wrote %s: %d samples, %d replicates each, mean mutual information %.4g"
          % (path, n, args.mc_samples, float(out["mutual_information"].mean())))
    if labels is None:
        return
    pred = out["mean_probs"].argmax(axis=1)
    print("accuracy: MC mean %.4f, deterministic eval forward %.4f"
          % (float(np.mean(pred == labels)), float(np.mean(out["eval_probs"].argmax(axis=1) == labels))))
    for c, acc in coverage_accuracy(pred, labels, out["mutual_information"]).items():
        print("  coverage %3d %% (lowest mutual information): accuracy %.4f" % (round(100 * c), acc))


if __name__ == "__main__":
    main()
