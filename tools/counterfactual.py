#!/usr/bin/env python
"""Counterfactual explanations of a Raindrop_v2 over a data split (raindrop_b200.counterfactual.counterfactual):

    python tools/counterfactual.py --checkpoint model.pt --data P19data/processed_data/PTdict_list.npy \\
        --split P19data/splits/phy19_split1_new.npy --part test --out cf.csv
    python tools/counterfactual.py --synthetic P19 --n-samples 512 --out cf.csv       # synthetic weights and data

The weights of the distance are the inverse median absolute deviation of each sensor's observed (normalised) values in
the train part, with the deviation floored at --mad-floor so a sensor with few distinct values cannot dominate the FISTA
step; the box is each sensor's 1st / 99th percentile there.  Writes one CSV row per sample (valid, distance, L0, the
sensors changed, and per sensor the largest change in original units: delta times the feature's std) and prints the
validity rate and the sensors changed most often.
"""
import argparse
import csv
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402
import torch  # noqa: E402


def load_parts(args, device):
    """(model, train part, evaluated part, feature std [N]); a part is (src, static, times, lengths)."""
    from raindrop_b200 import data as RD
    from raindrop_b200.synth import make_batch, model_config
    if args.synthetic:
        cfg = model_config(args.synthetic, dropout=args.dropout)
        if args.checkpoint:
            from ig_sensor_ranking import model_from_state_dict
            model = model_from_state_dict(torch.load(args.checkpoint, map_location="cpu"), args.nhead, args.seed, device,
                                          args.dropout)
        else:
            from bench import build_model
            model = build_model(cfg, device)
        parts = []
        for seed, n in ((args.seed + 1, args.n_train), (args.seed, args.n_samples)):
            b = make_batch(cfg, n, seed=seed, device=device)
            parts.append((b["src"], b["static"], b["times"], b["lengths"]))
        return model, parts[0], parts[1], np.ones(cfg["d_inp"])
    if not args.checkpoint:
        raise SystemExit("--data needs --checkpoint")
    from ig_sensor_ranking import model_from_state_dict
    model = model_from_state_dict(torch.load(args.checkpoint, map_location="cpu"), args.nhead, args.seed, device,
                                          args.dropout)
    raw = np.load(args.data, allow_pickle=True)
    is_list = raw.dtype == object and isinstance(raw.flat[0], dict)
    P_raw, minutes, static = RD.load_ptdict_list(args.data) if is_list else RD.load_array_dataset(args.data)
    n = len(P_raw)
    idx_train, idx = np.arange(n), np.arange(n)
    if args.split:
        sp = RD.load_split(args.split)
        idx_train, idx = sp[0], sp[("train", "val", "test").index(args.part)]
    mf, stdf = RD.feature_stats(torch.as_tensor(P_raw[idx_train]).to(device))
    out = []
    for ix in (idx_train, idx):
        st = None if (static is None or not model.static) else static[ix]
        P, Ps, Pt, _ = RD.tensorize_normalize(P_raw[ix], minutes[ix], st, np.zeros(len(ix), np.int64), mf, stdf,
                                              device=device)
        lengths = torch.sum(Pt > 0, dim=0)
        out.append((P, Ps, Pt, lengths))
    return model, out[0], out[1], stdf.detach().cpu().numpy().reshape(-1)


def sensor_stats(src, mad_floor):
    """Per sensor from the observed values of src [T, n, 2N]: (1 / max(MAD, floor), 1st and 99th percentiles)."""
    N = src.shape[2] // 2
    v, m = src[:, :, :N].detach().cpu().numpy(), src[:, :, N:].detach().cpu().numpy() > 0
    w, lo, hi = np.ones(N, np.float32), np.full(N, -np.inf, np.float32), np.full(N, np.inf, np.float32)
    for n in range(N):
        x = v[:, :, n][m[:, :, n]]
        if x.size < 2:
            continue
        w[n] = 1.0 / max(float(np.median(np.abs(x - np.median(x)))), mad_floor)
        lo[n], hi[n] = np.percentile(x, 1), np.percentile(x, 99)
    return w, lo, hi


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--checkpoint", help="state dict of a trained Raindrop_v2 (torch.save); --synthetic without it: "
                    "synthetic weights")
    ap.add_argument("--nhead", type=int, default=2)
    ap.add_argument("--dropout", type=float, default=0.2)
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--data", help="PTdict_list.npy (P12 / P19 / eICU: list of dicts; PAM: plain array)")
    src.add_argument("--synthetic", help="synthetic data of a raindrop_b200.synth configuration (P12, P19, PAM, ...)")
    ap.add_argument("--split", help="split file (idx_train, idx_val, idx_test); without it every sample is used")
    ap.add_argument("--part", default="test", choices=["train", "val", "test"])
    ap.add_argument("--n-samples", type=int, default=512, help="--synthetic: samples explained")
    ap.add_argument("--n-train", type=int, default=2048, help="--synthetic: samples the weights and bounds come from")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--batch-size", type=int, default=512)
    ap.add_argument("--mad-floor", type=float, default=0.25)
    ap.add_argument("--beta", type=float, default=0.1)
    ap.add_argument("--kappa", type=float, default=0.0)
    ap.add_argument("--n-search", type=int, default=5)
    ap.add_argument("--n-steps", type=int, default=100)
    ap.add_argument("--n-restarts", type=int, default=1)
    ap.add_argument("--step-size", type=float, default=0.01)
    ap.add_argument("--out", help="CSV of per-sample rows")
    args = ap.parse_args()
    from raindrop_b200.counterfactual import counterfactual
    device = torch.device("cuda")
    model, train, part, stdf = load_parts(args, device)
    model = model.to(device).eval()
    N = model.d_inp
    w, lo, hi = sensor_stats(train[0], args.mad_floor)
    rows, n_valid, changed = [], 0, np.zeros(N, np.int64)
    for s in range(0, part[0].shape[1], args.batch_size):
        sl = slice(s, s + args.batch_size)
        x = part[0][:, sl]
        r = counterfactual(model, x, None if part[1] is None else part[1][sl], part[2][:, sl], part[3][sl], weights=w,
                           lower=lo, upper=hi, beta=args.beta, kappa=args.kappa, n_search=args.n_search,
                           n_steps=args.n_steps, n_restarts=args.n_restarts, step_size=args.step_size, seed=args.seed)
        d = (r.src[:, :, :N].double() - x[:, :, :N].double()).cpu().numpy()       # [T, b, N], normalised units
        big = np.abs(d).max(axis=0) * stdf[None, :N]                              # largest change, original units
        sc = r.sensors_changed.cpu().numpy()
        for j in range(x.shape[1]):
            valid = bool(r.valid[j])
            n_valid += valid
            if valid:
                changed += sc[j]
            rows.append([s + j, int(valid), float(r.distance[j]), int(r.l0[j]), int(r.target[j]),
                         ";".join(str(n) for n in np.nonzero(sc[j])[0])] + [float(v) for v in big[j]])
    total = len(rows)
    print("validity rate: %.4f (%d of %d)" % (n_valid / max(total, 1), n_valid, total))
    order = np.argsort(-changed, kind="stable")[:10]
    print("sensors changed most often (sensor: valid samples): " +
          ", ".join("%d: %d" % (n, changed[n]) for n in order if changed[n] > 0))
    if args.out:
        with open(args.out, "w", newline="") as f:
            wr = csv.writer(f)
            wr.writerow(["sample", "valid", "distance", "l0", "target", "sensors_changed"] +
                        ["max_change_sensor_%d" % n for n in range(N)])
            wr.writerows(rows)


if __name__ == "__main__":
    main()
