#!/usr/bin/env python
"""Writes the TracIn influence of a data split's training samples on its test samples (raindrop_b200.influence) for one
or more checkpoints of a trained Raindrop_v2:

    python tools/tracin.py --checkpoint ep10.pt --checkpoint ep20.pt --lr 1e-4 --data P19data/processed_data/PTdict_list.npy \\
        --outcomes P19data/processed_data/arr_outcomes.npy --split P19data/splits/phy19_split1_new.npy --name P19
    python tools/tracin.py --checkpoint model.pt --synthetic P19 --n-samples 512 --n-test 32

The checkpoints, data, split and normalisation are read as tools/mc_uncertainty.py reads them (the first checkpoint
builds the model; every checkpoint must hold the same trained tensors).  Each test sample is scored with its predicted
class.  Files, under --out-dir with suffix _<name>.npy:
  tracin_proponents   int64 [n_test, k]: training indices (into the split's training part) of the k largest scores
  tracin_proponent_scores, tracin_opponents, tracin_opponent_scores: the scores, and the k most negative
  tracin_self_influence_order  int64 [n_train]: training indices by decreasing self-influence (candidate mislabels)
  tracin_self_influence  float64 [n_train]: sum_c lr_c ||g||^2 per training sample

--projection DIM scores through TracIn-RP sketches instead (influence.project / tracin_sketch: each gradient row projected
onto DIM random +-1 directions fixed by --projection-seed); --save-sketch PATH writes the training set's sketch and
--load-sketch PATH reuses one (it must match the checkpoints, fields, DIM and seed).  The files are the same; the
self-influence stays exact.

--method ekfac scores with EK-FAC influence functions instead (influence.ekfac_factors / ekfac_influence, the true
Fisher at the single checkpoint's weights, preconditioned by its inverse with --damping or 0.1 of each block's mean
eigenvalue); --save-factors PATH / --load-factors PATH write or reuse the training set's factors.  The files keep their
names; the self-influence is EK-FAC's sum_j G~_j^2 / (Lambda_j + lambda).
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from ig_sensor_ranking import model_from_state_dict  # noqa: E402


def top_k(scores, k):
    """(proponents, their scores, opponents, their scores) per row of scores [n_test, n_train] (numpy)."""
    k = min(k, scores.shape[1])
    order = np.argsort(-scores, axis=1, kind="stable")
    pro, opp = order[:, :k], order[:, ::-1][:, :k]
    return pro, np.take_along_axis(scores, pro, 1), opp, np.take_along_axis(scores, opp, 1)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--checkpoint", action="append", required=True, help="state dict (torch.save); repeat for several")
    ap.add_argument("--lr", type=float, action="append", help="learning rate of each checkpoint (default 1 each)")
    ap.add_argument("--nhead", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0, help="torch.manual_seed before building the model (R_u)")
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--data", help="PTdict_list.npy (P12 / P19 / eICU: list of dicts; PAM: plain array)")
    src.add_argument("--synthetic", help="synthetic samples of a raindrop_b200.synth configuration (P12, P19, PAM, ...)")
    ap.add_argument("--outcomes", help="arr_outcomes.npy: labels in column --label-col (required with --data)")
    ap.add_argument("--label-col", type=int, default=-1)
    ap.add_argument("--split", help="split file (idx_train, idx_val, idx_test); without it every sample is in both parts")
    ap.add_argument("--part", default="test", choices=["val", "test"], help="the part whose samples are scored")
    ap.add_argument("--n-samples", type=int, default=512, help="--synthetic: number of training samples")
    ap.add_argument("--n-test", type=int, default=32, help="--synthetic: number of test samples")
    ap.add_argument("--top-k", type=int, default=10)
    ap.add_argument("--fields", nargs="*", help="restrict to these state-dict keys (privacy.sqnorm_fields)")
    ap.add_argument("--projection", type=int, metavar="DIM", help="score through random-projection sketches of DIM dims")
    ap.add_argument("--projection-seed", type=int, default=0, help="seed of the projection's +-1 directions")
    ap.add_argument("--save-sketch", metavar="PATH", help="--projection: write the training set's sketch here")
    ap.add_argument("--load-sketch", metavar="PATH", help="--projection: reuse this training-set sketch")
    ap.add_argument("--method", default="tracin", choices=["tracin", "ekfac"],
                    help="ekfac: EK-FAC influence functions at the first checkpoint's weights (influence.ekfac_*)")
    ap.add_argument("--damping", type=float, help="--method ekfac: one damping for every block (default 0.1 mean)")
    ap.add_argument("--save-factors", metavar="PATH", help="--method ekfac: write the training set's EK-FAC factors here")
    ap.add_argument("--load-factors", metavar="PATH", help="--method ekfac: reuse these EK-FAC factors")
    ap.add_argument("--name", help="file name suffix (default: the synthetic configuration or 'dataset')")
    ap.add_argument("--out-dir", default=".")
    args = ap.parse_args()

    from raindrop_b200 import data as RD
    from raindrop_b200.influence import (EKFACFactors, GradientSketch, ekfac_factors, ekfac_influence, ekfac_self_influence,
                                         project, self_influence, tracin, tracin_sketch)
    from raindrop_b200.synth import make_batch, model_config
    if not torch.cuda.is_available():
        raise SystemExit("tracin runs on a CUDA device")
    if (args.save_sketch or args.load_sketch) and not args.projection:
        raise SystemExit("--save-sketch and --load-sketch need --projection")
    if (args.save_factors or args.load_factors or args.damping is not None) and args.method != "ekfac":
        raise SystemExit("--save-factors, --load-factors and --damping need --method ekfac")
    if args.method == "ekfac" and (args.projection or len(args.checkpoint) != 1):
        raise SystemExit("--method ekfac takes one --checkpoint and no --projection")
    lrs = args.lr or [1.0] * len(args.checkpoint)
    if len(lrs) != len(args.checkpoint):
        raise SystemExit("give one --lr per --checkpoint")
    device = torch.device("cuda", torch.cuda.current_device())
    sds = [torch.load(p, map_location="cpu") for p in args.checkpoint]
    model = model_from_state_dict(sds[0], args.nhead, args.seed, device).eval()
    ckpts = [({k: v.to(device) for k, v in sd.items()}, lr) for sd, lr in zip(sds, lrs)]
    N, T = model.d_inp, model.max_len
    if args.synthetic:
        cfg = model_config(args.synthetic)
        if cfg["d_inp"] != N or cfg["max_len"] != T or cfg["static"] != model.static:
            raise SystemExit("--synthetic %s does not match the checkpoint (d_inp %d, max_len %d)" % (args.synthetic, N, T))
        tr = make_batch(cfg, args.n_samples, seed=args.seed, device=device)
        te = make_batch(cfg, args.n_test, seed=args.seed + 1, device=device)
        train = RD.DeviceDataset(tr["src"], tr["static"], tr["times"], tr["y"], device=device)
        test = dict(src=te["src"], static=te["static"], times=te["times"], lengths=te["lengths"], y=None)
        name = args.name or args.synthetic
    else:
        if not args.outcomes:
            raise SystemExit("--data needs --outcomes: the training samples' gradients are of their labels")
        raw = np.load(args.data, allow_pickle=True)
        is_list = raw.dtype == object and isinstance(raw.flat[0], dict)
        P_raw, minutes, static = RD.load_ptdict_list(args.data) if is_list else RD.load_array_dataset(args.data)
        if P_raw.shape[1] != T or P_raw.shape[2] != N:
            raise SystemExit("data [n, T=%d, F=%d] does not match the checkpoint (max_len %d, d_inp %d)"
                             % (P_raw.shape[1], P_raw.shape[2], T, N))
        n = len(P_raw)
        idx_train, idx_test = np.arange(n), np.arange(n)
        if args.split:
            parts = RD.load_split(args.split)
            idx_train, idx_test = parts[0], parts[("train", "val", "test").index(args.part)]
        labels = np.asarray(np.load(args.outcomes, allow_pickle=True)).reshape(n, -1)[:, args.label_col].astype(np.int64)
        mf, stdf = RD.feature_stats(torch.as_tensor(P_raw[idx_train]).to(device))

        def part(idx):
            st = None if (static is None or not model.static) else static[idx]
            return RD.tensorize_normalize(P_raw[idx], minutes[idx], st, labels[idx], mf, stdf, device=device)
        P, Ps, Pt, y = part(idx_train)
        train = RD.DeviceDataset(P, Ps, Pt, y, device=device)
        P, Ps, Pt, _ = part(idx_test)
        test = dict(src=P, static=Ps, times=Pt, lengths=torch.sum(Pt > 0, dim=0), y=None)
        name = args.name or "dataset"

    if args.method == "ekfac":
        if args.load_factors:
            factors = EKFACFactors.load(args.load_factors, map_location=device)
        else:
            factors = ekfac_factors(model, train, fields=args.fields)
        if args.save_factors:
            factors.save(args.save_factors)
        scores = ekfac_influence(model, test, train, factors, damping=args.damping).cpu().numpy()
        si = ekfac_self_influence(model, train, factors, damping=args.damping).cpu().numpy()
    elif args.projection:
        kw = dict(checkpoints=ckpts, dim=args.projection, seed=args.projection_seed, fields=args.fields)
        if args.load_sketch:
            train_sketch = GradientSketch.load(args.load_sketch, map_location=device)
        else:
            train_sketch = project(model, train, **kw)
        if args.save_sketch:
            train_sketch.save(args.save_sketch)
        scores = tracin_sketch(project(model, test, **kw), train_sketch).cpu().numpy()
    else:
        scores = tracin(model, test, train, checkpoints=ckpts, fields=args.fields).cpu().numpy()
    if args.method != "ekfac":
        si = self_influence(model, train, checkpoints=ckpts, fields=args.fields).cpu().numpy()
    pro, pro_s, opp, opp_s = top_k(scores, args.top_k)
    out = dict(tracin_proponents=pro, tracin_proponent_scores=pro_s, tracin_opponents=opp, tracin_opponent_scores=opp_s,
               tracin_self_influence_order=np.argsort(-si, kind="stable"), tracin_self_influence=si)
    os.makedirs(args.out_dir, exist_ok=True)
    for k, v in out.items():
        np.save(os.path.join(args.out_dir, "%s_%s.npy" % (k, name)), v)
    print("wrote %d files to %s: %d test x %d training samples, %d checkpoint(s); highest self-influence: %s"
          % (len(out), args.out_dir, scores.shape[0], scores.shape[1], len(ckpts), out["tracin_self_influence_order"][:5]))


if __name__ == "__main__":
    main()
