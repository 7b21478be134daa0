#!/usr/bin/env python
"""How well the out-of-distribution scores of a trained Raindrop_v2 (raindrop_b200.ood) flag shifted data:

    python tools/ood_eval.py --checkpoint model.pt --data P19data/processed_data/PTdict_list.npy \\
        --outcomes P19data/processed_data/arr_outcomes.npy --split P19data/splits/phy19_split1_new.npy --part test
    python tools/ood_eval.py --synthetic P19 --n-train 4096 --n-samples 1024

The data arguments are those of tools/certify.py; without --checkpoint the model has the synthetic weights of
raindrop_b200.synth (a smoke run, not a trained model), and --synthetic draws the train part (--n-train samples) and the
evaluated part (--n-samples) from different seeds.  The detector is fitted on the train part (ood_fit, layer --layer);
the evaluated part is the in-distribution set.  Shifted copies of it are the out-of-distribution sets:
  missing sensors: a fraction --missing-ratios of the sensors zeroed per sample (data.removal_indices /
                   remove_features_, the leave-sensors-out setting of the Raindrop paper), numpy seed --seed;
  noise:           Gaussian noise of standard deviation --noise-sigmas (normalised units) on the observed values.
For each score (msp, energy, mahalanobis, knn) and shift it prints AUROC and FPR at 95 % TPR (ood_metrics), then one
JSON line.  --out writes the per-sample scores of every set to an .npz file.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from adv_robustness import load_split  # noqa: E402

SCORES = ("msp", "energy", "mahalanobis", "knn")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--checkpoint", help="state dict of a trained Raindrop_v2 (torch.save); default: synthetic weights")
    ap.add_argument("--nhead", type=int, default=2)
    ap.add_argument("--dropout", type=float, default=0.2)
    ap.add_argument("--seed", type=int, default=0, help="torch.manual_seed before building the model (R_u); data seed")
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--data", help="PTdict_list.npy (P12 / P19 / eICU: list of dicts; PAM: plain array)")
    src.add_argument("--synthetic", help="synthetic batches of a raindrop_b200.synth configuration (P12, P19, PAM, ...)")
    ap.add_argument("--outcomes", help="arr_outcomes.npy: labels in column --label-col")
    ap.add_argument("--label-col", type=int, default=-1)
    ap.add_argument("--split", help="split file (idx_train, idx_val, idx_test); without it every sample is used")
    ap.add_argument("--part", default="test", choices=["val", "test"], help="the in-distribution part")
    ap.add_argument("--n-train", type=int, default=4096, help="--synthetic: training samples")
    ap.add_argument("--n-samples", type=int, default=1024, help="--synthetic: evaluated samples")
    ap.add_argument("--batch-size", type=int, default=1024)
    ap.add_argument("--layer", default="hidden", choices=["hidden", "pooled"])
    ap.add_argument("--k", type=int, default=50)
    ap.add_argument("--missing-ratios", type=float, nargs="*", default=[0.3, 0.5, 0.7])
    ap.add_argument("--noise-sigmas", type=float, nargs="*", default=[0.5, 1.0, 2.0])
    ap.add_argument("--out", help="per-sample scores (.npz); default: not written")
    args = ap.parse_args()

    from raindrop_b200 import data as RD
    from raindrop_b200 import ood as OOD
    if not torch.cuda.is_available():
        raise SystemExit("ood_eval runs on a CUDA device")
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
    part = args.part
    if args.synthetic:
        n_eval, args.n_samples, args.seed = args.n_samples, args.n_train, args.seed + 1
        train = load_split(args, model, device)
        args.n_samples, args.seed = n_eval, args.seed - 1
    else:
        args.part = "train"
        train = load_split(args, model, device)
        args.part = part
    P, Pstatic, Ptime, _ = load_split(args, model, device)
    Ptr, Pstr, Pttr, ytr = train
    det = OOD.ood_fit(model, dict(src=Ptr, static=Pstr, times=Pttr, lengths=torch.sum(Pttr > 0, dim=0), y=ytr),
                      layer=args.layer)
    k = min(args.k, det.n_bank)

    def scores(Px):
        out = {s: [] for s in SCORES}
        for s in range(0, Px.shape[1], args.batch_size):
            e = min(Px.shape[1], s + args.batch_size)
            times = Ptime[:, s:e]
            r = OOD.ood_scores(model, det, Px[:, s:e].contiguous(), None if Pstatic is None else Pstatic[s:e], times,
                               torch.sum(times > 0, dim=0), k=k)
            for name in SCORES:
                out[name].append(getattr(r, name).double().cpu().numpy())
        return {name: np.concatenate(v) for name, v in out.items()}

    N = model.d_inp
    sets = {"in": scores(P)}
    np.random.seed(args.seed)
    for ratio in args.missing_ratios:
        Pm = P.clone()
        RD.remove_features_(Pm, RD.removal_indices(P.shape[1], N, ratio))
        sets["missing_%g" % ratio] = scores(Pm)
    g = torch.Generator(device=device).manual_seed(args.seed)
    for sigma in args.noise_sigmas:
        Pn = P.clone()
        obs = Pn[:, :, N:] > 0
        noise = sigma * torch.randn(Pn[:, :, :N].shape, generator=g, device=device)
        Pn[:, :, :N] = torch.where(obs, Pn[:, :, :N] + noise, Pn[:, :, :N])
        sets["noise_%g" % sigma] = scores(Pn)
    result = {}
    print("%d training samples (layer %s, rank %d, k %d), %d in-distribution samples" % (det.n, args.layer, det.rank, k,
                                                                                     P.shape[1]))
    print("%-14s" % "shift" + "".join("%24s" % s for s in SCORES))
    for name, sc in sets.items():
        if name == "in":
            continue
        m = {s: OOD.ood_metrics(sets["in"][s], sc[s]) for s in SCORES}
        result[name] = {s: dict(auroc=m[s]["auroc"], fpr_at_95_tpr=m[s]["fpr_at_95_tpr"]) for s in SCORES}
        print("%-14s" % name + "".join("   AUROC %.3f FPR95 %.3f" % (m[s]["auroc"], m[s]["fpr_at_95_tpr"])
                                       for s in SCORES))
    if args.out:
        np.savez(args.out, **{"%s/%s" % (name, s): v for name, sc in sets.items() for s, v in sc.items()})
    print(json.dumps(dict(layer=args.layer, rank=det.rank, k=k, n_train=det.n, n_in=int(P.shape[1]), shifts=result)))


if __name__ == "__main__":
    main()
