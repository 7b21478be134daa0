#!/usr/bin/env python
"""Which attribution method should I trust on this checkpoint?  Deletion / insertion AUC, AOPC and infidelity (raw and
normalised) of each method's player ranking, computed on the device by raindrop_b200.faithfulness:

    python tools/attribution_faithfulness.py --checkpoint model.pt --data P19data/processed_data/PTdict_list.npy \\
        --split P19data/splits/phy19_split1_new.npy --part test
    python tools/attribution_faithfulness.py --synthetic P19 --n-samples 256 --window 6

Methods: ig (integrated gradients summed per player by player_attributions), ablation, shapley, kernelshap, random
(uniform scores, seeded) and, with --density-scores FILE, a global sensor order such as an IG_density_scores_*.npy
(column 0, most important first) turned into a [P] score shared by every sample.  Players are sensors, or (sensor,
window) players with --window W.  Targets are the labels (--outcomes) or the predicted class, baselines zero.  Without
--checkpoint the model has the synthetic weights of raindrop_b200.synth (--synthetic only).

Prints one JSON line per method: mean and standard error over samples of every metric, and the card's name and power
limit.  It is an evaluation, not a test: nothing is thresholded.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_valuation import card  # noqa: E402
from ig_sensor_ranking import model_from_state_dict  # noqa: E402

METHODS = ("ig", "ablation", "shapley", "kernelshap", "random")
METRICS = ("deletion_auc", "insertion_auc", "aopc", "deletion_auc_prob", "insertion_auc_prob", "infidelity",
           "infidelity_normalized")


def load_inputs(args, model, device):
    """(src, static, times, y or None) of the evaluated samples."""
    from raindrop_b200 import data as RD
    from raindrop_b200.synth import make_batch, model_config
    N, T = model.d_inp, model.max_len
    if args.synthetic:
        b = make_batch(model_config(args.synthetic), args.n_samples, seed=args.seed, device=device)
        return b["src"], b["static"], b["times"], None
    raw = np.load(args.data, allow_pickle=True)
    is_list = raw.dtype == object and isinstance(raw.flat[0], dict)
    P_raw, minutes, static = RD.load_ptdict_list(args.data) if is_list else RD.load_array_dataset(args.data)
    if P_raw.shape[1] != T or P_raw.shape[2] != N:
        raise SystemExit("data [n, T=%d, F=%d] does not match the checkpoint (max_len %d, d_inp %d)"
                         % (P_raw.shape[1], P_raw.shape[2], T, N))
    labels = None
    if args.outcomes:
        labels = np.asarray(np.load(args.outcomes, allow_pickle=True)).reshape(len(P_raw), -1)[:, args.label_col]
    idx_train = idx = np.arange(len(P_raw))
    if args.split:
        parts = RD.load_split(args.split)
        idx_train, idx = parts[0], parts[("train", "val", "test").index(args.part)]
    idx = idx[:args.n_samples] if args.n_samples else idx
    mf, stdf = RD.feature_stats(torch.as_tensor(P_raw[idx_train]).to(device))
    st = None if (static is None or not model.static) else static[idx]
    y0 = labels[idx] if labels is not None else np.zeros(len(idx), dtype=np.int64)
    src, st, times, y = RD.tensorize_normalize(P_raw[idx], minutes[idx], st, y0, mf, stdf, device=device)
    return src, st, times, (y if labels is not None else None)


def density_scores(path, N, P):
    """[P] scores from a global sensor order (column 0 of an IG_density_scores_*.npy, most important first): sensor at
    position i scores N - i; a static player scores 0."""
    order = np.load(path, allow_pickle=True)[:, 0].astype(np.int64)
    if sorted(order.tolist()) != list(range(N)):
        raise SystemExit("%s: column 0 is not a permutation of the %d sensors" % (path, N))
    s = np.zeros(P, dtype=np.float32)
    s[order] = N - np.arange(N)
    return torch.from_numpy(s)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--checkpoint", help="state dict of a trained Raindrop_v2 (torch.save)")
    ap.add_argument("--nhead", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    src_arg = ap.add_mutually_exclusive_group(required=True)
    src_arg.add_argument("--data", help="PTdict_list.npy (P12 / P19: list of dicts; PAM: plain array)")
    src_arg.add_argument("--synthetic", help="a raindrop_b200.synth configuration (P12, P19, PAM, ...)")
    ap.add_argument("--outcomes", help="arr_outcomes.npy: labels in column --label-col (default: predicted class)")
    ap.add_argument("--label-col", type=int, default=-1)
    ap.add_argument("--split")
    ap.add_argument("--part", default="test", choices=["train", "val", "test"])
    ap.add_argument("--n-samples", type=int, default=256, help="samples evaluated (data: the first of the part)")
    ap.add_argument("--methods", default=",".join(METHODS))
    ap.add_argument("--density-scores", help="a global sensor order, e.g. IG_density_scores_P19.npy")
    ap.add_argument("--window", type=float, default=0.0, help="(sensor, window) players of this width in `times` units")
    ap.add_argument("--ig-steps", type=int, default=50)
    ap.add_argument("--shapley-samples", type=int, default=25)
    ap.add_argument("--kernel-shap-samples", type=int, default=None)
    ap.add_argument("--infidelity-samples", type=int, default=1000)
    ap.add_argument("--p-remove", type=float, default=0.5)
    ap.add_argument("--batch-size", type=int, default=128)
    args = ap.parse_args()
    if not args.checkpoint and not args.synthetic:
        ap.error("--data needs --checkpoint")

    from raindrop_b200 import attribution as A
    from raindrop_b200 import faithfulness as FA
    from raindrop_b200.synth import model_config, synth_weights
    if not torch.cuda.is_available():
        raise SystemExit("the faithfulness calls run on a CUDA device")
    device = torch.device("cuda", torch.cuda.current_device())
    if args.checkpoint:
        model = model_from_state_dict(torch.load(args.checkpoint, map_location="cpu"), args.nhead, args.seed, device)
    else:
        from raindrop_b200.models_rd import Raindrop_v2
        cfg = model_config(args.synthetic)
        torch.manual_seed(args.seed)
        model = Raindrop_v2(cfg["d_inp"], cfg["d_model"], cfg["nhead"], cfg["nhid"], cfg["nlayers"], 0.0,
                            cfg["max_len"], cfg["d_static"], cfg["MAX"], 0.5, "mean", cfg["n_classes"],
                            torch.ones(cfg["d_inp"], cfg["d_inp"]), **({} if cfg["static"] else {"static": False}))
        synth_weights(model, cfg, seed=args.seed)
        model = model.to(device)
    model.eval()
    P_all, S_all, T_all, y_all = load_inputs(args, model, device)
    N, n = model.d_inp, P_all.shape[1]
    n_windows = max(1, int(np.ceil(float(T_all.max()) / args.window))) if args.window else 1
    methods = [m for m in args.methods.split(",") if m]
    if args.density_scores:
        if args.window:
            ap.error("--density-scores ranks sensors: it does not take --window")
        methods.append("density")
    rows = {m: {k: [] for k in METRICS} for m in methods}
    gen = torch.Generator(device="cpu").manual_seed(args.seed)
    for s in range(0, n, args.batch_size):
        e = min(n, s + args.batch_size)
        src, times = P_all[:, s:e], T_all[:, s:e]
        lengths = torch.sum(times > 0, dim=0)
        static = None if S_all is None else S_all[s:e]
        target = None if y_all is None else y_all[s:e]
        mask = None
        if args.window:
            mask, _ = A.time_window_mask(times, args.window, n_windows=n_windows, sensor_groups=N)
        call = (model, src, static, times, lengths)
        players = dict(feature_mask=mask)
        for m in methods:
            if m == "ig":
                attr_src, attr_st = A.integrated_gradients(*call, target=target, n_steps=args.ig_steps)
                phi = FA.player_attributions(attr_src, attr_st if model.static else None, feature_mask=mask)
            elif m == "ablation":
                phi = A.feature_ablation(*call, target=target, **players)
            elif m == "shapley":
                phi = A.shapley_value_sampling(*call, target=target, n_samples=args.shapley_samples, seed=args.seed,
                                               **players)
            elif m == "kernelshap":
                phi = A.kernel_shap(*call, target=target, n_samples=args.kernel_shap_samples, seed=args.seed, **players)
            elif m == "random":
                G = N * n_windows if args.window else N
                phi = torch.rand(e - s, G + (1 if model.static else 0), generator=gen)
            elif m == "density":
                phi = density_scores(args.density_scores, N, N + (1 if model.static else 0))
            else:
                raise SystemExit("unknown method %r" % m)
            cur = FA.deletion_curves(*call, phi, target=target, **players)
            inf = FA.infidelity(*call, phi, target=target, n_samples=args.infidelity_samples, p_remove=args.p_remove,
                                seed=args.seed, **players)
            r = rows[m]
            r["deletion_auc"].append(cur.deletion_auc())
            r["insertion_auc"].append(cur.insertion_auc())
            r["aopc"].append(cur.aopc())
            r["deletion_auc_prob"].append(cur.deletion_auc("probability"))
            r["insertion_auc_prob"].append(cur.insertion_auc("probability"))
            r["infidelity"].append(inf.infidelity)
            r["infidelity_normalized"].append(FA.infidelity_from_moments(inf.moments, normalize=True))
    gpu = card()
    for m in methods:
        out = {"method": m, "samples": n, "players": "sensor x window %g" % args.window if args.window else "sensor",
               "card": gpu}
        for k, v in rows[m].items():
            x = torch.cat(v).cpu().numpy()
            out[k] = {"mean": float(x.mean()), "se": float(x.std(ddof=1) / np.sqrt(len(x))) if len(x) > 1 else 0.0}
        print(json.dumps(out))


if __name__ == "__main__":
    main()
