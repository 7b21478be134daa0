#!/usr/bin/env python
"""Writes IG_density_scores_<name>.npy, the sensor ranking the reference's leave-sensors-out experiment with
feature_removal_level='set' reads (code/Raindrop.py:227-231), from a trained Raindrop_v2 and a data set (or, with
--method ablation / shapley / kernelshap, Ablation_density_scores_<name>.npy / Shapley_density_scores_<name>.npy /
KernelSHAP_density_scores_<name>.npy):

    python tools/ig_sensor_ranking.py --checkpoint model.pt --data P19data/processed_data/PTdict_list.npy \\
        --outcomes P19data/processed_data/arr_outcomes.npy --split P19data/splits/phy19_split1_new.npy --part test \\
        --sensor-names sensors.txt --name P19
    python tools/ig_sensor_ranking.py --checkpoint model.pt --synthetic P19 --n-samples 512

The checkpoint is a state dict as code/Raindrop.py:374 saves it.  The hyper-parameters are read from its shapes; nhead
is not recoverable from them and defaults to the reference's 2.  R_u (code/models_rd.py:241) is not a registered
parameter, so it is not in the state dict; it comes from the model's construction after torch.manual_seed(--seed), as in
the reference.  Normalisation statistics are those of the split's training part (code/Raindrop.py:192-205).

Per batch, raindrop_b200.attribution.integrated_gradients (zero baselines, --steps Gauss-Legendre nodes, target = the
label when --outcomes is given, else the predicted class) attributes the value half of src; a sensor's score is the mean
over samples of sum_t |attribution|, and the ranking lists (index, name) in descending score.  Column 0 of the file is
what data.removal_indices(..., level="set", density_scores=...) takes.  The recipe behind the reference's shipped files
is not recorded, so this ranking is not claimed to reproduce them.

--method ablation / shapley rank by the attribution of REMOVING each sensor (zeroing its value columns, as the
experiment does; the static vector is held fixed): raindrop_b200.attribution.feature_ablation, or
shapley_value_sampling with --shapley-samples permutations (seed --seed), or kernel_shap with --kernel-shap-samples
coalitions (default 2P + 2048; seed --seed).  A sensor's score is the mean over samples of |attribution|; the file has
the same [N, 2] layout.

--window W with --method ablation / shapley / kernelshap attributes (sensor, time window) cells instead
(raindrop_b200.attribution.time_window_mask, windows of W units of `times`, padding rows in no window) and writes
<Method>_time_sensor_scores_<name>.npy: float64 [n_windows, N], the mean over samples of |attribution| per (window,
sensor).  n_windows = max(1, ceil(max(times) / W)) over the whole data set, so every batch shares the layout.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def model_from_state_dict(sd, nhead, seed, device, dropout=0.0):
    """Raindrop_v2 with the hyper-parameters the state dict's shapes give (code/Raindrop.py:245-251), weights loaded.
    The dropout probability is not in the state dict; it only matters for training-mode forwards."""
    from raindrop_b200.models_rd import Raindrop_v2
    static = "emb.weight" in sd
    d_inp, C = sd["ob_propagation.nodewise_weights"].shape          # [n_nodes, T * d_ob]
    nhid, D = sd["transformer_encoder.layers.0.linear1.weight"].shape
    d_model = D - 16
    d_ob = d_model // d_inp
    nlayers = len({k.split(".")[2] for k in sd if k.startswith("transformer_encoder.layers.")})
    d_static = sd["emb.weight"].shape[1] if static else 1
    n_classes = sd["mlp_static.2.weight"].shape[0]
    torch.manual_seed(seed)
    kw = {} if static else {"static": False}
    m = Raindrop_v2(d_inp, d_model, nhead, nhid, nlayers, dropout, C // d_ob, d_static, 100, 0.5, "mean", n_classes,
                    torch.ones(d_inp, d_inp), **kw)
    m.load_state_dict(sd)
    return m.to(device).eval()


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--checkpoint", required=True, help="state dict of a trained Raindrop_v2 (torch.save)")
    ap.add_argument("--nhead", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0, help="torch.manual_seed before building the model (R_u)")
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--data", help="PTdict_list.npy (P12 / P19 / eICU: list of dicts; PAM: plain array)")
    src.add_argument("--synthetic", help="synthetic batches of a raindrop_b200.synth configuration (P12, P19, PAM, ...)")
    ap.add_argument("--outcomes", help="arr_outcomes.npy: labels in column --label-col (default: predicted class)")
    ap.add_argument("--label-col", type=int, default=-1)
    ap.add_argument("--split", help="split file (idx_train, idx_val, idx_test); without it every sample is used")
    ap.add_argument("--part", default="test", choices=["train", "val", "test"])
    ap.add_argument("--n-samples", type=int, default=512, help="--synthetic: number of samples")
    ap.add_argument("--sensor-names", help="text file, one sensor name per line (default: the indices)")
    ap.add_argument("--method", default="ig", choices=["ig", "ablation", "shapley", "kernelshap"])
    ap.add_argument("--steps", type=int, default=50, help="--method ig: Gauss-Legendre nodes per attribution")
    ap.add_argument("--shapley-samples", type=int, default=25, help="--method shapley: permutations per batch")
    ap.add_argument("--kernel-shap-samples", type=int, default=None,
                    help="--method kernelshap: sampled coalitions per batch (default 2P + 2048)")
    ap.add_argument("--window", type=float, default=0.0,
                    help="--method ablation / shapley / kernelshap: (sensor, time window) players, windows of W units of times")
    ap.add_argument("--batch-size", type=int, default=128)
    ap.add_argument("--name", help="file name suffix (default: the synthetic configuration or 'dataset')")
    ap.add_argument("--out-dir", default=".")
    args = ap.parse_args()
    if args.window and args.method == "ig":
        ap.error("--window needs --method ablation, shapley or kernelshap")

    from raindrop_b200 import data as RD
    from raindrop_b200.attribution import (feature_ablation, integrated_gradients, kernel_shap, sensor_importance,
                                           sensor_ranking, shapley_value_sampling, time_window_mask)
    from raindrop_b200.synth import make_batch, model_config
    device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else None
    if device is None:
        raise SystemExit("attribution runs on a CUDA device")
    model = model_from_state_dict(torch.load(args.checkpoint, map_location="cpu"), args.nhead, args.seed, device)
    N, T = model.d_inp, model.max_len

    if args.synthetic:
        cfg = model_config(args.synthetic)
        if cfg["d_inp"] != N or cfg["max_len"] != T or cfg["static"] != model.static:
            raise SystemExit("--synthetic %s does not match the checkpoint (d_inp %d, max_len %d)" % (args.synthetic, N, T))
        b = make_batch(cfg, args.n_samples, seed=args.seed, device=device)
        P, Pstatic, Ptime, y = b["src"], b["static"], b["times"], None
        name = args.name or args.synthetic
    else:
        raw = np.load(args.data, allow_pickle=True)
        is_list = raw.dtype == object and isinstance(raw.flat[0], dict)
        P_raw, minutes, static = RD.load_ptdict_list(args.data) if is_list else RD.load_array_dataset(args.data)
        if P_raw.shape[1] != T or P_raw.shape[2] != N:
            raise SystemExit("data [n, T=%d, F=%d] does not match the checkpoint (max_len %d, d_inp %d)"
                             % (P_raw.shape[1], P_raw.shape[2], T, N))
        labels = None
        if args.outcomes:
            labels = np.asarray(np.load(args.outcomes, allow_pickle=True)).reshape(len(P_raw), -1)[:, args.label_col]
        n = len(P_raw)
        idx_train, idx = np.arange(n), np.arange(n)
        if args.split:
            parts = RD.load_split(args.split)
            idx_train, idx = parts[0], parts[("train", "val", "test").index(args.part)]
        mf, stdf = RD.feature_stats(torch.as_tensor(P_raw[idx_train]).to(device))
        st = None if (static is None or not model.static) else static[idx]
        y0 = labels[idx] if labels is not None else np.zeros(len(idx), dtype=np.int64)
        P, Pstatic, Ptime, y = RD.tensorize_normalize(P_raw[idx], minutes[idx], st, y0, mf, stdf, device=device)
        if labels is None:
            y = None
        name = args.name or "dataset"
    names = None
    if args.sensor_names:
        with open(args.sensor_names) as f:
            names = [s.strip() for s in f if s.strip()]

    n_windows = 1
    if args.window:
        n_windows = max(1, int(np.ceil(float(Ptime.max()) / args.window)))
    total = torch.zeros(n_windows * N, dtype=torch.float64, device=device)
    n = P.shape[1]
    for s in range(0, n, args.batch_size):
        e = min(n, s + args.batch_size)
        src, times = P[:, s:e], Ptime[:, s:e]
        lengths = torch.sum(times > 0, dim=0)
        static = None if Pstatic is None else Pstatic[s:e]
        target = None if y is None else y[s:e]
        if args.method == "ig":
            attr_src, _ = integrated_gradients(model, src, static, times, lengths, target=target, n_steps=args.steps)
            total += sensor_importance(attr_src, N).double() * (e - s)
            continue
        fixed = (None, static)                  # statics held fixed: only sensors are players that change the input
        mask = None
        if args.window:
            mask, _ = time_window_mask(times, args.window, n_windows=n_windows, sensor_groups=N)
        if args.method == "ablation":
            attr, _ = feature_ablation(model, src, static, times, lengths, target=target, baselines=fixed,
                                       feature_mask=mask)
        elif args.method == "kernelshap":
            attr, _ = kernel_shap(model, src, static, times, lengths, target=target, baselines=fixed,
                                  n_samples=args.kernel_shap_samples, seed=args.seed, feature_mask=mask)
        else:
            attr, _ = shapley_value_sampling(model, src, static, times, lengths, target=target, baselines=fixed,
                                             n_samples=args.shapley_samples, seed=args.seed, feature_mask=mask)
        total[:attr.shape[1]] += attr.double().abs().sum(dim=0)      # a batch may not reach the last windows
    prefix = {"ig": "IG", "ablation": "Ablation", "shapley": "Shapley", "kernelshap": "KernelSHAP"}[args.method]
    if args.window:
        scores = (total / n).view(n_windows, N).cpu().numpy()
        out = os.path.join(args.out_dir, "%s_time_sensor_scores_%s.npy" % (prefix, name))
        np.save(out, scores)
        print("wrote %s: [%d windows of %g, %d sensors]" % (out, n_windows, args.window, N))
        return
    ranking = sensor_ranking(total / n, names)
    out = os.path.join(args.out_dir, "%s_density_scores_%s.npy" % (prefix, name))
    np.save(out, ranking)
    print("wrote %s: %d sensors, top 5 %s" % (out, N, ranking[:5].tolist()))


if __name__ == "__main__":
    main()
