#!/usr/bin/env python
"""KNN-Shapley data valuation of a Raindrop_v2 training split (raindrop_b200.valuation.knn_shapley):

    python tools/data_valuation.py --checkpoint model.pt --data P19data/processed_data/PTdict_list.npy \\
        --outcomes P19data/processed_data/arr_outcomes.npy --split splits/phy19_split1_new.npy      # against val
    python tools/data_valuation.py --checkpoint model.pt --synthetic P19 --leave-one-out
    python tools/data_valuation.py --planted-noise 0.1 --removal 0.05,0.1,0.2

With a checkpoint, the data, split and normalisation are read as tools/tracin.py reads them; the training part is valued
against the validation part (or, with --leave-one-out, every training record against the others).  Writes
KNNShapley_values_<name>.npy ([n_train] float64, in training-split order) and prints the lowest-valued records.

--planted-noise P: tools/attribution_lds.py's planted synthetic label, a share P of the training labels flipped, one model
trained on it; prints how well "lowest value first" finds the flipped labels (AUROC, precision at P n) in leave-one-out
mode and against a clean validation set, next to TracIn, EK-FAC and TRAK self-influence (largest first), and the mean
kNN utility, so a reader can see whether the features separate the classes at all.  --removal F1,F2,..: retrains without
the lowest-valued share F against a random share of the same size and prints each model's test AUROC.  An evaluation,
not a test: there is no threshold.  Prints one JSON line with the card's name and power limit.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402


def detection(scores, flipped, share):
    """(AUROC of ranking the flipped records by scores, larger first; precision among the top share n)."""
    from raindrop_b200.ood import _auroc
    top = np.argsort(-scores, kind="stable")[:max(1, int(round(share * len(scores))))]
    return _auroc(scores[flipped], scores[~flipped]), float(flipped[top].mean())


def test_auroc(model, te):
    from raindrop_b200.ood import _auroc
    with torch.no_grad():
        z, _, _ = model.forward(te["src"], te["static"], te["times"], te["lengths"])
    p = torch.softmax(z.double(), 1)[:, 1].cpu().numpy()
    y = te["y"].cpu().numpy().astype(bool)
    return _auroc(p[y], p[~y])


def planted(a):
    from attribution_lds import card, planted_data, train_model
    from raindrop_b200 import influence as IF
    from raindrop_b200 import valuation as VA
    from raindrop_b200.data import DeviceDataset
    from raindrop_b200.synth import model_config
    cfg = model_config(a.shape, dropout=0.2)
    tr = planted_data(cfg, a.n_train, a.seed, a.planted_noise)
    clean = planted_data(cfg, a.n_train, a.seed, 0.0)
    flipped = (tr["y"] != clean["y"]).numpy()
    va = {k: (v.cuda() if v is not None else None) for k, v in planted_data(cfg, a.n_val, a.seed + 1000, 0.0).items()}
    te = {k: (v.cuda() if v is not None else None) for k, v in planted_data(cfg, a.n_val, a.seed + 2000, 0.0).items()}
    ds = DeviceDataset(tr["src"], tr["static"], tr["times"], tr["y"])
    train = {k: (v.cuda() if v is not None else None) for k, v in tr.items()}
    model = train_model(cfg, ds, torch.arange(a.n_train), 1000, a.epochs, a.batch_size, a.lr, a.seed)
    out = dict(card=card(), shape=a.shape, n_train=a.n_train, n_val=a.n_val, planted_noise=a.planted_noise, k=a.k,
               flipped=int(flipped.sum()), model_test_auroc=test_auroc(model, te))
    loo = VA.knn_shapley(model, train, k=a.k, layer=a.layer)
    val = VA.knn_shapley(model, train, va, k=a.k, layer=a.layer)
    out["knn_utility_loo"] = loo.utility.mean().item()
    out["knn_utility_val"] = val.utility.mean().item()
    scores = {"knn_shapley_loo": -loo.values.cpu().numpy(), "knn_shapley_val": -val.values.cpu().numpy(),
              "tracin_self": IF.self_influence(model, train).cpu().numpy(),
              "ekfac_self": IF.ekfac_self_influence(model, train, IF.ekfac_factors(model, train)).cpu().numpy()}
    feats = IF.trak_features(model, train, dim=a.projection, seed=a.seed)
    scores["trak_self"] = np.asarray(torch.as_tensor(IF.trak_self_influence(feats)).cpu())
    out["detection"] = {k: dict(zip(("auroc", "precision_at_p"), detection(np.asarray(v, dtype=np.float64), flipped,
                                                                            a.planted_noise))) for k, v in scores.items()}
    if a.removal:
        rng = np.random.default_rng(a.seed)
        order = np.argsort(val.values.cpu().numpy(), kind="stable")
        out["removal"] = {}
        for f in (float(x) for x in a.removal.split(",")):
            m = int(round(f * a.n_train))
            keep_low = np.sort(order[m:])
            keep_rnd = np.sort(rng.permutation(a.n_train)[m:])
            res = {}
            for what, keep in (("lowest_removed", keep_low), ("random_removed", keep_rnd)):
                mdl = train_model(cfg, ds, torch.from_numpy(keep), 1000, a.epochs, a.batch_size, a.lr, a.seed)
                res[what] = test_auroc(mdl, te)
            out["removal"]["%g" % f] = res
    print(json.dumps(out), flush=True)


def checkpoint(a):
    from attribution_lds import card
    from ig_sensor_ranking import model_from_state_dict
    from raindrop_b200 import data as RD
    from raindrop_b200 import valuation as VA
    from raindrop_b200.synth import make_batch, model_config
    device = torch.device("cuda", torch.cuda.current_device())
    model = model_from_state_dict(torch.load(a.checkpoint, map_location="cpu"), a.nhead, a.seed, device).eval()
    N, T = model.d_inp, model.max_len
    if a.synthetic:
        cfg = model_config(a.synthetic)
        if cfg["d_inp"] != N or cfg["max_len"] != T or cfg["static"] != model.static:
            raise SystemExit("--synthetic %s does not match the checkpoint (d_inp %d, max_len %d)" % (a.synthetic, N, T))
        tr = make_batch(cfg, a.n_train, seed=a.seed, device=device)
        va = make_batch(cfg, a.n_val, seed=a.seed + 1, device=device)
        train = RD.DeviceDataset(tr["src"], tr["static"], tr["times"], tr["y"], device=device)
        val = RD.DeviceDataset(va["src"], va["static"], va["times"], va["y"], device=device)
        name = a.name or a.synthetic
    else:
        if not (a.outcomes and a.split):
            raise SystemExit("--data needs --outcomes and --split")
        raw = np.load(a.data, allow_pickle=True)
        is_list = raw.dtype == object and isinstance(raw.flat[0], dict)
        P_raw, minutes, static = RD.load_ptdict_list(a.data) if is_list else RD.load_array_dataset(a.data)
        n = len(P_raw)
        idx_train, idx_val = RD.load_split(a.split)[:2]
        labels = np.asarray(np.load(a.outcomes, allow_pickle=True)).reshape(n, -1)[:, a.label_col].astype(np.int64)
        mf, stdf = RD.feature_stats(torch.as_tensor(P_raw[idx_train]).to(device))

        def part(idx):
            st = None if (static is None or not model.static) else static[idx]
            return RD.DeviceDataset(*RD.tensorize_normalize(P_raw[idx], minutes[idx], st, labels[idx], mf, stdf,
                                                            device=device), device=device)
        train, val = part(idx_train), part(idx_val)
        name = a.name or "dataset"
    res = VA.knn_shapley(model, train, None if a.leave_one_out else val, k=a.k, layer=a.layer)
    v = res.values.cpu().numpy()
    path = os.path.join(a.out_dir, "KNNShapley_values_%s.npy" % name)
    np.save(path, v)
    low = np.argsort(v, kind="stable")[:a.top_k]
    print("lowest-valued training records (split position: value):")
    for i in low:
        print("  %6d: %+.6e" % (i, v[i]))
    print(json.dumps(dict(card=card(), name=name, n_train=int(v.size), leave_one_out=res.leave_one_out, k=a.k,
                          layer=a.layer, mean_knn_utility=res.utility.mean().item(), values=path)), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--checkpoint", help="state dict (torch.save) of the model whose features are used")
    ap.add_argument("--nhead", type=int, default=2)
    ap.add_argument("--data", help="PTdict_list.npy (P12 / P19 / eICU: list of dicts; PAM: plain array)")
    ap.add_argument("--synthetic", help="synthetic records of a raindrop_b200.synth configuration")
    ap.add_argument("--outcomes", help="arr_outcomes.npy: labels in column --label-col")
    ap.add_argument("--label-col", type=int, default=-1)
    ap.add_argument("--split", help="split file (idx_train, idx_val, idx_test)")
    ap.add_argument("--leave-one-out", action="store_true", help="value every training record against the others")
    ap.add_argument("--planted-noise", type=float, help="evaluate on planted synthetic data with this share flipped")
    ap.add_argument("--removal", help="--planted-noise: shares to remove and retrain without, e.g. 0.05,0.1,0.2")
    ap.add_argument("--shape", default="P19", help="--planted-noise: the synthetic configuration (2 classes)")
    ap.add_argument("--n-train", type=int, default=2000)
    ap.add_argument("--n-val", type=int, default=500)
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--lr", type=float, default=1e-3)
    ap.add_argument("--projection", type=int, default=4096, help="--planted-noise: TRAK's projection dims")
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--layer", default="hidden", choices=["hidden", "pooled"])
    ap.add_argument("--top-k", type=int, default=20)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--name")
    ap.add_argument("--out-dir", default=".")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("data_valuation runs on a CUDA device")
    if a.planted_noise is not None:
        if not 0.0 < a.planted_noise < 1.0:
            raise SystemExit("--planted-noise must lie in (0, 1)")
        planted(a)
    elif a.checkpoint and (a.data or a.synthetic):
        checkpoint(a)
    else:
        raise SystemExit("give --checkpoint with --data or --synthetic, or --planted-noise")


if __name__ == "__main__":
    main()
