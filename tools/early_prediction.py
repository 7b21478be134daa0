#!/usr/bin/env python
"""How early would a trained Raindrop_v2 have known?  AUROC / AUPRC as a function of the hours observed, and the share
of positives alarmed by each horizon (raindrop_b200.early):

    python tools/early_prediction.py --checkpoint model.pt --data P19data/processed_data/PTdict_list.npy \\
        --outcomes P19data/processed_data/arr_outcomes.npy --split P19data/splits/phy19_split1_new.npy --part test \\
        --horizons 6 12 24 48 --specificity 0.9
    python tools/early_prediction.py --synthetic P19 --n-samples 512 --horizons 2 5 10 20

The data arguments are those of tools/adv_robustness.py; without --checkpoint the model has the synthetic weights of
raindrop_b200.synth (a smoke run, not a trained model).  --horizons are in the units of times: hours for data read by
raindrop_b200.data (the files store minutes).  The full record (horizon +inf) is always added last.  Positives are the
samples of class --cls.  The alarm threshold is fixed on the full records of the negatives: the --specificity quantile
of their probability of --cls, so that about that share of them never alarm on the whole record; a positive counts as
alarmed by horizon h when some prefix up to h reaches the threshold.  Prints one row per horizon, then one JSON line.
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
    ap.add_argument("--seed", type=int, default=0, help="torch.manual_seed before building the model (R_u); data seed")
    src = ap.add_mutually_exclusive_group(required=True)
    src.add_argument("--data", help="PTdict_list.npy (P12 / P19 / eICU: list of dicts; PAM: plain array)")
    src.add_argument("--synthetic", help="synthetic batches of a raindrop_b200.synth configuration (P12, P19, PAM, ...)")
    ap.add_argument("--outcomes", help="arr_outcomes.npy: labels in column --label-col")
    ap.add_argument("--label-col", type=int, default=-1)
    ap.add_argument("--split", help="split file (idx_train, idx_val, idx_test); without it every sample is used")
    ap.add_argument("--part", default="test", choices=["train", "val", "test"])
    ap.add_argument("--n-samples", type=int, default=512, help="--synthetic: number of samples")
    ap.add_argument("--batch-size", type=int, default=512)
    ap.add_argument("--horizons", type=float, nargs="+", default=[6.0, 12.0, 24.0, 48.0])
    ap.add_argument("--cls", type=int, default=1, help="the positive class")
    ap.add_argument("--specificity", type=float, default=0.9, help="share of full-record negatives below the threshold")
    args = ap.parse_args()

    from raindrop_b200.early import PrefixResult, first_alarm, horizon_metrics, prefix_predict
    if not 0.0 < args.specificity < 1.0:
        raise SystemExit("--specificity must lie in (0, 1)")
    if not torch.cuda.is_available():
        raise SystemExit("early_prediction runs on a CUDA device")
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
    horizons = sorted(args.horizons) + [float("inf")]
    n = P.shape[1]
    parts = []
    t0 = time.perf_counter()
    for s in range(0, n, args.batch_size):
        e = min(n, s + args.batch_size)
        times = Ptime[:, s:e]
        r = prefix_predict(model, P[:, s:e], None if Pstatic is None else Pstatic[s:e], times,
                           torch.sum(times > 0, dim=0), horizons=horizons)
        parts.append(PrefixResult(r.logits.cpu(), r.cutoffs.cpu(), r.lengths.cpu()))
    torch.cuda.synchronize()
    elapsed = time.perf_counter() - t0
    res = PrefixResult(*(torch.cat([getattr(p, f) for p in parts]) for f in ("logits", "cutoffs", "lengths")))
    y = labels.cpu().numpy()
    m = horizon_metrics(res, y, cls=args.cls)
    prob = torch.softmax(res.logits.double(), dim=2)[:, :, args.cls].numpy()
    pos = y == args.cls
    threshold = float(np.quantile(prob[~pos, -1], args.specificity, method="higher"))
    alarm = first_alarm(res, threshold, cls=args.cls)
    alarmed = [float(np.mean((alarm[pos] >= 0) & (alarm[pos] <= k))) for k in range(len(horizons))]
    mean_len = res.lengths.double().mean(0).tolist()
    print("%d samples (%d of class %d), %d horizons in %.2f s; threshold %.4f at specificity %g on full records"
          % (n, int(pos.sum()), args.cls, len(horizons), elapsed, threshold, args.specificity))
    print("%10s %12s %8s %8s %10s" % ("horizon", "mean length", "AUROC", "AUPRC", "alarmed"))
    for k, h in enumerate(horizons):
        print("%10g %12.2f %8.4f %8.4f %10.4f" % (h, mean_len[k], m["auroc"][k], m["auprc"][k], alarmed[k]))
    print(json.dumps(dict(samples=n, positives=int(pos.sum()), cls=args.cls, seconds=elapsed,
                          horizons=[h if np.isfinite(h) else "inf" for h in horizons], mean_length=mean_len,
                          auroc=m["auroc"].tolist(), auprc=m["auprc"].tolist(), specificity=args.specificity,
                          threshold=threshold, alarmed=alarmed)))


if __name__ == "__main__":
    main()
