#!/usr/bin/env python
"""Out-of-distribution detection: ood_fit and ood_scores against the torch path a user writes without them.

    python tools/bench_ood.py [--config P19] [--n-train 31000] [--batch 3880] [--k 50] [--steps 5]

fit:     one ood_fit call on --n-train synthetic samples (features, float64 moments, host eigendecomposition and the kNN
         bank), host clock around a device synchronise; median of --fit-steps calls after one warm-up call.
scores:  one ood_scores call at B = --batch against the full bank (all scores), CUDA events with an L2 flush outside
         each pair, median over --steps calls (bench.py's protocol).
torch:   the same scores from the same features with torch on the device: the eval features (ood.features, timed
         apart), then Mahalanobis as torch.mm((f - mu) W) and per-class distances, kNN as F.normalize, torch.mm against
         the bank and torch.topk, msp / energy with torch.softmax / logsumexp (fp32, TF32 off as torch's default).
Prints one JSON line, with the card's name, power limit and SM clock read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from bench import L2_FLUSH_BYTES, build_model, timed_steps  # noqa: E402
from raindrop_b200.synth import make_batch, model_config  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return "nvidia-smi unavailable (%r)" % (exc,)


def torch_scores(det, f, logits, k):
    """The torch path on given features: (msp, energy, mahalanobis, knn, knn_index)."""
    W = torch.from_numpy(det.W).to(device=f.device, dtype=torch.float32)
    mu = torch.from_numpy(det.mean).to(device=f.device, dtype=torch.float32)
    M = torch.from_numpy(det.class_proj).to(device=f.device, dtype=torch.float32)
    z = torch.mm(f - mu, W)
    d = (z[:, None, :] - M[None, :, :]).pow(2).sum(2)
    maha = d.min(1).values
    q = F.normalize(f, dim=1)
    bank = det.bank[:det.n_bank, :f.shape[1]]
    s, idx = torch.topk(torch.mm(q, bank.t()), k, dim=1)
    msp = -torch.softmax(logits, 1).max(1).values
    energy = -torch.logsumexp(logits, 1)
    return msp, energy, maha, 2 - 2 * s[:, -1], idx


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--config", default="P19")
    ap.add_argument("--n-train", type=int, default=31000)
    ap.add_argument("--batch", type=int, default=3880)
    ap.add_argument("--k", type=int, default=50)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--fit-steps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ood measures the H100 path: no CUDA device")
    from raindrop_b200 import ood as OOD
    dev = torch.device("cuda", torch.cuda.current_device())
    cfg = model_config(args.config, dropout=0.2)
    model = build_model(cfg, dev).eval()
    model._plan.obprop_mode = 0
    train = make_batch(cfg, args.n_train, seed=21, device=dev)
    q = make_batch(cfg, args.batch, seed=22, device=dev)
    qa = (q["src"], q["static"], q["times"], q["lengths"])
    flush = torch.empty(L2_FLUSH_BYTES // 4, device=dev)

    fit_t = []
    for i in range(args.fit_steps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        det = OOD.ood_fit(model, train)
        torch.cuda.synchronize()
        if i:
            fit_t.append((time.perf_counter() - t0) * 1e3)

    state = {}

    def ours():
        state["res"] = OOD.ood_scores(model, det, *qa, k=args.k)

    def feats():
        state["f"] = OOD.features(model, *qa)

    def base():
        f, lg = state["f"]
        state["base"] = torch_scores(det, f, lg, args.k)

    for fn in (ours, feats, base):
        fn()
        fn()
    torch.cuda.synchronize()
    t_ours = timed_steps(ours, args.steps, flush)
    t_feat = timed_steps(feats, args.steps, flush)
    t_base = timed_steps(base, args.steps, flush)
    med = lambda v: float(np.median(v))
    res, (msp, energy, maha, knn, idx) = state["res"], state["base"]
    agree = dict(knn_max_abs=float((res.knn - knn).abs().max()),
                 mahalanobis_max_rel=float(((res.mahalanobis - maha).abs() / (maha.abs() + 1)).max()),
                 knn_index_first_equal=float((res.knn_index[:, 0] == idx[:, 0]).float().mean()))
    torch_total = med(t_feat) + med(t_base)
    print(json.dumps(dict(metric="ood", config=args.config, n_train=args.n_train, batch=args.batch, k=args.k,
                          rank=det.rank, fit_ms=med(fit_t), scores_ms=med(t_ours), features_ms=med(t_feat),
                          torch_scoring_ms=med(t_base), torch_total_ms=torch_total,
                          speedup_vs_torch=torch_total / med(t_ours), agreement=agree, card=card())))


if __name__ == "__main__":
    main()
