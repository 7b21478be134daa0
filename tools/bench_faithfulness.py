#!/usr/bin/env python
"""Times raindrop_b200.faithfulness.deletion_curves and infidelity against a torch loop that builds the removed copies
with tensor ops and runs the module's eval forward in chunks of the same row count:

    python tools/bench_faithfulness.py               # P19 B=128 sensors and window-6 players, P19 B=3880, PAM cells

Synthetic weights and batches (raindrop_b200.synth), ob-prop mode auto.  Curves at the default counts, infidelity with
--samples replicates at p_remove 0.5.  Times are CUDA-event medians over --reps calls after --warmup; the maximal
difference of the loop's curve values from the device call's is printed.  One JSON line per shape, with the card's
name and power limit read in the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from bench_valuation import card, timed  # noqa: E402
from raindrop_b200 import attribution as A  # noqa: E402
from raindrop_b200 import faithfulness as F  # noqa: E402
from raindrop_b200.models_rd import Raindrop_v2  # noqa: E402
from raindrop_b200.synth import make_batch, model_config, synth_weights  # noqa: E402

# (name, config, B, players: "sensor", window width, or "cell")
SHAPES = [("P19-B128-sensor", "P19", 128, "sensor"), ("P19-B128-window6", "P19", 128, 6.0),
          ("P19-B3880-sensor", "P19", 3880, "sensor"), ("PAM-B8-cell", "PAM", 8, "cell")]


def torch_loop(model, d, cells, keep_rows, tgt, chunk_rows):
    """F at the target of every keep row [R*B, P] (row j = r*B + b): removed copies built with tensor ops, module
    forward on chunks of chunk_rows rows."""
    src, st = d["src"], d["static"]
    T, B, N2 = src.shape
    N = N2 // 2
    P = keep_rows.shape[1]
    G = P - (1 if st is not None else 0)
    ids = torch.where((cells < 0) | (cells >= G), G, cells).expand(T, B, N)
    out = []
    per = max(1, chunk_rows // B)
    for r0 in range(0, keep_rows.shape[0] // B, per):
        k = keep_rows[r0 * B:(r0 + per) * B].bool().view(-1, B, P)
        R = k.shape[0]
        kk = torch.cat([k[:, :, :G], torch.ones(R, B, 1, dtype=torch.bool, device=src.device)], dim=2)
        kept = torch.gather(kk.unsqueeze(1).expand(R, T, B, G + 1), 3, ids.unsqueeze(0).expand(R, T, B, N))
        val = torch.where(kept, src[None, :, :, :N], 0.0)
        x = torch.cat([val, src[None, :, :, N:].expand(R, T, B, N)], 3).permute(1, 0, 2, 3).reshape(T, R * B, N2)
        s = None if st is None else torch.where(k[:, :, P - 1:], st[None], 0.0).reshape(R * B, -1)
        with torch.no_grad():
            lg = model.forward(x, s, d["times"].repeat(1, R), d["lengths"].repeat(R))[0]
        out.append(lg.view(R, B, -1).gather(2, tgt.view(1, B, 1).expand(R, B, 1))[..., 0])
    return torch.cat(out)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--samples", type=int, default=64, help="infidelity replicates")
    ap.add_argument("--shapes", default=",".join(s[0] for s in SHAPES))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_faithfulness.py measures on the GPU and needs CUDA")
    dev_card = card()
    for name, cname, B, players in SHAPES:
        if name not in a.shapes.split(","):
            continue
        cfg = model_config(cname, dropout=0.0)
        torch.manual_seed(1)
        model = Raindrop_v2(cfg["d_inp"], cfg["d_model"], cfg["nhead"], cfg["nhid"], cfg["nlayers"], 0.0,
                            cfg["max_len"], cfg["d_static"], cfg["MAX"], 0.5, "mean", cfg["n_classes"],
                            torch.ones(cfg["d_inp"], cfg["d_inp"]), **({} if cfg["static"] else {"static": False}))
        synth_weights(model, cfg, seed=3)
        model = model.cuda().eval()
        d = {k: (v.cuda() if v is not None else None) for k, v in make_batch(cfg, B, seed=2).items()}
        T, N = cfg["max_len"], cfg["d_inp"]
        if players == "sensor":
            kw, cells = {}, torch.arange(N, device="cuda").view(1, 1, N)
        elif players == "cell":
            cells = torch.arange(T * N, device="cuda").view(T, 1, N)
            kw = dict(feature_mask=cells[:, 0].cpu())
        else:
            mask, _ = A.time_window_mask(d["times"], players, sensor_groups=N)
            kw, cells = dict(feature_mask=mask.cpu()), mask.long()
        P = int(cells.max()) + 1 + (1 if cfg["static"] else 0)
        phi = torch.randn(B, P, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
        args = (model, d["src"], d["static"], d["times"], d["lengths"], phi)
        t_cur, cur = timed(lambda: F.deletion_curves(*args, **kw), a.warmup, a.reps)
        t_inf, inf = timed(lambda: F.infidelity(*args, n_samples=a.samples, **kw), a.warmup, a.reps)
        counts = torch.as_tensor(cur.counts, device="cuda").long()
        rank = cur.rank.long()
        top = rank[None] < counts.view(-1, 1, 1)                                  # [K, B, P]
        keep = torch.cat([~top, top]).to(torch.uint8).view(-1, P)
        rows = cur.deletion_logits.shape[0] * 2 * len(counts)
        chunk = min(rows, 4096)
        t_loop, vals = timed(lambda: torch_loop(model, d, cells, keep, cur.target, chunk), a.warmup, a.reps)
        ref = torch.stack([cur.deletion.T, cur.insertion.T]).reshape(-1, B)
        # the infidelity loop: the same number of removed copies (torch's own uniform draws), the fp64 moments
        g = torch.Generator(device="cuda").manual_seed(7)
        keep_i = (torch.rand(a.samples * B, P, device="cuda", generator=g) >= 0.5).to(torch.uint8)

        def inf_loop():
            fr = torch_loop(model, d, cells, keep_i, cur.target, chunk).double()
            aa = ((1 - keep_i.double()).view(-1, B, P) * phi.double()).sum(2)
            dd = cur.clean.double() - fr
            return torch.stack([aa.sum(0), dd.sum(0), (aa * aa).sum(0), (aa * dd).sum(0), (dd * dd).sum(0)], 1)
        t_inf_loop, _ = timed(inf_loop, a.warmup, a.reps)
        print(json.dumps(dict(shape=name, B=B, players=P, counts=len(counts), curves_ms=round(t_cur, 3),
                              curves_torch_loop_ms=round(t_loop, 3), infidelity_ms=round(t_inf, 3),
                              infidelity_torch_loop_ms=round(t_inf_loop, 3),
                              infidelity_samples=a.samples, curve_max_diff=float((vals - ref).abs().max()),
                              infidelity_mean=float(inf.infidelity.mean()), card=dev_card)), flush=True)


if __name__ == "__main__":
    main()
