#!/usr/bin/env python
"""Throughput of input gradients (the attribution workload: saliency maps, integrated gradients).

    python tools/bench_input_grad.py [--config P19] [--steps 30] [--warmup 5] [--ig-steps M]

One call = eval-mode models_rd.Raindrop_v2.forward with frozen parameters (requires_grad_(False)) on the configuration's
per-GPU batch, then torch.autograd.grad(logits[:, 0].sum(), [src, static, times]).  Timing follows bench.py: an L2 flush
before every call outside the CUDA-event pair, median over calls.  Prints one JSON line with samples/s, ms per call, this
library's kernel launches per call (rd_launch_count; torch's own ops are not counted) and the card's name and power limit.

--ig-steps M [--ig-rows R] compares two ways of computing M-step integrated gradients (Gauss-Legendre nodes, zero
baselines, target = the labels) of the same batch instead: one raindrop_b200.attribution.integrated_gradients call
(internal_batch_size R), and the hand-written Python loop of M input-gradient calls on interpolated copies of the batch
with host-side summing.  The two are timed in
the same session, alternating call by call; samples/s counts the B samples of one call.

--ablation or --shapley-samples M [--coalition-rows R] compare, the same way, one raindrop_b200.attribution
feature_ablation / shapley_value_sampling call (one player per sensor plus the static vector, zero baselines, target =
the labels, internal_batch_size R) with the hand-written loop of B-row module forwards over the same coalitions
(P + 1 forwards for ablation; m*(P-1) + 2 for M permutations) summing F in fp64 tensors.  With --window W the players
are (sensor, time window) cells instead: feature_mask = time_window_mask(times, W, sensor_groups=d_inp) (W in the units
of `times`; padding rows belong to no player), and the loop removes the same cells.

--kernel-shap-samples M compares, the same way, one kernel_shap call over M sampled coalitions (seed 0; the same
players, --window included) with the loop of M + 2 B-row module forwards over the same coalitions followed by the same
fp64 solve (the operator [K | k] is computed once, outside the timing, for both).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import BENCH_CONFIGS, L2_FLUSH_BYTES, build_model, summarize, timed_steps  # noqa: E402
from raindrop_b200.synth import make_batch, model_config  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return "nvidia-smi unavailable (%r)" % (exc,)


def launches_of(lib, fn):
    torch.cuda.synchronize()
    n0 = lib.rd_launch_count()
    fn()
    torch.cuda.synchronize()
    return int(lib.rd_launch_count() - n0)


def ig_compare(args, lib, cfg_name, model, b, device):
    """Alternating timing of one integrated_gradients call and of the loop of M input-gradient calls."""
    from raindrop_b200.attribution import _default_steps_per_chunk, integrated_gradients, quadrature
    M = args.ig_steps
    B = b["src"].shape[1]
    N = b["src"].shape[2] // 2
    a32, w32 = (torch.tensor(v, dtype=torch.float32) for v in quadrature(M, "gausslegendre"))
    nodes = list(zip(a32.tolist(), w32.tolist()))
    src, static, times, lengths, y = b["src"], b["static"], b["times"], b["lengths"], b["y"]

    def batched():
        integrated_gradients(model, src, static, times, lengths, target=y, n_steps=M, internal_batch_size=args.ig_rows)

    def loop():
        acc_src = torch.zeros_like(src)
        acc_st = torch.zeros_like(static) if static is not None else None
        for a, w in nodes:
            xs = src.clone()
            xs[:, :, :N] *= a
            xs.requires_grad_(True)
            leaves = [xs]
            if static is not None:
                leaves.append((static * a).requires_grad_(True))
            logits, _, _ = model.forward(xs, leaves[1] if static is not None else None, times, lengths)
            g = torch.autograd.grad(logits.gather(1, y[:, None]).sum(), leaves)
            acc_src.add_(g[0], alpha=w)
            if static is not None:
                acc_st.add_(g[1], alpha=w)
        return src * acc_src, (static * acc_st if static is not None else None)

    for _ in range(max(1, args.warmup)):
        batched()
        loop()
    n_batched, n_loop = launches_of(lib, batched), launches_of(lib, loop)
    flush = torch.empty(L2_FLUSH_BYTES // 4, dtype=torch.float32, device=device)
    t_b, t_l = [], []
    for _ in range(args.steps):           # alternate: one timed call of each per round
        t_b += timed_steps(batched, 1, flush)
        t_l += timed_steps(loop, 1, flush)
    sb, sl = summarize(t_b, 1, device), summarize(t_l, 1, device)
    steps_per_chunk = min(M, max(1, args.ig_rows // B)) if args.ig_rows else \
        _default_steps_per_chunk(lib, model._plan.dims(B, False), M)
    res = {"metric": "integrated gradients, %d steps, samples/s (%s-shape synthetic)" % (M, cfg_name), "batch": B,
           "ig_steps": M, "ig_rows": args.ig_rows, "steps_per_chunk": steps_per_chunk, "steps": args.steps, "card": card()}
    for tag, t, n in (("batched", sb, n_batched), ("loop", sl, n_loop)):
        res[tag] = {"samples_per_s": round(B / (t["median"] * 1e-3), 1), "ms_per_call": round(t["median"], 4),
                    "ms_p90": round(t["p90"], 4), "launches_per_call": n}
    res["speedup_batched_over_loop"] = round(sl["median"] / sb["median"], 3)
    print(json.dumps(res), flush=True)


def coalition_compare(args, lib, cfg_name, model, b, device):
    """Alternating timing of one feature_ablation / shapley_value_sampling call and of the loop of module forwards."""
    from raindrop_b200.attribution import (_default_coalitions_per_chunk, feature_ablation, kernel_shap,
                                           kernel_shap_operator, sample_coalitions, sample_permutations,
                                           shapley_value_sampling, time_window_mask)
    src, static, times, lengths, y = b["src"], b["static"], b["times"], b["lengths"], b["y"]
    B, N = src.shape[1], src.shape[2] // 2
    mask, G = None, N
    if args.window:
        mask, n_win = time_window_mask(times, args.window, sensor_groups=N)
        G = n_win * N
        cell_player = mask.long()                              # id -1 indexes the appended "kept" entry below
    P = G + (1 if static is not None else 0)
    M = args.shapley_samples
    K = args.kernel_shap_samples
    orders = sample_permutations(P, M, 0).tolist() if M else None
    n_coal = M * (P - 1) if M else P
    if K:
        Z, w = sample_coalitions(P, K, 0)
        n_coal = Z.shape[0]
        op = torch.tensor(kernel_shap_operator(Z, w), dtype=torch.float64, device=device)
        keeps = torch.tensor(Z, dtype=torch.bool, device=device)
        zw = torch.tensor(Z * w[:, None], dtype=torch.float64, device=device)

    def batched():
        if K:
            kernel_shap(model, src, static, times, lengths, target=y, n_samples=K, seed=0,
                        internal_batch_size=args.coalition_rows, feature_mask=mask)
        elif M:
            shapley_value_sampling(model, src, static, times, lengths, target=y, n_samples=M, seed=0,
                                   internal_batch_size=args.coalition_rows, feature_mask=mask)
        else:
            feature_ablation(model, src, static, times, lengths, target=y, internal_batch_size=args.coalition_rows,
                             feature_mask=mask)

    kept = torch.ones(1, dtype=torch.bool, device=device)

    def F(keep):                  # keep: [P] bool device tensor; players = sensors or cells, then the static vector
        x = src.clone()
        k = keep[:N] if mask is None else torch.cat([keep[:G], kept])[cell_player]
        x[:, :, :N] = torch.where(k, src[:, :, :N], 0.0)
        st = None if static is None else torch.where(keep[G], static, 0.0)
        logits, _, _ = model.forward(x, st, times, lengths)
        return logits.gather(1, y[:, None])[:, 0].double()

    ones = torch.ones(P, dtype=torch.bool, device=device)

    def loop():
        fx = F(ones)
        attr = torch.zeros(B, P, dtype=torch.float64, device=device)
        if K:
            fx0 = F(~ones)
            v = torch.stack([F(k) for k in keeps])                              # [M, B]
            r = zw.T @ (v - fx0[None, :])                                        # [P, B]
            return (op[:, :P] @ r + op[:, P:] * (fx - fx0)[None, :]).T
        if not M:
            for g in range(P):
                keep = ones.clone()
                keep[g] = False
                attr[:, g] = fx - F(keep)
            return attr
        fx0 = F(~ones)
        for p in orders:
            keep = ~ones
            prev = fx0
            for k, g in enumerate(p):
                keep = keep.clone()
                keep[g] = True
                cur = fx if k == P - 1 else F(keep)
                attr[:, g] += cur - prev
                prev = cur
        return attr / M

    for _ in range(max(1, args.warmup)):
        batched()
        loop()
    n_batched, n_loop = launches_of(lib, batched), launches_of(lib, loop)
    flush = torch.empty(L2_FLUSH_BYTES // 4, dtype=torch.float32, device=device)
    t_b, t_l = [], []
    for _ in range(args.steps):           # alternate: one timed call of each per round
        t_b += timed_steps(batched, 1, flush)
        t_l += timed_steps(loop, 1, flush)
    sb, sl = summarize(t_b, 1, device), summarize(t_l, 1, device)
    cc = min(n_coal, max(1, args.coalition_rows // B)) if args.coalition_rows else \
        _default_coalitions_per_chunk(lib, model._plan.dims(B, False), P, n_coal)
    what = "Shapley-value sampling, %d permutations" % M if M else "leave-one-out ablation"
    if K:
        what = "KernelSHAP, %d coalitions" % n_coal
    if args.window:
        what += " over (sensor, %g-unit time window) players" % args.window
    res = {"metric": "%s, %d players, samples/s (%s-shape synthetic)" % (what, P, cfg_name), "batch": B,
           "players": P, "window": args.window, "shapley_samples": M, "kernel_shap_samples": K, "coalitions": n_coal, "coalition_rows": args.coalition_rows,
           "coalitions_per_chunk": cc, "steps": args.steps, "card": card()}
    for tag, t, n in (("batched", sb, n_batched), ("loop", sl, n_loop)):
        res[tag] = {"samples_per_s": round(B / (t["median"] * 1e-3), 1), "ms_per_call": round(t["median"], 4),
                    "ms_p90": round(t["p90"], 4), "launches_per_call": n}
    res["speedup_batched_over_loop"] = round(sl["median"] / sb["median"], 3)
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="P19", choices=sorted(BENCH_CONFIGS))
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ig-steps", type=int, default=0, help="compare M-step integrated gradients, batched vs loop")
    ap.add_argument("--ig-rows", type=int, default=None,
                    help="internal_batch_size of the batched call ((sample, step) rows per chunk; default: 1 GiB scratch)")
    ap.add_argument("--ablation", action="store_true", help="compare leave-one-out sensor ablation, batched vs loop")
    ap.add_argument("--shapley-samples", type=int, default=0,
                    help="compare M-permutation sensor Shapley-value sampling, batched vs loop")
    ap.add_argument("--kernel-shap-samples", type=int, default=0,
                    help="compare KernelSHAP over M sampled coalitions, batched vs loop")
    ap.add_argument("--coalition-rows", type=int, default=None,
                    help="internal_batch_size of the batched ablation / Shapley call ((sample, coalition) rows per "
                         "chunk; default: 1 GiB scratch)")
    ap.add_argument("--window", type=float, default=0.0,
                    help="with --ablation / --shapley-samples / --kernel-shap-samples: (sensor, time window) players, "
                         "windows of W units of times")
    args = ap.parse_args()
    coalitions = args.ablation or args.shapley_samples > 0 or args.kernel_shap_samples > 0
    if args.window and not coalitions:
        ap.error("--window needs --ablation, --shapley-samples or --kernel-shap-samples")
    from raindrop_b200 import lib as L
    lib = L.load()
    device = torch.device("cuda", 0)
    cfg_name, batch, _, opts, _ = BENCH_CONFIGS[args.config]
    cfg = model_config(cfg_name, dropout=0.2)
    model = build_model(cfg, device).eval().requires_grad_(False)
    b = {k: (v.to(device) if v is not None else None) for k, v in make_batch(cfg, batch, seed=2000, **opts).items()}
    if args.ig_steps > 0:
        ig_compare(args, lib, cfg_name, model, b, device)
        return
    if coalitions:
        coalition_compare(args, lib, cfg_name, model, b, device)
        return
    src = b["src"].clone().requires_grad_(True)
    times = b["times"].clone().requires_grad_(True)
    static = b["static"].clone().requires_grad_(True) if b["static"] is not None else None
    inputs = [t for t in (src, static, times) if t is not None]

    def call():
        logits, _, _ = model.forward(src, static, times, b["lengths"])
        torch.autograd.grad(logits[:, 0].sum(), inputs)

    for _ in range(max(1, args.warmup)):
        call()
    torch.cuda.synchronize()
    n0 = lib.rd_launch_count()
    call()
    launches = int(lib.rd_launch_count() - n0)
    flush = torch.empty(L2_FLUSH_BYTES // 4, dtype=torch.float32, device=device)
    t = summarize(timed_steps(call, args.steps, flush), 1, device)
    print(json.dumps({"metric": "input gradients, samples/s (%s-shape synthetic)" % cfg_name,
                      "value": round(batch / (t["median"] * 1e-3), 1), "unit": "samples/s", "batch": batch,
                      "ms_per_call": round(t["median"], 4), "ms_p90": round(t["p90"], 4), "launches_per_call": launches,
                      "steps": args.steps, "card": card()}), flush=True)


if __name__ == "__main__":
    main()
