#!/usr/bin/env python
"""Monte Carlo dropout: one raindrop_b200.uncertainty.mc_dropout call against the loop a user writes without it.

    python tools/bench_mc_dropout.py [--config P19] [--samples 32] [--batch B] [--steps 20] [--warmup 3] [--rows R]

batched: one mc_dropout call (n_samples M, internal_batch_size R, default: the largest chunk whose scratch fits in
1 GiB) returning the per-sample statistics on the device.
loop:    M training-mode module forwards under no_grad (model.train(); each forward advances the model's dropout
         counter, as it does for a user), the logits stacked and copied to the host, and mc_dropout_from_logits there.
The two are timed in the same session, alternating call by call, with an L2 flush before every call outside the
CUDA-event pair; medians over --steps calls (bench.py's protocol, as tools/bench_input_grad.py).  Prints one JSON line
with ms per call, samples/s, this library's kernel launches per call and the card's name, power limit and SM clock read
in the same run.
"""
import argparse
import ctypes as C
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
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return "nvidia-smi unavailable (%r)" % (exc,)


def launches_of(lib, fn):
    torch.cuda.synchronize()
    n0 = lib.rd_launch_count()
    fn()
    torch.cuda.synchronize()
    return int(lib.rd_launch_count() - n0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="P19", choices=sorted(BENCH_CONFIGS))
    ap.add_argument("--samples", type=int, default=32, help="Monte Carlo replicates M")
    ap.add_argument("--batch", type=int, default=None, help="samples per call (default: the configuration's batch)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rows", type=int, default=None, help="internal_batch_size of the batched call")
    args = ap.parse_args()
    from raindrop_b200 import lib as L
    from raindrop_b200.attribution import _largest_chunk
    from raindrop_b200.uncertainty import mc_dropout, mc_dropout_from_logits
    lib = L.load()
    device = torch.device("cuda", 0)
    cfg_name, batch, _, opts, _ = BENCH_CONFIGS[args.config]
    B = args.batch or batch
    M = args.samples
    cfg = model_config(cfg_name, dropout=0.2)
    model = build_model(cfg, device).eval().requires_grad_(False)
    b = {k: (v.to(device) if v is not None else None) for k, v in make_batch(cfg, B, seed=2000, **opts).items()}
    src, static, times, lengths = b["src"], b["static"], b["times"], b["lengths"]
    plan = model._prepare(device)

    def batched():
        return mc_dropout(model, src, static, times, lengths, n_samples=M, seed=1, step=0, internal_batch_size=args.rows)

    def loop():
        model.train()
        with torch.no_grad():
            logits = torch.stack([model(src, static, times, lengths)[0] for _ in range(M)])
        model.eval()
        return mc_dropout_from_logits(logits.cpu())

    rng0 = plan.rng_state.clone()
    for _ in range(max(1, args.warmup)):
        batched()
        loop()
    n_batched, n_loop = launches_of(lib, batched), launches_of(lib, loop)
    flush = torch.empty(L2_FLUSH_BYTES // 4, dtype=torch.float32, device=device)
    t_b, t_l = [], []
    for _ in range(args.steps):           # alternate: one timed call of each per round
        t_b += timed_steps(batched, 1, flush)
        t_l += timed_steps(loop, 1, flush)
    plan.rng_state.copy_(rng0)
    sb, sl = summarize(t_b, 1, device), summarize(t_l, 1, device)
    dims = plan.dims(B, True)
    cc = min(M, max(1, args.rows // B)) if args.rows else \
        _largest_chunk(lambda c: lib.rd_mc_dropout_scratch_bytes(C.byref(dims), c), M)
    res = {"metric": "Monte Carlo dropout, %d replicates, samples/s (%s-shape synthetic)" % (M, cfg_name), "batch": B,
           "samples": M, "rows": args.rows, "replicates_per_chunk": cc, "steps": args.steps, "card": card()}
    for tag, t, n in (("batched", sb, n_batched), ("loop", sl, n_loop)):
        res[tag] = {"samples_per_s": round(B / (t["median"] * 1e-3), 1), "ms_per_call": round(t["median"], 4),
                    "ms_p90": round(t["p90"], 4), "launches_per_call": n}
    res["speedup_batched_over_loop"] = round(sl["median"] / sb["median"], 3)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
