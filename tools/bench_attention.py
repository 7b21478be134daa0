#!/usr/bin/env python
"""The training step's tensor-core attention kernels on their own, at the step's shape.

    python tools/bench_attention.py [--config P19] [--batch 128] [--reps 50] [--stamps]

Runs rd_temporal_attention_fwd and rd_temporal_attention_bwd with impl 1 (attn_tc_fwd_kernel<false>,
attn_tc_bwd_kernel) at B = 128, H = 2, T = 60, hd = 76 for P19, attention dropout 0.2, on random Q, K, V, dO and the
key lengths of the synthetic P19 batch (synth.make_batch, uniform on [2, T]).  Every call is preceded by an L2 flush
(256 MiB write) outside the CUDA-event pair.  Reported, medians over --reps calls:
  call     CUDA events around the library call (one launch each);
  kernel   the kernel's device time from torch.profiler, in a separate run.
floor = 3 x (MACs of the products) at 1,024 TF32 MAC per clock per SM on all SMs at the card's maximum SM clock: the
forward has 2 products of T x T x hd per (sample, head), the backward 5.  Prints a table and one JSON line, with the
card's name, power limit and clocks read in the same run.

--stamps adds each kernel's per-CTA phase table (rd_debug_attention_timing, clock64 of warp 0's thread 0, converted at
the card's maximum SM clock) from 5 more calls, each after an L2 flush: the busiest CTA (longest start-to-end) of the
call whose busiest CTA is the median, and the mean over CTAs.  A build that stamps fewer points shows them as '-'.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from raindrop_b200 import lib as L  # noqa: E402
from raindrop_b200.synth import make_batch, model_config  # noqa: E402

L2_FLUSH_BYTES = 256 << 20
MAC_PER_CLK_SM = 1024
RNG = (0x5EED1234, 11)
# (label, slot) in stamp order; slot 0 is the start (after the grid-dependency wait), 12 the end
PHASES = {
    "fwd": [("staging landed", 1), ("S = Q K^T", 2), ("probabilities written", 3), ("O = P V", 4), ("stored", 12)],
    "bwd": [("staging landed", 1), ("S + dP", 2), ("dS / Pd written", 3), ("dV", 4), ("dQ", 5), ("dK, stored", 12)],
}
KERNELS = {"fwd": "attn_tc_fwd_kernel", "bwd": "attn_tc_bwd_kernel"}


def card():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
    return r.stdout.strip()


def stamp_table(lib, call, flush, nctas, max_mhz, phases, dev, reps=5):
    """per-phase us (busiest CTA and mean over CTAs) from the call whose busiest CTA is the median of `reps`"""
    buf = torch.zeros(nctas, 16, dtype=torch.int64, device=dev)
    runs = []
    for _ in range(reps):
        buf.zero_()
        flush.zero_()
        lib.rd_debug_attention_timing(C.c_void_p(buf.data_ptr()))
        try:
            call()
            torch.cuda.synchronize()
        finally:
            lib.rd_debug_attention_timing(None)
        s = buf.cpu().double()
        total = (s[:, 12] - s[:, 0]) / max_mhz
        busiest = int(torch.argmax(total))
        rows, prev = [], s[:, 0]
        for name, slot in phases:
            if bool((s[:, slot] > 0).all()):
                d = (s[:, slot] - prev) / max_mhz
                rows.append((name, float(d[busiest]), float(d.mean())))
                prev = s[:, slot]
            else:
                rows.append((name, None, None))
        rows.append(("total", float(total[busiest]), float(total.mean())))
        runs.append(rows)
    runs.sort(key=lambda r: r[-1][1])
    return runs[len(runs) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="P19")
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--dropout", type=float, default=0.2)
    ap.add_argument("--stamps", action="store_true", help="also print the per-CTA phase tables")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_attention.py needs a GPU")
    lib = L.load()
    dev = torch.device("cuda")
    info = card()
    max_mhz = float(info.split(",")[-1])
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    cfg = model_config(args.config, dropout=args.dropout)
    B, H, T = args.batch, cfg["nhead"], cfg["max_len"]
    D = cfg["d_model"] + 16
    hd = D // H
    p = args.dropout
    g = torch.Generator(device="cpu").manual_seed(0)
    qkv = torch.randn(T, B, 3 * D, generator=g).to(dev)
    dctx = torch.randn(T, B, D, generator=g).to(dev)
    lengths = make_batch(cfg, B, seed=1)["lengths"].to(dev)
    rng = torch.tensor(RNG, dtype=torch.int64, device=dev)
    ctx = torch.empty(T, B, D, device=dev)
    dqkv = torch.empty(T, B, 3 * D, device=dev)
    flush = torch.empty(L2_FLUSH_BYTES // 4, dtype=torch.float32, device=dev)
    st = L.stream_ptr(dev)

    calls = {
        "fwd": lambda: L.check(lib.rd_temporal_attention_fwd(qkv.data_ptr(), lengths.data_ptr(), B, H, T, hd, p,
                                                             rng.data_ptr(), L.SITE_ATTN, 1, ctx.data_ptr(), st), "fwd"),
        "bwd": lambda: L.check(lib.rd_temporal_attention_bwd(qkv.data_ptr(), dctx.data_ptr(), lengths.data_ptr(), B, H, T,
                                                             hd, p, rng.data_ptr(), L.SITE_ATTN, 1, dqkv.data_ptr(), st),
                               "bwd"),
    }
    for _ in range(3):
        for c in calls.values():
            c()
    torch.cuda.synchronize()
    t_call = {k: [] for k in calls}
    for _ in range(args.reps):
        for k, c in calls.items():
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            c()
            e1.record()
            e1.synchronize()
            t_call[k].append(e0.elapsed_time(e1) * 1000.0)

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            for c in calls.values():
                flush.zero_()
                c()
        torch.cuda.synchronize()
    kern = {k: [] for k in calls}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            for k, name in KERNELS.items():
                if name in e.name:
                    kern[k].append(e.device_time if hasattr(e, "device_time") else e.cuda_time)

    peak_mac_per_us = MAC_PER_CLK_SM * sms * max_mhz
    macs = {"fwd": 2 * B * H * T * T * hd, "bwd": 5 * B * H * T * T * hd}
    nv = lengths.clamp(0, T).double()
    print("card: %s (name, power limit W, SM clock, max SM clock MHz); %d SMs" % (info, sms))
    print("config %s: B %d, H %d, T %d, hd %d, dropout %.2f; key lengths mean %.1f (min %d, max %d)" %
          (args.config, B, H, T, hd, p, float(nv.mean()), int(nv.min()), int(nv.max())))
    out = {"card": info, "sms": sms, "config": args.config, "B": B, "H": H, "T": T, "hd": hd, "dropout": p}
    for k in calls:
        tc, tk = statistics.median(t_call[k]), statistics.median(kern[k]) if kern[k] else float("nan")
        floor_us = 3.0 * macs[k] / peak_mac_per_us
        print("%s: call %.1f us (range %.1f - %.1f); %s %.1f us; 3xTF32 floor %.1f us (floor fraction %.3f)" %
              (k, tc, min(t_call[k]), max(t_call[k]), KERNELS[k], tk, floor_us, floor_us / tk))
        out[k] = {"call_us": tc, "call_us_range": [min(t_call[k]), max(t_call[k])], "kernel_us": tk, "floor_us": floor_us}
    if args.stamps:
        for k, c in calls.items():
            rows = stamp_table(lib, c, flush, B * H, max_mhz, PHASES[k], dev)
            print("%s phases, us at %.0f MHz (%d CTAs)" % (KERNELS[k], max_mhz, B * H))
            print("%-26s %10s %10s" % ("phase", "busiest", "mean"))
            for name, bu, me in rows:
                print("%-26s %10s %10s" % (name, "-" if bu is None else "%.2f" % bu, "-" if me is None else "%.2f" % me))
            out[k]["stamps"] = rows
    print(json.dumps(out))


if __name__ == "__main__":
    main()
