#!/usr/bin/env python
"""The grouped weight-gradient launch of one training step on its own, against its tensor-core floor.

    python tools/bench_wgrad.py [--config P19] [--reps 50]

Runs the step's ten weight-gradient problems (per encoder layer dW of linear2 D x nhid, linear1 nhid x D, out_proj
D x D and in_proj 3D x D at T * B rows; the two ob-prop lin_value weights C x C at B * N rows) through ONE
rd_linear_wgrad_group call, i.e. one tc_wgrad_kernel launch and one wgrad_reduce_kernel launch.  Every call is preceded
by an L2 flush (256 MiB write) outside the CUDA-event pair.  Reported, medians over --reps calls:
  call     CUDA events around the library call (both launches);
  kernels  tc_wgrad_kernel and wgrad_reduce_kernel device time from torch.profiler, in a separate run.
floor = 3 * sum(rows * Nout * (Kin + 1)) MACs (3xTF32 counted as three products, the bias column included) at 1,024 TF32
MAC per clock per SM on all SMs at the card's maximum SM clock (the data-sheet rate).  Prints a table and one JSON line,
with the card's name, power limit and clocks read in the same run.

--stamps adds the kernel's per-CTA phase breakdown (rd_debug_wgrad_timing) from 5 more calls, each after an L2 flush:
for the busiest CTA (longest start-to-end) and the mean over CTAs, in us at the CTA's own clock rate, of the call whose
busiest CTA is the median.
"""
import argparse
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
from raindrop_b200.synth import model_config  # noqa: E402

L2_FLUSH_BYTES = 256 << 20
MAC_PER_CLK_SM = 1024
BATCH = {"P12": 32, "P19": 128, "PAM": 256, "LARGE": 512}     # bench.py's per-GPU batch


def card():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
    return r.stdout.strip()


def problems(config, batch):
    """(name, rows, Nout, Kin) of the step's weight gradients, in the order the backward queues them"""
    cfg = model_config(config)
    D = cfg["d_model"] + 16
    nhid, C = cfg["nhid"], cfg["max_len"] * cfg["d_ob"]
    m2, m1 = cfg["max_len"] * batch, batch * cfg["d_inp"]
    enc = [("linear2", m2, D, nhid), ("linear1", m2, nhid, D), ("out_proj", m2, D, D), ("in_proj", m2, 3 * D, D)]
    return enc + enc + [("ob-prop lin_value", m1, C, C)] * 2


STAMP_PHASES = [("total", None), ("transposer: wait X", 3), ("transposer: transpose + store", 4),
                ("transposer: other", None), ("issuer: wait empty stage", 11), ("issuer: issue loads", 12),
                ("issuer: other", None), ("MMA: wait full stage", 5), ("MMA: epilogue", 6)]


def stamp_breakdown(lib, call, flush, sms, dev, reps=5):
    """per-phase us of the busiest and the mean CTA (rd_debug_wgrad_timing), from the median of `reps` calls"""
    import ctypes as C
    buf = torch.zeros(sms, 16, dtype=torch.int64, device=dev)
    runs = []
    for _ in range(reps):
        buf.zero_()
        flush.zero_()
        lib.rd_debug_wgrad_timing(C.c_void_p(buf.data_ptr()))
        try:
            call()
            torch.cuda.synchronize()
        finally:
            lib.rd_debug_wgrad_timing(None)
        s = buf.cpu().double()
        s = s[s[:, 7] > 0]                                   # launched CTAs
        mhz = (s[:, 1] - s[:, 0]) / s[:, 7] * 1000.0          # cycles per ns -> MHz, per CTA
        us = {name: s[:, slot] / mhz for name, slot in STAMP_PHASES if slot is not None}
        us["total"] = (s[:, 1] - s[:, 0]) / mhz
        # each producer thread's time outside its measured phases (item walk, loop), from the start to its own end
        us["transposer: other"] = (s[:, 9] - s[:, 0] - s[:, 3] - s[:, 4]) / mhz
        us["issuer: other"] = (s[:, 13] - s[:, 0] - s[:, 11] - s[:, 12]) / mhz
        us = {name: us[name] for name, _ in STAMP_PHASES}
        us["k-blocks"] = s[:, 8]
        busiest = int(torch.argmax(us["total"]))
        runs.append({"busiest": {k: float(v[busiest]) for k, v in us.items()},
                     "mean": {k: float(v.mean()) for k, v in us.items()}, "ctas": int(s.shape[0]),
                     "mhz": float(mhz.mean())})
    runs.sort(key=lambda r: r["busiest"]["total"])
    return runs[len(runs) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="P19", choices=sorted(BATCH))
    ap.add_argument("--batch", type=int, default=None)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--stamps", action="store_true", help="also print the per-CTA phase breakdown")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_wgrad.py needs a GPU")
    lib = L.load()
    dev = torch.device("cuda")
    info = card()
    max_mhz = float(info.split(",")[-1])
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    peak_mac_per_us = MAC_PER_CLK_SM * sms * max_mhz
    flush = torch.empty(L2_FLUSH_BYTES // 4, dtype=torch.float32, device=dev)
    st = L.stream_ptr(dev)
    g = torch.Generator(device="cpu").manual_seed(0)
    probs = problems(args.config, args.batch or BATCH[args.config])

    keep = []
    items = (L.RdWgradItem * len(probs))()
    for i, (_, rows, nout, kin) in enumerate(probs):
        dy, x = torch.randn(rows, nout, generator=g).to(dev), torch.randn(rows, kin, generator=g).to(dev)
        dw, db = torch.empty(nout, kin, device=dev), torch.empty(nout, device=dev)
        part = torch.empty(max(1, lib.rd_linear_wgrad_partial_bytes(rows, nout, kin) // 4), device=dev)
        keep += [dy, x, dw, db, part]
        items[i].d_out, items[i].x, items[i].rows, items[i].out_features, items[i].in_features = \
            dy.data_ptr(), x.data_ptr(), rows, nout, kin
        items[i].d_weight, items[i].d_bias, items[i].partial = dw.data_ptr(), db.data_ptr(), part.data_ptr()

    def call():
        L.check(lib.rd_linear_wgrad_group(items, len(probs), st), "rd_linear_wgrad_group")

    for _ in range(3):
        call()
    torch.cuda.synchronize()
    t_call = []
    for _ in range(args.reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()
        e1.record()
        e1.synchronize()
        t_call.append(e0.elapsed_time(e1) * 1000.0)

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            flush.zero_()
            call()
        torch.cuda.synchronize()
    kern = {"tc_wgrad_kernel": [], "wgrad_reduce_kernel": []}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            for k in kern:
                if k in e.name:
                    kern[k].append(e.device_time if hasattr(e, "device_time") else e.cuda_time)
    useful = sum(rows * nout * (kin + 1) for _, rows, nout, kin in probs)
    floor_us = 3.0 * useful / peak_mac_per_us
    tk = {k: statistics.median(v) if v else float("nan") for k, v in kern.items()}
    tc = statistics.median(t_call)

    print("card: %s (name, power limit W, SM clock, max SM clock MHz); %d SMs; config %s" % (info, sms, args.config))
    print("%-20s %7s %5s %5s" % ("problem", "rows", "Nout", "Kin"))
    for name, rows, nout, kin in probs:
        print("%-20s %7d %5d %5d" % (name, rows, nout, kin))
    print("useful 3xTF32 MACs %.3f G, floor %.1f us" % (3.0 * useful / 1e9, floor_us))
    print("call %.1f us (range %.1f - %.1f); tc_wgrad_kernel %.1f us (floor fraction %.3f); wgrad_reduce_kernel %.1f us" %
          (tc, min(t_call), max(t_call), tk["tc_wgrad_kernel"], floor_us / tk["tc_wgrad_kernel"], tk["wgrad_reduce_kernel"]))
    out = {"card": info, "sms": sms, "config": args.config, "problems": probs, "floor_us": floor_us,
           "call_us": tc, "call_us_range": [min(t_call), max(t_call)], "kernel_us": tk,
           "floor_frac_kernel": floor_us / tk["tc_wgrad_kernel"]}
    if args.stamps:
        st = stamp_breakdown(lib, call, flush, sms, dev)
        print("phase breakdown, us (%d CTAs, mean clock %.0f MHz)" % (st["ctas"], st["mhz"]))
        print("%-30s %10s %10s" % ("phase", "busiest", "mean"))
        for k in st["busiest"]:
            print("%-30s %10.1f %10.1f" % (k, st["busiest"][k], st["mean"][k]))
        out["stamps"] = st
    print(json.dumps(out))


if __name__ == "__main__":
    main()
