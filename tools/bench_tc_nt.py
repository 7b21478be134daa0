#!/usr/bin/env python
"""Each tc_nt_kernel shape of the P19 (B = 128) training step on its own, against its tensor-core floor.

    python tools/bench_tc_nt.py [--reps 50] [--rows 7680] [--obprop-rows 4352]

Encoder shapes (rows x N x K, error-compensated 3xTF32) run through rd_linear_fwd: in_proj 456 x 152, out_proj and
K1.Wo 152 x 152, linear1 and K2.W2 272 x 152, linear2 and gF.W1 152 x 272, dqkv.Win 152 x 456.  The ob-prop layer
(240 x 240, error-compensated at this row count) runs through rd_obprop_fwd.  Every call is preceded by an L2 flush
(256 MiB write) outside the CUDA-event pair; medians over --reps calls.  Two times per shape:
  call    CUDA events around the library call: the tc_nt launch plus the split of the weight into hi / lo that the
          call does first (one small launch);
  kernel  the tc_nt kernel alone, from its %globaltimer stamps (rd_debug_gemm_timing): latest CTA end minus earliest
          CTA start after the grid dependency wait.
floor = 3 * rows * N * K MACs at 1,024 TF32 MAC per clock per SM on all SMs at the card's maximum SM clock (the
data-sheet rate; 3xTF32 counted as three products).  Prints a table and one JSON line, with the card's name, power
limit and clocks read in the same run.
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

from raindrop_b200 import lib as L  # noqa: E402

L2_FLUSH_BYTES = 256 << 20
MAC_PER_CLK_SM = 1024


def card():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
    return r.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rows", type=int, default=7680)          # T * B at P19, B = 128
    ap.add_argument("--obprop-rows", type=int, default=4352)   # B * N at P19, B = 128
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tc_nt.py needs a GPU")
    lib = L.load()
    dev = torch.device("cuda")
    info = card()
    max_mhz = float(info.split(",")[-1])
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    peak_mac_per_us = MAC_PER_CLK_SM * sms * max_mhz
    flush = torch.empty(L2_FLUSH_BYTES // 4, dtype=torch.float32, device=dev)
    stamps = torch.zeros(sms * 8, dtype=torch.int64, device=dev)
    st = L.stream_ptr(dev)
    g = torch.Generator(device="cpu").manual_seed(0)

    def rnd(*shape, scale=1.0):
        return (scale * torch.randn(*shape, generator=g)).to(dev)

    shapes = [("in_proj", args.rows, 456, 152, 0), ("out_proj, K1.Wo", args.rows, 152, 152, 0),
              ("linear1, K2.W2", args.rows, 272, 152, 1), ("linear2, gF.W1", args.rows, 152, 272, 0),
              ("dqkv.Win", args.rows, 152, 456, 0), ("ob-prop layer", args.obprop_rows, 240, 240, -1)]
    rows_out = []
    for name, M, N, K, relu in shapes:
        x, w, b = rnd(M, K), rnd(N, K, scale=K ** -0.5), rnd(N, scale=0.1)
        out = torch.empty(M, N, dtype=torch.float32, device=dev)
        if relu >= 0:
            scratch = torch.empty(lib.rd_linear_scratch_bytes(K, N) // 4 + 64, dtype=torch.float32, device=dev)
            call = lambda: L.check(lib.rd_linear_fwd(x.data_ptr(), w.data_ptr(), b.data_ptr(), M, K, N, relu,  # noqa: E731
                                                     out.data_ptr(), scratch.data_ptr(), st), "rd_linear_fwd")
        else:
            ns = (0.5 + torch.rand(17, generator=g)).to(dev)
            scratch = torch.empty(lib.rd_obprop_fwd_scratch_bytes(M, N) // 4 + 64, dtype=torch.float32, device=dev)
            call = lambda: L.check(lib.rd_obprop_fwd(x.data_ptr(), w.data_ptr(), b.data_ptr(), ns.data_ptr(), 17,  # noqa: E731
                                                     M, N, out.data_ptr(), scratch.data_ptr(), st), "rd_obprop_fwd")
        for _ in range(3):
            call()
        t_call, t_kern = [], []
        for _ in range(args.reps):
            flush.zero_()
            stamps.zero_()
            lib.rd_debug_gemm_timing(C.c_void_p(stamps.data_ptr()))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call()
            e1.record()
            e1.synchronize()
            lib.rd_debug_gemm_timing(None)
            t_call.append(e0.elapsed_time(e1) * 1000.0)
            s = stamps.view(-1, 8).cpu()
            used = s[:, 0] > 0
            t_kern.append((s[used, 7].max() - s[used, 0].min()).item() / 1000.0)
        floor_us = 3.0 * M * N * K / peak_mac_per_us
        tc, tk = statistics.median(t_call), statistics.median(t_kern)
        rows_out.append({"shape": name, "rows": M, "N": N, "K": K, "call_us": tc, "call_us_range": [min(t_call), max(t_call)],
                         "kernel_us": tk, "floor_us": floor_us, "floor_frac_call": floor_us / tc,
                         "floor_frac_kernel": floor_us / tk})
    print("card: %s (name, power limit W, SM clock, max SM clock MHz); %d SMs" % (info, sms))
    print("%-18s %6s %4s %4s %9s %9s %8s %7s %7s" % ("shape", "rows", "N", "K", "call us", "kernel us", "floor us",
                                                     "f(call)", "f(kern)"))
    for r in rows_out:
        print("%-18s %6d %4d %4d %9.2f %9.2f %8.2f %7.3f %7.3f" % (r["shape"], r["rows"], r["N"], r["K"], r["call_us"],
                                                                r["kernel_us"], r["floor_us"], r["floor_frac_call"],
                                                                r["floor_frac_kernel"]))
    print(json.dumps({"card": info, "sms": sms, "shapes": rows_out}))


if __name__ == "__main__":
    main()
