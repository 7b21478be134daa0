#!/usr/bin/env python
"""Laplace approximation: laplace_fit and laplace_predictive against the loop a user writes without them.

    python tools/bench_laplace.py [--config P19] [--n-train 4096] [--batches 128,3880] [--samples 100] [--steps 5]

fit:        one laplace_fit call on --n-train synthetic samples (true Fisher, delta by log Z), host clock around a
            device synchronise; median of --fit-steps calls after one warm-up call.
predictive: laplace_predictive per batch size and link (probit; mc with --samples draws), CUDA events with an L2 flush
            outside each pair, medians over --steps calls (bench.py's protocol).
loop:       the covariance of --loop-samples samples by a host loop of per-sample, per-class torch.autograd.grad through
            the drop-in module (one forward per class: its backward cannot retain the graph), the gradient rotated
            into the EK-FAC bases with torch matmuls per block and contracted with the weights; its time per sample is
            multiplied by B for the per-batch figure (marked extrapolated).
gram:       the Gram kernels (laplace_gram_kernel + laplace_fold_kernel) of one covariance call at the largest batch,
            from torch.profiler in a separate run; achieved bytes/s = the rows read (C * B * bucket * 4 bytes) plus the
            weights (bucket * 4 bytes) over the kernel time, against the 3.35 TB/s HBM3 figure of the H100 SXM data sheet.
Prints one JSON line, with the card's name, power limit and SM clock read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import L2_FLUSH_BYTES, build_model, summarize, timed_steps  # noqa: E402
from raindrop_b200.synth import make_batch, model_config  # noqa: E402

HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet, 700 W


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return "nvidia-smi unavailable (%r)" % (exc,)


def loop_covariance(model, la, src, static, times, lengths):
    """Sigma [B, C, C] float64 by per-sample, per-class autograd through the module and a torch rotation."""
    from raindrop_b200 import influence as IF
    f = la.factors
    layout = IF.grad_layout(model)
    ldg = IF._bucket_length(layout)
    w = torch.from_numpy(IF.ekfac_weights(f, damping=la.prior_precision / la.n) / la.n).to(src.device)
    blocks = [(w_, b_, nout, kin, torch.from_numpy(QA).to(src.device), torch.from_numpy(QS).to(src.device))
              for (w_, b_, nout, kin), (QA, QS) in zip(IF.kfac_blocks(model), f.bases)]
    off = {k: o for k, o, _ in layout}
    params = model.used_parameters()
    out = []
    for b in range(src.shape[1]):
        rows = []
        for c in range(model._plan.n_classes):      # one forward per class: the module's backward runs once per graph
            logits = model(src[:, b:b + 1], None if static is None else static[b:b + 1], times[:, b:b + 1],
                           lengths[b:b + 1])[0]
            gs = torch.autograd.grad(logits[0, c], params)
            g = torch.zeros(ldg, dtype=torch.float64, device=src.device)
            for (k, o, s), t in zip(layout, gs):
                g[o:o + t.numel()] = t.reshape(-1).double()
            for wk, bk, nout, kin, QA, QS in blocks:
                M = torch.cat([g[off[wk]:off[wk] + nout * kin].view(nout, kin), g[off[bk]:off[bk] + nout, None]], 1)
                Mt = QS.T @ M @ QA
                g[off[wk]:off[wk] + nout * kin] = Mt[:, :kin].reshape(-1)
                g[off[bk]:off[bk] + nout] = Mt[:, kin]
            rows.append(g)
        J = torch.stack(rows)
        out.append((J * w) @ J.T)
    return torch.stack(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="P19")
    ap.add_argument("--n-train", type=int, default=4096)
    ap.add_argument("--batches", default="128,3880")
    ap.add_argument("--samples", type=int, default=100)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--fit-steps", type=int, default=3)
    ap.add_argument("--loop-samples", type=int, default=16)
    args = ap.parse_args()
    from raindrop_b200 import lib as L
    from raindrop_b200.laplace import _cov_batch, _forward, laplace_fit, laplace_predictive
    from raindrop_b200 import influence as IF
    lib = L.load()
    device = torch.device("cuda", 0)
    cfg = model_config(args.config, dropout=0.2)
    model = build_model(cfg, device).eval()
    tr = {k: (v.to(device) if v is not None else None) for k, v in make_batch(cfg, args.n_train, seed=3000).items()}
    res = {"metric": "Laplace approximation (%s-shape synthetic, %d training samples)" % (args.config, args.n_train),
           "card": card()}

    laplace_fit(model, tr)
    t_fit = []
    for _ in range(args.fit_steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        la = laplace_fit(model, tr)
        torch.cuda.synchronize()
        t_fit.append(time.perf_counter() - t0)
    res["fit_s"] = round(float(np.median(t_fit)), 4)
    res["prior_precision"] = la.prior_precision
    res["log_marginal_likelihood"] = la.log_marginal_likelihood()

    flush = torch.empty(L2_FLUSH_BYTES // 4, dtype=torch.float32, device=device)
    batches = [int(x) for x in args.batches.split(",")]
    bq = {}
    for B in batches:
        b = {k: (v.to(device) if v is not None else None) for k, v in make_batch(cfg, B, seed=4000 + B).items()}
        a = (b["src"], b["static"], b["times"], b["lengths"])
        bq[B] = a
        row = {}
        for link in ("probit", "mc"):
            fn = lambda: laplace_predictive(model, la, *a, link=link, n_samples=args.samples)
            fn()
            t = summarize(timed_steps(fn, args.steps, flush), 1, device)
            row[link] = {"ms_per_call": round(t["median"], 3), "ms_p90": round(t["p90"], 3),
                         "samples_per_s": round(B / (t["median"] * 1e-3), 1)}
        res["predictive_B%d" % B] = row

    # the autograd loop on a few samples, checked against the device result
    a = bq[batches[0]]
    k = min(args.loop_samples, a[0].shape[1])
    sub = (a[0][:, :k], None if a[1] is None else a[1][:k], a[2][:, :k], a[3][:k])
    ref = loop_covariance(model, la, *sub)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ref = loop_covariance(model, la, *sub)
    torch.cuda.synchronize()
    per_sample = (time.perf_counter() - t0) / k
    got = laplace_predictive(model, la, *sub).logit_cov
    res["loop_ms_per_sample"] = round(per_sample * 1e3, 3)
    res["loop_vs_device_max_rel"] = float(((got - ref).norm(dim=(1, 2)) / ref.norm(dim=(1, 2))).max())
    for B in batches:
        res["loop_ms_B%d_extrapolated" % B] = round(per_sample * B * 1e3, 1)
        res["speedup_probit_over_loop_B%d" % B] = round(per_sample * B * 1e3 / res["predictive_B%d" % B]["probit"]["ms_per_call"], 2)

    # Gram kernel bandwidth at the largest batch's covariance chunk
    B = batches[-1]
    plan = model._plan
    Rc = min(B, _cov_batch(lib, plan))
    a = bq[B]
    with torch.no_grad():
        cl, dims, ws, _, _ = _forward(model, a[0][:, :Rc], None if a[1] is None else a[1][:Rc], a[2][:, :Rc], a[3][:Rc])
        w = torch.from_numpy(IF.ekfac_weights(la.factors, damping=la.prior_precision / la.n) / la.n).float().to(device)
        bases = la.factors.bases_flat.to(device)
        sc = torch.empty(lib.rd_laplace_logit_cov_scratch_bytes(C.byref(dims)) // 4, device=device)
        cov = torch.empty(Rc, plan.n_classes, plan.n_classes, dtype=torch.float64, device=device)
        call = lambda: L.check(lib.rd_raindrop_v2_laplace_logit_cov(C.byref(dims), C.byref(cl.params), L.ptr(cl.st),
                                                                    cl.ln.data_ptr(), plan.node_scale.data_ptr(),
                                                                    ws.data_ptr(), bases.data_ptr(), w.data_ptr(),
                                                                    sc.data_ptr(), cov.data_ptr(), L.stream_ptr(device)),
                               "rd_raindrop_v2_laplace_logit_cov")
        call()
        reps = 10
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                call()
            torch.cuda.synchronize()
    gram_us = fold_us = total_us = 0.0
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if "laplace_gram_kernel" in e.key:
            gram_us += us / reps
        elif "laplace_fold_kernel" in e.key:
            fold_us += us / reps
        total_us += us / reps
    ldg = IF._bucket_length(IF.grad_layout(model))
    nbytes = 4 * (plan.n_classes * Rc * ldg + ldg)
    res["gram"] = {"samples": Rc, "bucket": ldg, "bytes": nbytes, "gram_kernel_us": round(gram_us, 2),
                   "fold_kernel_us": round(fold_us, 2), "cov_call_kernels_us": round(total_us, 1),
                   "achieved_TB_per_s": round(nbytes / (gram_us * 1e-6) / 1e12, 3) if gram_us else None,
                   "share_of_3.35_TB_per_s": round(nbytes / (gram_us * 1e-6) / HBM_BYTES_PER_S, 3) if gram_us else None}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
