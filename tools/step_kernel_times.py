"""Per-kernel device time of one training step on the GPU (torch.profiler, CUDA activities).

    python tools/step_kernel_times.py [--config P19] [--batch 128] [--out DIR] [--repeat 20]

Builds the bench.py model (seeded synthetic weights, dropout 0.2), warms the TrainStep up, then
  1. times --repeat CUDA-graph replays with CUDA events (profiler off) -> the step time, median;
  2. profiles one eager enqueue and one graph replay, each in a profiler session of its own, and prints per kernel:
     name, launches, total us and share of the summed kernel time, plus that sum against the event step time.
The launches of `tc_nt_kernel` are also listed one by one in step order with their grid and time, so that each GEMM
shape of the step can be followed across builds.  With --out DIR the tables are also written to DIR/step_kernel_times.json.
"""
import argparse
import collections
import json
import os
import re
import statistics
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from helpers import build_dropin, to_dev  # noqa: E402
from raindrop_b200.synth import make_batch, model_config  # noqa: E402
from raindrop_b200.train import TrainStep  # noqa: E402


def short_name(name):
    """'void rd::(anonymous namespace)::tc_nt_kernel<72, true>(CUtensorMap_st, ...)' -> 'tc_nt_kernel<72, true>'"""
    name = re.sub(r"^void\s+", "", name.replace("(anonymous namespace)::", ""))
    depth = 0
    for i, ch in enumerate(name):          # drop the parameter list: the first '(' outside template brackets
        depth += (ch == "<") - (ch == ">")
        if ch == "(" and depth == 0:
            name = name[:i]
            break
    return re.sub(r"\b\w+::", "", name)


def kernel_events(run):
    """Runs `run()` under the profiler; returns the device kernels in launch order: (name, us, grid, smem)."""
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    evs = [e for e in trace.get("traceEvents", []) if e.get("cat") == "kernel" and e.get("ph") == "X"]
    evs.sort(key=lambda e: e["ts"])
    return [(short_name(e["name"]), float(e["dur"]), e.get("args", {}).get("grid"),
             e.get("args", {}).get("shared memory")) for e in evs]


def table(evs, step_us):
    agg = collections.OrderedDict()
    for name, us, _, _ in evs:
        n, t = agg.get(name, (0, 0.0))
        agg[name] = (n + 1, t + us)
    total = sum(t for _, t in agg.values())
    rows = sorted(([k, n, t] for k, (n, t) in agg.items()), key=lambda r: -r[2])
    return rows, total


def report(title, evs, step_us):
    rows, total = table(evs, step_us)
    print("\n== %s: %d launches, kernel sum %.1f us, CUDA-event step %.1f us (graph replay, median) ==" %
          (title, len(evs), total, step_us))
    print("%-58s %8s %10s %7s" % ("kernel", "launches", "total us", "share"))
    for name, n, t in rows:
        print("%-58s %8d %10.1f %6.1f%%" % (name[:58], n, t, 100.0 * t / total if total else 0.0))
    nt = [(i, us, grid, smem) for i, (name, us, grid, smem) in enumerate(evs) if name.startswith("tc_nt_kernel")]
    print("tc_nt_kernel launches in step order (index in the step, grid, dynamic smem, us):")
    for i, us, grid, smem in nt:
        print("  #%-3d grid %-16s smem %-7s %7.1f" % (i, grid, smem, us))
    print("tc_nt_kernel: %d launches, %.1f us = %.1f %% of the kernel sum" %
          (len(nt), sum(x[1] for x in nt), 100.0 * sum(x[1] for x in nt) / total if total else 0.0))
    return {"title": title, "launches": len(evs), "kernel_sum_us": total, "step_us": step_us,
            "kernels": [{"name": n_, "launches": c, "total_us": t} for n_, c, t in rows],
            "tc_nt": [{"index": i, "grid": g, "smem": s, "us": u} for i, u, g, s in nt]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="P19")
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--repeat", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("step_kernel_times.py needs a GPU")
    cfg = model_config(args.config, dropout=0.2)
    batch = to_dev(make_batch(cfg, args.batch, seed=1))

    m_graph = build_dropin(cfg, 4).train()
    ts = TrainStep(m_graph, args.batch, use_graph=True)
    ts.load_batch(batch)
    for _ in range(3):
        ts.step()
    torch.cuda.synchronize()
    times = []
    for _ in range(args.repeat):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ts.step()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) * 1000.0)
    step_us = statistics.median(times)

    graph_evs = kernel_events(ts.step)

    m_eager = build_dropin(cfg, 4).train()
    te = TrainStep(m_eager, args.batch, use_graph=False)
    te.load_batch(batch)
    for _ in range(3):
        te.step()
    torch.cuda.synchronize()
    eager_evs = kernel_events(te.step)

    print("device: %s, config %s, B = %d, step %.1f us (median of %d graph replays, range %.1f - %.1f)" %
          (torch.cuda.get_device_name(), args.config, args.batch, step_us, len(times), min(times), max(times)))
    res = {"device": torch.cuda.get_device_name(), "config": args.config, "batch": args.batch,
           "step_us_median": step_us, "step_us_all": times,
           "eager": report("eager enqueue", eager_evs, step_us),
           "graph": report("graph replay", graph_evs, step_us)}
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "step_kernel_times.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
