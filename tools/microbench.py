"""Scratch micro-benchmarks of single kernels (the benchmark of record is bench.py)."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from raindrop_b200 import functional as RF
from raindrop_b200.synth import model_config, make_batch
from raindrop_b200.train import TrainStep
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from helpers import build_dropin, to_dev


def timeit(fn, n=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(n + 1)]
    ev[0].record()
    for i in range(n):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    ts = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(n))
    return ts[len(ts) // 2], ts[0]


def layer_bench(C, N, B):
    rows = B * N
    x = torch.randn(rows, C, device="cuda")
    W = torch.randn(C, C, device="cuda") / C ** 0.5
    b = torch.randn(C, device="cuda")
    s = torch.ones(N, device="cuda")
    fn = lambda: RF.ObPropLayerFunction.apply(x, W, b, s, N)
    med, best = timeit(fn)
    gb = rows * C * 8 / 1e9
    tf = 2 * rows * C * C / 1e12
    print("obprop layer C=%d rows=%d: median %.3f ms best %.3f ms -> %.0f GB/s (%.1f%% of the 3.35 TB/s H100 data sheet), %.1f TFLOP/s"
          % (C, rows, med, best, gb / (best * 1e-3), 100 * gb / (best * 1e-3) / 3350.0, tf / (best * 1e-3)))


if __name__ == "__main__":
    print(torch.cuda.get_device_name(0), "TC=", os.environ.get("RD_OBPROP_TC", "1"))
    layer_bench(240, 34, 16384)
    layer_bench(240, 34, 128)
    layer_bench(860, 36, 1024)
    layer_bench(1024, 128, 512)
    layer_bench(2400, 17, 1024)
    cfg = model_config("P19", dropout=0.2)
    model = build_dropin(cfg, 4).train()
    d = to_dev(make_batch(cfg, 128, seed=1))
    opt = torch.optim.Adam(model.parameters(), lr=1e-4)
    def eager_step():
        logits, _, _ = model.forward(d["src"], d["static"], d["times"], d["lengths"])
        loss = torch.nn.functional.cross_entropy(logits, d["y"])
        opt.zero_grad(); loss.backward(); opt.step()
    med, best = timeit(eager_step, n=20)
    print("eager train step B=128: median %.3f ms best %.3f ms -> %.0f samples/s" % (med, best, 128 / med * 1e3))
    def fwd_only():
        with torch.no_grad():
            model.forward(d["src"], d["static"], d["times"], d["lengths"])
    med, best = timeit(fwd_only, n=20)
    print("eager forward B=128: median %.3f ms" % med)
    for B in (128, 1024):
        m2 = build_dropin(cfg, 4).train()
        ts = TrainStep(m2, B, use_graph=True)
        ts.load_batch(to_dev(make_batch(cfg, B, seed=1)))
        ts.capture()
        med, best = timeit(ts.step, n=30)
        print("graph train step B=%d: median %.3f ms best %.3f ms -> %.0f samples/s" % (B, med, best, B / med * 1e3))
