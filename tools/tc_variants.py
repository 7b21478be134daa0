"""Times the message-passing kernel back to back and with an L2 flush (debug aid)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from raindrop_b200 import lib as L
lib = L.load()
def rn(t):
    i = t.contiguous().view(torch.int32); return ((i + 0x1000) & ~0x1FFF).view(torch.float32)
N, C, rows = 34, 240, 16384 * 34
x = rn(torch.randn(rows, C, device="cuda")); W = rn(torch.randn(C, C, device="cuda") / C ** 0.5)
b = torch.zeros(C, device="cuda"); s = torch.ones(N, device="cuda"); y = torch.empty_like(x)
fn = lambda: L.check(lib.rd_obprop_fwd(x.data_ptr(), W.data_ptr(), b.data_ptr(), s.data_ptr(), N, rows, C, y.data_ptr(), None, L.stream_ptr()), "f")
for _ in range(5): fn()
torch.cuda.synchronize()
def b2b(n=20):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize(); return e0.elapsed_time(e1) / n
flush = torch.empty(64 << 20, device="cuda")
def flushed(mode, n=20):
    ts = []
    for _ in range(n):
        if mode >= 1: flush.zero_()
        if mode >= 2: flush.sum()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1))
    ts.sort(); return ts[len(ts) // 2], ts[0]
gb = rows * C * 8 / 1e9
for name, t in (("back-to-back", b2b()), ("sync each, no flush", flushed(0)[0]), ("write flush", flushed(1)[0]), ("write+read flush", flushed(2)[0])):
    print("%-22s %.4f ms  %.0f GB/s  %.1f%% of the 3.35 TB/s H100 data sheet" % (name, t, gb / t * 1e3, 100 * gb / t * 1e3 / 3350.0))
