"""One CUDA-graph replay of the training step between cudaProfilerStart/Stop (warm caches, kernels in graph order):
    ncu --profile-from-start off --graph-profiling node --cache-control none --clock-control none \
        --metrics gpu__time_duration.sum --csv --log-file launches_graph.csv python tools/profile_graph.py
"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import torch
from raindrop_b200.synth import model_config, make_batch
from raindrop_b200.train import TrainStep
from helpers import build_dropin, to_dev

B = int(sys.argv[1]) if len(sys.argv) > 1 else 128
cfg = model_config("P19", dropout=0.2)
m = build_dropin(cfg, 4).train()
ts = TrainStep(m, B, use_graph=True)
ts.load_batch(to_dev(make_batch(cfg, B, seed=1)))
for _ in range(5):
    ts.step()
torch.cuda.synchronize()
torch.cuda.profiler.start()
ts.step()
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("loss", ts.loss.item())
