"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/per_sample_grads.npz from the reference's own, unmodified files
(oracle/ref_harness.py) on CPU; leaves every other fixture untouched:

    RAINDROP_REFERENCE=<checkout of mims-harvard/Raindrop> python tools/make_influence_golden.py      # from the repo root

Per-sample gradients of CrossEntropy(logits_b, y_b) (one-sample backwards of the reference model in eval mode) with
respect to every trained tensor, laid out as a gradient row of raindrop_b200.influence (used_param_fields order, each
tensor at an offset rounded up to 4), and the float64 TracIn matrix G G^T between each case's samples.  Keys
"<case>.G" (float64 rows) for the TINY cases; "<case>.field_l2" [B, fields] for the P12-shape case, whose rows are too
large to store.  Inputs are make_batch(cfg, B, seed) and weights synth_weights(seed=21), as the tests regenerate them.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from oracle import ref_harness  # noqa: E402
from oracle.make_golden import GOLDEN  # noqa: E402
from raindrop_b200.functional import used_param_fields  # noqa: E402
from raindrop_b200.synth import make_batch, model_config, synth_weights  # noqa: E402

# (case, configuration, B, data seed); the full rows are stored for FULL
CASES = [("tiny", "TINY", 3, 61), ("tiny8", "TINY8", 4, 62), ("p12", "P12", 2, 63)]
FULL = ["tiny", "tiny8"]
WEIGHT_SEED = 21


def rows(cfg, B, seed):
    model = ref_harness.build_reference_model(cfg).eval()
    synth_weights(model, cfg, seed=WEIGHT_SEED)
    batch = make_batch(cfg, B, seed=seed)
    keys = [k for k, _ in used_param_fields(cfg["nlayers"], cfg["static"])]      # the gradient-row order
    params = dict(model.named_parameters())
    logits, _, _ = model.forward(batch["src"], batch["static"], batch["times"], batch["lengths"])
    G, l2 = [], []
    for b in range(B):
        gs = torch.autograd.grad(F.cross_entropy(logits[b:b + 1], batch["y"][b:b + 1]), [params[k] for k in keys],
                                 retain_graph=True)
        parts = []
        for g in gs:
            v = g.detach().double().reshape(-1)
            parts += [v, torch.zeros((-v.numel()) % 4, dtype=torch.float64)]
        G.append(torch.cat(parts))
        l2.append([float(g.double().norm()) for g in gs])
    return torch.stack(G).numpy(), np.array(l2), keys


def main():
    torch.set_num_threads(8)
    out = {}
    for name, cfg_name, B, seed in CASES:
        cfg = model_config(cfg_name, dropout=0.2)
        G, l2, keys = rows(cfg, B, seed)
        out[name + ".tracin"] = G @ G.T
        out[name + ".field_l2"] = l2
        if name in FULL:
            out[name + ".G"] = G
        print("%-6s B=%d bucket=%d  |g| %s" % (name, B, G.shape[1], np.round(np.sqrt(np.diag(G @ G.T)), 4)))
    meta = dict(cases=[list(c) for c in CASES], full=FULL, weight_seed=WEIGHT_SEED, loss="cross_entropy", mode="eval",
                torch=torch.__version__, reference_commit="892eb57", generator="tools/make_influence_golden.py")
    out["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    path = os.path.join(GOLDEN, "per_sample_grads.npz")
    np.savez_compressed(path, **out)
    print("per_sample_grads  %d arrays, %d bytes" % (len(out), os.path.getsize(path)))


if __name__ == "__main__":
    main()
