"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/trak_margin_grads.npz from the reference's own, unmodified files
(oracle/ref_harness.py) on CPU; leaves every other fixture untouched:

    RAINDROP_REFERENCE=<checkout of mims-harvard/Raindrop> python tools/make_trak_golden.py      # from the repo root

Per-sample gradients of the margin m_b = z_y - log sum_{c != y} exp(z_c) (one-sample backwards of the reference model in
eval mode) with respect to every trained tensor, laid out as a gradient row of raindrop_b200.influence, and
Q_b = sigmoid(-m_b).  Keys "<case>.G" (float64 rows) and "<case>.Q".  Inputs are make_batch(cfg, B, seed) and weights
synth_weights(seed=21), as the tests regenerate them.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import ref_harness  # noqa: E402
from oracle.make_golden import GOLDEN  # noqa: E402
from raindrop_b200.functional import used_param_fields  # noqa: E402
from raindrop_b200.synth import make_batch, model_config, synth_weights  # noqa: E402

# (case, configuration, B, data seed): 2 and 8 classes
CASES = [("tiny", "TINY", 3, 71), ("tiny8", "TINY8", 4, 72)]
WEIGHT_SEED = 21


def margin(logits, y):
    others = torch.ones_like(logits, dtype=torch.bool)
    others[torch.arange(len(y)), y] = False
    rest = logits.masked_fill(~others, float("-inf"))
    return logits.gather(1, y[:, None])[:, 0] - torch.logsumexp(rest, dim=1)


def rows(cfg, B, seed):
    model = ref_harness.build_reference_model(cfg).eval()
    synth_weights(model, cfg, seed=WEIGHT_SEED)
    batch = make_batch(cfg, B, seed=seed)
    keys = [k for k, _ in used_param_fields(cfg["nlayers"], cfg["static"])]      # the gradient-row order
    params = dict(model.named_parameters())
    logits, _, _ = model.forward(batch["src"], batch["static"], batch["times"], batch["lengths"])
    m = margin(logits, batch["y"])
    G = []
    for b in range(B):
        gs = torch.autograd.grad(m[b], [params[k] for k in keys], retain_graph=True)
        parts = []
        for g in gs:
            v = g.detach().double().reshape(-1)
            parts += [v, torch.zeros((-v.numel()) % 4, dtype=torch.float64)]
        G.append(torch.cat(parts))
    Q = torch.sigmoid(-m.detach().double())
    return torch.stack(G).numpy(), Q.numpy()


def main():
    torch.set_num_threads(8)
    out = {}
    for name, cfg_name, B, seed in CASES:
        cfg = model_config(cfg_name, dropout=0.2)
        G, Q = rows(cfg, B, seed)
        out[name + ".G"], out[name + ".Q"] = G, Q
        print("%-6s B=%d bucket=%d  |g| %s  Q %s" % (name, B, G.shape[1], np.round(np.linalg.norm(G, axis=1), 4),
                                                     np.round(Q, 4)))
    meta = dict(cases=[list(c) for c in CASES], weight_seed=WEIGHT_SEED, output="margin", mode="eval",
                torch=torch.__version__, reference_commit="892eb57", generator="tools/make_trak_golden.py")
    out["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    path = os.path.join(GOLDEN, "trak_margin_grads.npz")
    np.savez_compressed(path, **out)
    print("trak_margin_grads  %d arrays, %d bytes" % (len(out), os.path.getsize(path)))


if __name__ == "__main__":
    main()
