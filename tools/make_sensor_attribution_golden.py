"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/sensor_attribution.npz from the reference's own, unmodified files
(oracle/ref_harness.py) on CPU; leaves every other fixture untouched:

    RAINDROP_REFERENCE=<checkout of mims-harvard/Raindrop> python tools/make_sensor_attribution_golden.py   # repo root

Sensor-level attribution of F = logits[b, target[b]] of the reference model in eval mode, for the integrated-gradients
cases of oracle/make_golden.py (inputs and weights regenerated from their seeds).  Players are sensor groups (default
one per sensor) plus, when the model has statics, the static vector; removing a player zeroes the value columns of its
sensors (the reference's leave-sensors-out removal) or the static vector, the mask half, times and lengths unchanged.
Every coalition value v(S) = F(x with the players outside S removed) is one row of a reference forward.

    "<case>.ablation"          [B, P]  v(all) - v(all but g), every case
    "<case>.shapley"           [B, P]  exact Shapley values, sum over all 2^P coalitions S not containing g of
                                       |S|! (P-|S|-1)! / P! (v(S + g) - v(S)) in fp64 (TINY cases)
    "tiny_dense.shapley_grouped" the same over the sensor groups meta["groups"]["tiny_dense"] plus the static player
    "<case>.endpoint_logits"   [2, B, n_classes]: logits at the zero baseline and at x
    "<case>.target"            [B]: the labels, or the argmax at x (tiny_t0)
"""
import itertools
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import ref_harness  # noqa: E402
from oracle.make_golden import CASES, GOLDEN, sparse_structure  # noqa: E402
from raindrop_b200.synth import make_batch, model_config, synth_weights  # noqa: E402

# case -> target: "labels" or None = argmax of the logits at x
SHAPLEY = {"tiny_dense": "labels", "tiny_sparse": "labels", "tiny8_nostatic": "labels", "tiny_t0": None}
ABLATION_ONLY = {"p19_b5_leave10": "labels", "p12_b2": "labels", "pam_b2": "labels"}
GROUPS = {"tiny_dense": [0, 0, 1, 1, 2]}


def coalition_values(forward, batch, groups, masks, target):
    """v[S, b] = logits[b, target[b]] of the input whose players outside S are zeroed, S = rows of `masks` [n_S, P]
    (bool, players = the groups of `groups` [N], then the static player), in fp64; one forward on n_S * B rows."""
    src, static, times, lengths = batch["src"], batch["static"], batch["times"], batch["lengths"]
    N = src.shape[2] // 2
    B = src.shape[1]
    groups = torch.as_tensor(groups)
    xs, ss = [], []
    for keep in masks:
        x = src.clone()
        x[:, :, :N] *= torch.as_tensor(keep)[groups].to(x.dtype)
        xs.append(x)
        if static is not None:
            ss.append(static * float(keep[-1]))
    n = len(masks)
    logits = forward(torch.cat(xs, dim=1), torch.cat(ss, dim=0) if static is not None else None, times.repeat(1, n),
                     lengths.repeat(n))
    return logits.view(n, B, -1).gather(2, target.view(1, B, 1).expand(n, B, 1))[:, :, 0].double()


def ablation(forward, batch, groups, P, target):
    masks = [np.ones(P, dtype=bool)] + [np.arange(P) != g for g in range(P)]
    v = coalition_values(forward, batch, groups, masks, target)
    return (v[0][None, :] - v[1:]).T                                    # [B, P]


def exact_shapley(forward, batch, groups, P, target):
    masks = [np.array(bits, dtype=bool) for bits in itertools.product([False, True], repeat=P)]
    v = coalition_values(forward, batch, groups, masks, target)
    index = {m.tobytes(): i for i, m in enumerate(masks)}
    phi = torch.zeros(v.shape[1], P, dtype=torch.float64)
    for m, i in index.items():
        keep = np.frombuffer(m, dtype=bool)
        s = int(keep.sum())
        for g in np.nonzero(~keep)[0]:
            w = math.factorial(s) * math.factorial(P - s - 1) / math.factorial(P)
            with_g = keep.copy()
            with_g[g] = True
            phi[:, g] += w * (v[index[with_g.tobytes()]] - v[i])
    return phi


def main():
    torch.set_num_threads(8)
    out = {}
    for name, cfg_name, B, dseed, wseed, opt in CASES:
        if name not in SHAPLEY and name not in ABLATION_ONLY:
            continue
        tmode = SHAPLEY.get(name, ABLATION_ONLY.get(name))
        cfg = model_config(cfg_name, dropout=0.2)
        if "sparse" in opt:
            cfg["global_structure"] = sparse_structure(cfg["d_inp"], opt["sparse"])
        model = ref_harness.build_reference_model(cfg).eval()
        synth_weights(model, cfg, seed=wseed)
        batch = make_batch(cfg, B, seed=dseed, first_time_zero=opt.get("first_time_zero", False),
                           zero_sensors=opt.get("zero_sensors", 0))

        def forward(s, st, t, ln):
            with torch.no_grad():
                return model.forward(s, st, t, ln)[0]
        src, static = batch["src"], batch["static"]
        N = src.shape[2] // 2
        x0 = src.clone()
        x0[:, :, :N] = 0
        ends = torch.stack([forward(x0, None if static is None else torch.zeros_like(static), batch["times"],
                                    batch["lengths"]),
                            forward(src, static, batch["times"], batch["lengths"])])
        target = batch["y"] if tmode == "labels" else ends[1].argmax(dim=1)
        P = N + (1 if static is not None else 0)
        groups = np.arange(N)
        out[name + ".ablation"] = ablation(forward, batch, groups, P, target).float().numpy()
        if name in SHAPLEY:
            phi = exact_shapley(forward, batch, groups, P, target)
            out[name + ".shapley"] = phi.float().numpy()
            f = ends.gather(2, target.view(1, -1, 1).expand(2, -1, 1))[:, :, 0].double()
            eff = float((phi.sum(dim=1) - (f[1] - f[0])).abs().max())
            print("%-16s P=%d  efficiency residual %.2e" % (name, P, eff))
        if name in GROUPS:
            g = np.asarray(GROUPS[name])
            Pg = int(g.max()) + 1 + (1 if static is not None else 0)
            out[name + ".shapley_grouped"] = exact_shapley(forward, batch, g, Pg, target).float().numpy()
        out[name + ".endpoint_logits"] = ends.numpy()
        out[name + ".target"] = target.numpy()
        print("%-16s ablation max %.3e" % (name, float(np.abs(out[name + ".ablation"]).max())))
    meta = dict(shapley=SHAPLEY, ablation_only=ABLATION_ONLY, groups=GROUPS, baseline="zeros", mode="eval",
                torch=torch.__version__, reference_commit="892eb57", generator="tools/make_sensor_attribution_golden.py")
    out["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(GOLDEN, "sensor_attribution.npz"), **out)
    print("sensor_attribution  %d arrays" % len(out))


if __name__ == "__main__":
    main()
