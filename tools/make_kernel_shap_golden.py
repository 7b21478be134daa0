"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/kernel_shap.npz from the reference's own, unmodified files
(oracle/ref_harness.py) on CPU; leaves every other fixture untouched:

    RAINDROP_REFERENCE=<checkout of mims-harvard/Raindrop> python tools/make_kernel_shap_golden.py   # repo root

The value of EVERY coalition of the TINY cases of make_sensor_attribution_golden.py, so that any coalition set -- the
exhaustive one or a sampled one -- can be checked against reference values: v(S) = logits[b, target[b]] of the reference
model in eval mode on the input whose players outside S are zeroed (the zero baseline), in fp64.  Players and removal
are those of make_sensor_attribution_golden.py (sensors, sensor groups) and make_cell_attribution_golden.py (a map of
the value cells), whose coalition_values this script calls.

    "coalitions_<P>"            [2^P, P] uint8: the coalition index, row i = the i-th tuple of
                                itertools.product([0, 1], repeat=P) (player 0 is the most significant bit)
    "<case>.values"             [2^P, B] fp64: v(S) per sensor player (plus the static player), rows as coalitions_<P>
    "tiny_dense.values_grouped" the same over the sensor groups meta["groups"] plus the static player
    "tiny_dense.cells"          [T, B, N] int32: the cell map of make_cell_attribution_golden.py's tiny_dense case
    "tiny_dense.values_cells"   the same over its players plus the static player
    "<case>.endpoint_logits"    [2, B, n_classes]: logits at the zero baseline and at x
    "<case>.target"             [B]: the labels, or the argmax at x (tiny_t0)
"""
import itertools
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import make_cell_attribution_golden as cell_golden  # noqa: E402
import make_sensor_attribution_golden as sensor_golden  # noqa: E402
from oracle import ref_harness  # noqa: E402
from oracle.make_golden import CASES, GOLDEN, sparse_structure  # noqa: E402
from raindrop_b200.synth import make_batch, model_config, synth_weights  # noqa: E402

CELL_CASE = "tiny_dense"


def coalition_index(P):
    return np.array(list(itertools.product([0, 1], repeat=P)), dtype=np.uint8)


def main():
    torch.set_num_threads(8)
    out = {}
    for name, cfg_name, B, dseed, wseed, opt in CASES:
        if name not in sensor_golden.SHAPLEY:
            continue
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
        target = batch["y"] if sensor_golden.SHAPLEY[name] == "labels" else ends[1].argmax(dim=1)
        extra = 1 if static is not None else 0

        def values(groups_or_cells, P, by_cells=False):
            masks = coalition_index(P).astype(bool)
            out.setdefault("coalitions_%d" % P, coalition_index(P))
            fn = cell_golden.coalition_values if by_cells else sensor_golden.coalition_values
            return fn(forward, batch, groups_or_cells, list(masks), target).numpy()

        out[name + ".values"] = values(np.arange(N), N + extra)
        if name in sensor_golden.GROUPS:
            g = np.asarray(sensor_golden.GROUPS[name])
            out[name + ".values_grouped"] = values(g, int(g.max()) + 1 + extra)
        if name == CELL_CASE:
            cells, _ = cell_golden.cell_map(name, batch, N)
            out[name + ".cells"] = cells.to(torch.int32).numpy()
            out[name + ".values_cells"] = values(cells, int(cells.max()) + 1 + extra, by_cells=True)
        out[name + ".endpoint_logits"] = ends.numpy()
        out[name + ".target"] = target.numpy()
        print("%-16s P=%d  %d coalitions x B=%d" % (name, N + extra, out[name + ".values"].shape[0], B))
    meta = dict(cases=sensor_golden.SHAPLEY, groups=sensor_golden.GROUPS, cell_case=CELL_CASE, baseline="zeros",
                mode="eval", torch=torch.__version__, reference_commit="892eb57",
                generator="tools/make_kernel_shap_golden.py")
    out["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(GOLDEN, "kernel_shap.npz"), **out)
    print("kernel_shap  %d arrays" % len(out))


if __name__ == "__main__":
    main()
