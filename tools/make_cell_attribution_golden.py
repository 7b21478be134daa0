"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/cell_attribution.npz from the reference's own, unmodified files
(oracle/ref_harness.py) on CPU; leaves every other fixture untouched:

    RAINDROP_REFERENCE=<checkout of mims-harvard/Raindrop> python tools/make_cell_attribution_golden.py   # repo root

Attribution over players of a map of the value cells (feature_mask of raindrop_b200.attribution) of F =
logits[b, target[b]] of the reference model in eval mode, for cases of oracle/make_golden.py (inputs and weights
regenerated from their seeds).  Cell (t, b, n) of the value half belongs to player cells[t, b, n] (-1: no player); when
the model has statics the static vector is player G = max id + 1.  Removing a player zeroes its cells (the zero
baseline) or the static vector; the mask half, times and lengths are unchanged.  Every coalition value v(S) = F(x with
the players outside S removed) is one row of a reference forward.

    "<case>.cells"            [T, B, N] int32: the map (a [T, N] map is stored broadcast over the batch)
    "<case>.ablation"         [B, P]  v(all) - v(all but g), every case
    "<case>.shapley"          [B, P]  exact Shapley values by subset enumeration in fp64 (TINY cases)
    "<case>.endpoint_logits"  [2, B, n_classes]: logits at the zero baseline and at x
    "<case>.target"           [B]: the labels, or the argmax at x (tiny_t0)

Maps (meta["maps"]):
    tiny_dense      [T, N] shared by the batch: 2 index windows (t < T/2, t >= T/2) x groups [0, 0, 1, 1, 2], id = w*3 + g
    tiny_t0         per sample: time_window_mask(times, max(times) / 2, n_windows=2, sensor_groups=[0, 0, 1, 1, 2])
    p19_b5_leave10, p12_b2, pam_b2   per sample: time_window_mask(times, window, sensor_groups=d_inp)
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
from raindrop_b200.attribution import time_window_mask  # noqa: E402
from raindrop_b200.synth import make_batch, model_config, synth_weights  # noqa: E402

# case -> target: "labels" or None = argmax of the logits at x
SHAPLEY = {"tiny_dense": "labels", "tiny_t0": None}
ABLATION_ONLY = {"p19_b5_leave10": "labels", "p12_b2": "labels", "pam_b2": "labels"}
TINY_GROUPS = [0, 0, 1, 1, 2]
WINDOWS = {"p19_b5_leave10": 12.0, "p12_b2": 12.0, "pam_b2": 100.0}     # in the units of `times`
ROWS_PER_FORWARD = 256


def cell_map(name, batch, N):
    """(cells [T, B, N] int64, description) of a case."""
    times = batch["times"]
    T, B = times.shape
    if name == "tiny_dense":
        w = (torch.arange(T) >= T // 2).long()
        cells = (w[:, None] * 3 + torch.as_tensor(TINY_GROUPS)[None, :])[:, None, :].expand(T, B, N)
        return cells, dict(kind="[T, N]", index_windows=2, groups=TINY_GROUPS)
    if name == "tiny_t0":
        window = float(times.max()) / 2
        cells, n_win = time_window_mask(times, window, n_windows=2, sensor_groups=TINY_GROUPS)
        return cells.long(), dict(kind="time_window_mask", window=window, n_windows=n_win, groups=TINY_GROUPS)
    cells, n_win = time_window_mask(times, WINDOWS[name], sensor_groups=N)
    return cells.long(), dict(kind="time_window_mask", window=WINDOWS[name], n_windows=n_win, groups=N)


def coalition_values(forward, batch, cells, masks, target):
    """v[S, b] = logits[b, target[b]] of the input whose players outside S are zeroed, S = rows of `masks` [n_S, P]
    (bool; players = the ids of `cells` [T, B, N], then the static player), in fp64; forwards of ROWS_PER_FORWARD rows."""
    src, static, times, lengths = batch["src"], batch["static"], batch["times"], batch["lengths"]
    N = src.shape[2] // 2
    B = src.shape[1]
    G = int(cells.max()) + 1
    out = []
    per = max(1, ROWS_PER_FORWARD // B)
    for s in range(0, len(masks), per):
        xs, ss = [], []
        for keep in masks[s:s + per]:
            k = torch.cat([torch.as_tensor(keep[:G]), torch.ones(1, dtype=torch.bool)])   # id -1 -> the last: kept
            x = src.clone()
            x[:, :, :N] *= k[cells].to(x.dtype)
            xs.append(x)
            if static is not None:
                ss.append(static * float(keep[-1]))
        n = len(xs)
        logits = forward(torch.cat(xs, dim=1), torch.cat(ss, dim=0) if static is not None else None, times.repeat(1, n),
                         lengths.repeat(n))
        out.append(logits.view(n, B, -1).gather(2, target.view(1, B, 1).expand(n, B, 1))[:, :, 0].double())
    return torch.cat(out, dim=0)


def ablation(forward, batch, cells, P, target):
    masks = [np.ones(P, dtype=bool)] + [np.arange(P) != g for g in range(P)]
    v = coalition_values(forward, batch, cells, masks, target)
    return (v[0][None, :] - v[1:]).T                                    # [B, P]


def exact_shapley(forward, batch, cells, P, target):
    masks = [np.array(bits, dtype=bool) for bits in itertools.product([False, True], repeat=P)]
    v = coalition_values(forward, batch, cells, masks, target)
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
    out, maps = {}, {}
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
        cells, maps[name] = cell_map(name, batch, N)
        G = int(cells.max()) + 1
        P = G + (1 if static is not None else 0)
        out[name + ".cells"] = cells.to(torch.int32).numpy()
        out[name + ".ablation"] = ablation(forward, batch, cells, P, target).float().numpy()
        if name in SHAPLEY:
            phi = exact_shapley(forward, batch, cells, P, target)
            out[name + ".shapley"] = phi.float().numpy()
            f = ends.gather(2, target.view(1, -1, 1).expand(2, -1, 1))[:, :, 0].double()
            eff = float((phi.sum(dim=1) - (f[1] - f[0])).abs().max())
            print("%-16s P=%d  efficiency residual %.2e" % (name, P, eff))
        out[name + ".endpoint_logits"] = ends.numpy()
        out[name + ".target"] = target.numpy()
        print("%-16s P=%d  ablation max %.3e" % (name, P, float(np.abs(out[name + ".ablation"]).max())))
    meta = dict(shapley=SHAPLEY, ablation_only=ABLATION_ONLY, maps=maps, baseline="zeros", mode="eval",
                torch=torch.__version__, reference_commit="892eb57", generator="tools/make_cell_attribution_golden.py")
    out["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(GOLDEN, "cell_attribution.npz"), **out)
    print("cell_attribution  %d arrays" % len(out))


if __name__ == "__main__":
    main()
