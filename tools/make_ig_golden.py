"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/integrated_gradients.npz from the reference's own, unmodified files
(oracle/ref_harness.py) on CPU; leaves every other fixture untouched:

    RAINDROP_REFERENCE=<checkout of mims-harvard/Raindrop> python tools/make_ig_golden.py      # from the repo root

Integrated gradients of F = logits[b, target[b]] with respect to src (value half) and static, eval mode, zero baselines,
for the cases of oracle/make_golden.py (inputs and weights regenerated from their seeds).  For every quadrature node the
reference model runs on the interpolated inputs and torch.autograd.grad gives dF/d(inputs); the attributions are
(x - x') * sum_k w_k grad_k.  Nodes and weights are raindrop_b200.attribution.quadrature, rounded to fp32 as the device
path reads them.  Keys "<case>.attr_src" / ".attr_static" (full tensors for the TINY cases, fingerprints "#sample" /
"#stats" for the larger ones), "<case>.endpoint_logits" [2, B, n_classes] (at the baseline, at x) and "<case>.delta" [B]
(sum of the attributions - (F(x) - F(x'))), always in full.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import ref_harness  # noqa: E402
from oracle.make_golden import CASES, GOLDEN, fingerprint, sparse_structure  # noqa: E402
from raindrop_b200.attribution import quadrature  # noqa: E402
from raindrop_b200.synth import make_batch, model_config, synth_weights  # noqa: E402

# case -> (method, n_steps, target: "labels" or None = argmax of the logits at x)
FULL = {"tiny_dense": ("gausslegendre", 16, "labels"), "tiny_sparse": ("gausslegendre", 16, "labels"),
        "tiny8_nostatic": ("gausslegendre", 16, "labels"), "tiny_t0": ("riemann_trapezoid", 9, None)}
FINGERPRINT = {"p19_b5_leave10": ("gausslegendre", 16, "labels"), "p12_b2": ("gausslegendre", 16, "labels"),
               "pam_b2": ("gausslegendre", 16, "labels")}


def ig_reference(forward, batch, target, method, n_steps):
    """(attr_src, attr_static | None, endpoint_logits [2, B, ncls], delta [B], target) with zero baselines; `forward`
    maps (src, static, times, lengths) to logits."""
    src, static, times, lengths = batch["src"], batch["static"], batch["times"], batch["lengths"]
    N = src.shape[2] // 2
    with torch.no_grad():
        x0 = src.clone()
        x0[:, :, :N] = 0
        ends = torch.stack([forward(x0, None if static is None else torch.zeros_like(static), times, lengths),
                            forward(src, static, times, lengths)])
    if target is None:
        target = ends[1].argmax(dim=1)
    a32, w32 = (torch.from_numpy(v.astype(np.float32)) for v in quadrature(n_steps, method))
    g_src = torch.zeros(src.shape, dtype=torch.float64)
    g_st = None if static is None else torch.zeros(static.shape, dtype=torch.float64)
    for a, w in zip(a32, w32):
        xs = src.clone()
        xs[:, :, :N] = a * src[:, :, :N]
        xs.requires_grad_(True)
        leaves = [xs]
        ss = None
        if static is not None:
            ss = (a * static).requires_grad_(True)
            leaves.append(ss)
        logits = forward(xs, ss, times, lengths)
        grads = torch.autograd.grad(logits.gather(1, target[:, None]).sum(), leaves)
        g_src += float(w) * grads[0].double()
        if static is not None:
            g_st += float(w) * grads[1].double()
    attr_src = (src.double() * g_src)
    attr_src[:, :, N:] = 0
    attr_st = None if static is None else static.double() * g_st
    total = attr_src.sum(dim=(0, 2)) + (0 if attr_st is None else attr_st.sum(dim=1))
    f = ends.gather(2, target.view(1, -1, 1).expand(2, -1, 1))[:, :, 0].double()
    delta = total - (f[1] - f[0])
    return attr_src.float(), None if attr_st is None else attr_st.float(), ends, delta.float(), target


def main():
    torch.set_num_threads(8)
    out = {}
    for name, cfg_name, B, dseed, wseed, opt in CASES:
        spec = FULL.get(name) or FINGERPRINT.get(name)
        if spec is None:
            continue
        method, n_steps, tmode = spec
        cfg = model_config(cfg_name, dropout=0.2)
        if "sparse" in opt:
            cfg["global_structure"] = sparse_structure(cfg["d_inp"], opt["sparse"])
        model = ref_harness.build_reference_model(cfg).eval()
        synth_weights(model, cfg, seed=wseed)
        batch = make_batch(cfg, B, seed=dseed, first_time_zero=opt.get("first_time_zero", False),
                           zero_sensors=opt.get("zero_sensors", 0))

        def forward(s, st, t, ln):
            return model.forward(s, st, t, ln)[0]
        attr_src, attr_st, ends, delta, target = ig_reference(forward, batch, batch["y"] if tmode == "labels" else None,
                                                              method, n_steps)
        tensors = {"attr_src": attr_src}
        if attr_st is not None:
            tensors["attr_static"] = attr_st
        for k, t in tensors.items():
            if name in FULL:
                out["%s.%s" % (name, k)] = t.numpy()
            else:
                fp = fingerprint(t)
                out["%s.%s#sample" % (name, k)] = fp["sample"]
                out["%s.%s#stats" % (name, k)] = np.array([fp["sum"], fp["asum"], fp["l2"]], dtype=np.float64)
        out[name + ".endpoint_logits"] = ends.numpy()
        out[name + ".delta"] = delta.numpy()
        out[name + ".target"] = target.numpy()
        print("%-16s %s n=%d  attr_src max %.3e  delta %s" % (name, method, n_steps, float(attr_src.abs().max()),
                                                               np.array2string(delta.numpy(), precision=3)))
    meta = dict(full={k: list(v) for k, v in FULL.items()}, fingerprint={k: list(v) for k, v in FINGERPRINT.items()},
                baseline="zeros", mode="eval", torch=torch.__version__, reference_commit="892eb57",
                generator="tools/make_ig_golden.py")
    out["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(GOLDEN, "integrated_gradients.npz"), **out)
    print("integrated_gradients  %d arrays" % len(out))


if __name__ == "__main__":
    main()
