"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/input_grads.npz from the reference's own, unmodified files
(oracle/ref_harness.py) on CPU; leaves every other fixture untouched:

    RAINDROP_REFERENCE=<checkout of mims-harvard/Raindrop> python tools/make_input_grad_golden.py      # from the repo root

Gradients of the cross-entropy loss with respect to the model INPUTS src, static and times, eval mode, for the cases of
oracle/make_golden.py (inputs and weights regenerated from their seeds) and for legacy Raindrop v1 on the setup of
make_golden.v1_case().  Keys "<case>.d_src" / ".d_static" / ".d_times": full tensors for the TINY cases, fingerprints
("#sample" / "#stats", as make_golden stores them) for the larger ones.
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
from oracle.make_golden import CASES, GOLDEN, fingerprint, sparse_structure  # noqa: E402
from raindrop_b200.synth import CONFIGS, make_batch, model_config, synth_weights  # noqa: E402

FULL = ["tiny_dense", "tiny_t0", "tiny_sparse", "tiny8_nostatic"]
FINGERPRINT = ["p19_b5_leave10", "p12_b2", "pam_b2"]


def v2_cases(out):
    for name, cfg_name, B, dseed, wseed, opt in CASES:
        if name not in FULL + FINGERPRINT:
            continue
        cfg = model_config(cfg_name, dropout=0.2)
        if "sparse" in opt:
            cfg["global_structure"] = sparse_structure(cfg["d_inp"], opt["sparse"])
        model = ref_harness.build_reference_model(cfg).eval()
        synth_weights(model, cfg, seed=wseed)
        batch = make_batch(cfg, B, seed=dseed, first_time_zero=opt.get("first_time_zero", False),
                           zero_sensors=opt.get("zero_sensors", 0))
        inputs = {"d_src": batch["src"].clone().requires_grad_(True),
                  "d_times": batch["times"].clone().requires_grad_(True)}
        if batch["static"] is not None:
            inputs["d_static"] = batch["static"].clone().requires_grad_(True)
        logits, _, _ = model.forward(inputs["d_src"], inputs.get("d_static"), inputs["d_times"], batch["lengths"])
        grads = torch.autograd.grad(F.cross_entropy(logits, batch["y"]), list(inputs.values()))
        for k, g in zip(inputs, grads):
            if name in FULL:
                out["%s.%s" % (name, k)] = g.numpy()
            else:
                fp = fingerprint(g)
                out["%s.%s#sample" % (name, k)] = fp["sample"]
                out["%s.%s#stats" % (name, k)] = np.array([fp["sum"], fp["asum"], fp["l2"]], dtype=np.float64)
        print("%-18s %s" % (name, ", ".join("%s max %.3e" % (k, float(g.abs().max())) for k, g in zip(inputs, grads))))


def v1_case(out):
    ref = ref_harness.load_reference()
    cfg = dict(CONFIGS["P12"]); cfg["name"] = "P12"
    batch = make_batch(dict(cfg, d_ob=2), 3, seed=77)
    torch.manual_seed(5)
    gs = (torch.rand(36, 36) < 0.5).float() * torch.rand(36, 36)
    model = ref.Raindrop(36, 72, 2, 144, 2, 0.2, 215, 9, 100, 0.5, "mean", 2, gs.clone()).eval()
    with torch.no_grad():
        model.encoder.weight.uniform_(-0.3, 0.3)
        model.emb.weight.uniform_(-0.3, 0.3)
    static = batch["static"].clone().requires_grad_(True)
    times = batch["times"].clone().requires_grad_(True)
    logits, _, _ = model.forward(batch["src"], static, times, batch["lengths"])
    d_static, d_times = torch.autograd.grad(F.cross_entropy(logits, batch["y"]), [static, times])
    out["v1_p12_b3.d_static"], out["v1_p12_b3.d_times"] = d_static.numpy(), d_times.numpy()


def main():
    torch.set_num_threads(8)
    out = {}
    v2_cases(out)
    v1_case(out)
    meta = dict(full=FULL + ["v1_p12_b3"], fingerprint=FINGERPRINT, loss="cross_entropy", mode="eval",
                torch=torch.__version__, reference_commit="892eb57", generator="tools/make_input_grad_golden.py")
    out["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(GOLDEN, "input_grads.npz"), **out)
    print("input_grads  %d arrays" % len(out))


if __name__ == "__main__":
    main()
