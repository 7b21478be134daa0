"""GPU: the tile plan of tc_nt_kernel does not change what it computes.

Every output element is the same sequence of fp32 products whatever the tile width (k-blocks in order; per 8-wide k-step
lo.hi, hi.lo, hi.hi into one accumulator), so every plan must give bitwise the same result.  RD_TC_NT_BN=<width> forces a
width for every tc_nt launch of the width's mode it can serve (it is read at each launch; launches of the other mode keep
their default plan); each run is compared with the default plan:
  * one eager training step (dropout 0.2) of P19 at B = 127 under every error-compensated width: encoder rows 7620 and
    ob-prop rows 4318 (not multiples of 64), N x K in {152, 272, 456}^2, ob-prop C = 240 error-compensated.  Flag sets:
    dropout + residual + keep bits, relu + dropout, gate, residual, the plain product, and on the ob-prop side
    relu + scale, permuted store + relu + scale, gate + scale;
  * one eager training step of PAM at B = 16 under every single-pass width: the ob-prop layers (272 rows, C = 2400) run
    single pass with relu + scale + TF32 rounding (layer 1), permuted store + relu + scale (layer 2) and gate + scale
    (backward);
    both compare logits, loss, every gradient, the updated parameters and the whole workspace (activations and the
    dropout keep bits the GEMM epilogue stores);
  * one Monte Carlo dropout call (P19, B = 5, 6 replicates) under every error-compensated width: the replicate-major
    dropout epilogues (dropout + residual + replicate rows, relu + dropout + replicate rows); the replicates' logits and
    all statistics are compared;
  * one ob-prop layer forward on its own at C = 240 (error-compensated) and C = 1024, 2400 (single pass, relu + scale),
    against an fp64 product: within 4e-6 normwise for the error-compensated mode, and for the single pass against the
    fp64 product of the TF32-rounded operands within fp32 accumulation error; and bitwise across the widths.
"""
import os

import numpy as np
import pytest
import torch

from helpers import build_dropin, to_dev

pytestmark = pytest.mark.gpu

EXACT_WIDTHS = [48, 80, 96, 120, 136, 152, 184, 232]
FAST_WIDTHS = [64, 96, 128, 160, 192, 224, 240, 256]


class forced_width:
    def __init__(self, bn):
        self.bn = bn

    def __enter__(self):
        if self.bn is not None:
            os.environ["RD_TC_NT_BN"] = str(self.bn)

    def __exit__(self, *exc):
        os.environ.pop("RD_TC_NT_BN", None)


def train_step_outputs(config, B, bn):
    from raindrop_b200.synth import make_batch, model_config
    from raindrop_b200.train import TrainStep
    cfg = model_config(config, dropout=0.2)
    m = build_dropin(cfg, 4).train()
    ts = TrainStep(m, B, use_graph=False)
    ts.load_batch(to_dev(make_batch(cfg, B, seed=3)))
    ts.ws.zero_()
    with forced_width(bn):
        ts.step()
        torch.cuda.synchronize()
    return {"logits": ts.logits.clone(), "loss": ts.loss.clone(), "grad": ts.flat_g.clone(), "param": ts.flat_p.clone(),
            "ws": ts.ws.clone()}


_default_steps = {}


def same_bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("config,B,bn", [("P19", 127, w) for w in EXACT_WIDTHS] + [("PAM", 16, w) for w in FAST_WIDTHS])
def test_train_step_bitwise_across_plans(config, B, bn):
    if config not in _default_steps:
        _default_steps[config] = train_step_outputs(config, B, None)
    ref = _default_steps[config]
    got = train_step_outputs(config, B, bn)
    for k in ref:
        assert same_bits(got[k], ref[k]), (config, bn, k, int((got[k] != ref[k]).sum()))


def mc_dropout_outputs(bn):
    from raindrop_b200.synth import make_batch, model_config
    from raindrop_b200.uncertainty import mc_dropout
    cfg = model_config("P19", dropout=0.2)
    m = build_dropin(cfg, 4).eval()
    b = to_dev(make_batch(cfg, 5, seed=11))
    with forced_width(bn):
        r = mc_dropout(m, b["src"], b["static"], b["times"], b["lengths"], n_samples=6, seed=123, return_samples=True)
        torch.cuda.synchronize()
    return {k: getattr(r, k).clone() for k in ("samples", "mean_probs", "variance", "predictive_entropy",
                                                "expected_entropy", "mutual_information")}


_default_mc = []


@pytest.mark.parametrize("bn", EXACT_WIDTHS)
def test_mc_dropout_bitwise_across_plans(bn):
    if not _default_mc:
        _default_mc.append(mc_dropout_outputs(None))
    ref = _default_mc[0]
    got = mc_dropout_outputs(bn)
    for k in ref:
        assert torch.equal(got[k], ref[k]), (bn, k)


def tf32_rna(a):
    """cvt.rna.tf32.f32 in numpy: round the low 13 mantissa bits to nearest, ties away from zero."""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def obprop_layer(x, w, b, s, mod, bn):
    from raindrop_b200.functional import ObPropLayerFunction
    with forced_width(bn), torch.no_grad():
        out = ObPropLayerFunction.apply(x, w, b, s, mod)
        torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("C,rows", [(240, 4318), (1024, 1030), (2400, 301)])
def test_obprop_layer_plans(C, rows):
    exact = 2.0 * rows * C * C <= 2.0e9
    gen = torch.Generator().manual_seed(C)
    x = torch.randn(rows, C, generator=gen).cuda()
    w = (torch.randn(C, C, generator=gen) / C ** 0.5).cuda()
    b = (0.1 * torch.randn(C, generator=gen)).cuda()
    mod = 17
    s = (0.5 + torch.rand(mod, generator=gen)).cuda()
    out0 = obprop_layer(x, w, b, s, mod, None)

    xd, wd, bd, sd = (t.double().cpu().numpy() for t in (x, w, b, s))
    if not exact:
        xd, wd = tf32_rna(x.cpu().numpy()).astype(np.float64), tf32_rna(w.cpu().numpy()).astype(np.float64)
    pre = xd @ wd.T + bd
    ref = np.maximum(pre, 0.0) * sd[np.arange(rows) % mod][:, None]
    err = np.abs(out0.double().cpu().numpy() - ref).max() / np.abs(ref).max()
    # single pass: the only error left is fp32 accumulation over K = C products, first-order bound K * 2^-24
    assert err < (4e-6 if exact else C * 2.0 ** -24), (C, err)

    for bn in (EXACT_WIDTHS if exact else FAST_WIDTHS):
        if -(-C // bn) > 64:
            continue
        out = obprop_layer(x, w, b, s, mod, bn)
        assert same_bits(out, out0), (C, bn, int((out != out0).sum()))
