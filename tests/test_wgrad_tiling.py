"""GPU: the grouped weight-gradient kernel (tc_wgrad_kernel) under every tile width it is instantiated for.

dW = dY^T X and db = sum_r dY[r, :] through rd_linear_wgrad_group, every element within its engine's componentwise bound
of an fp64 product (test_wgrad_operators.check_public):
  * the ten problems of the P19 (B = 128) and PAM (B = 256) training steps in one group, under every width forced with
    RD_TC_WGRAD_BN (read at each call).  The row splits depend on the group's shapes alone, so every width computes each
    output element as the same product sequence: the results are bitwise equal across widths;
  * M and N tails (Nout, Kin not multiples of 64 / of the width), rows below 32 and rows not a multiple of 32;
  * two calls of the same group are bitwise equal;
  * one P19 training step from identical state, this kernel against the CUDA-core split-K path (RD_TC_WGRAD=0, read
    once per process, hence two subprocesses): every weight and bias gradient within 2e-5 normwise, logits and loss
    bitwise equal (the weight gradients come last in the backward and feed nothing else of the step).
"""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from test_wgrad_operators import check_public

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIDTHS = [32, 64, 96, 128, 144, 160]
BATCH = {"P19": 128, "PAM": 256}


def step_problems(config):
    from raindrop_b200.synth import model_config
    cfg = model_config(config)
    B = BATCH[config]
    D, nhid, C = cfg["d_model"] + 16, cfg["nhid"], cfg["max_len"] * cfg["d_ob"]
    m2, m1 = cfg["max_len"] * B, B * cfg["d_inp"]
    enc = [(m2, D, nhid), (m2, nhid, D), (m2, D, D), (m2, 3 * D, D)]
    return enc + enc + [(m1, C, C)] * 2


class Group:
    """inputs, outputs and partial buffers of one rd_linear_wgrad_group call"""

    def __init__(self, shapes, seed=3):
        from raindrop_b200 import lib as L
        self.L, self.lib = L, L.load()
        g = torch.Generator().manual_seed(seed)
        self.items = (L.RdWgradItem * len(shapes))()
        self.ins, self.outs, self.parts = [], [], []
        for i, (rows, nout, kin) in enumerate(shapes):
            dY = torch.randn(rows, nout, generator=g).cuda()
            X = torch.randn(rows, kin, generator=g).cuda()
            dW, db = torch.empty(nout, kin, device="cuda"), torch.empty(nout, device="cuda")
            part = torch.empty(max(1, self.lib.rd_linear_wgrad_partial_bytes(rows, nout, kin) // 4), device="cuda")
            it = self.items[i]
            it.d_out, it.x, it.rows, it.out_features, it.in_features = dY.data_ptr(), X.data_ptr(), rows, nout, kin
            it.d_weight, it.d_bias, it.partial = dW.data_ptr(), db.data_ptr(), part.data_ptr()
            self.ins.append((dY, X)); self.outs.append((dW, db)); self.parts.append(part)

    def run(self, bn=None):
        if bn is not None:
            os.environ["RD_TC_WGRAD_BN"] = str(bn)
        try:
            for dW, db in self.outs:
                dW.fill_(float("nan")); db.fill_(float("nan"))
            self.L.check(self.lib.rd_linear_wgrad_group(self.items, len(self.outs), self.L.stream_ptr()), "rd_linear_wgrad_group")
            torch.cuda.synchronize()
        finally:
            os.environ.pop("RD_TC_WGRAD_BN", None)
        return [(dW.clone(), db.clone()) for dW, db in self.outs]

    def check_fp64(self, res, tag, bn=None):
        check_public(self.ins, res, "tiling %s" % (tag,), bn)


def same_bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("config", ["P19", "PAM"])
def test_step_problems_every_width(config):
    grp = Group(step_problems(config))
    ref = grp.run()
    grp.check_fp64(ref, (config, "default"))
    for bn in WIDTHS:
        got = grp.run(bn)
        grp.check_fp64(got, (config, bn), bn)
        for (a, b), (c, d) in zip(got, ref):
            assert same_bits(a, c) and same_bits(b, d), (config, bn, tuple(a.shape))


@pytest.mark.parametrize("shapes", [
    [(17, 20, 36)],                                       # rows < 32
    [(1000, 68, 100), (333, 200, 16)],                    # rows not a multiple of 32; M and N tails
    [(5000, 456, 152), (31, 16, 16), (777, 860, 860)],    # a full-width tail, the smallest shape, a wide one
])
def test_tails_every_width(shapes):
    grp = Group(shapes, seed=len(shapes))
    ref = grp.run()
    grp.check_fp64(ref, "default")
    for bn in WIDTHS:
        got = grp.run(bn)
        grp.check_fp64(got, bn, bn)
        for (a, b), (c, d) in zip(got, ref):
            assert same_bits(a, c) and same_bits(b, d), (bn, tuple(a.shape))


def test_repeat_bitwise():
    grp = Group(step_problems("P19"))
    a, b = grp.run(), grp.run()
    for (x, y), (u, v) in zip(a, b):
        assert same_bits(x, u) and same_bits(y, v)


STEP_SCRIPT = r"""
import sys
import numpy as np
import torch
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
from helpers import build_dropin, to_dev
from raindrop_b200.synth import make_batch, model_config
from raindrop_b200.train import TrainStep
cfg = model_config("P19", dropout=0.2)
m = build_dropin(cfg, 4).train()
ts = TrainStep(m, 128, use_graph=False)
ts.load_batch(to_dev(make_batch(cfg, 128, seed=3)))
ts.step()
torch.cuda.synchronize()
sizes = [p.numel() for p in m.used_parameters()]
np.savez(sys.argv[2], logits=ts.logits.cpu().numpy(), loss=ts.loss.cpu().numpy(), grad=ts.flat_g.cpu().numpy(),
         offsets=np.array(ts.offsets), sizes=np.array(sizes))
"""


def test_train_step_against_cuda_core_path():
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for tag, env in (("tc", {}), ("cc", {"RD_TC_WGRAD": "0"})):
            path = os.path.join(d, tag + ".npz")
            r = subprocess.run([sys.executable, "-c", STEP_SCRIPT, ROOT, path], env={**os.environ, **env},
                               capture_output=True, text=True, timeout=600)
            assert r.returncode == 0, r.stderr[-3000:]
            out[tag] = dict(np.load(path))
    tc, cc = out["tc"], out["cc"]
    assert np.array_equal(tc["logits"].view(np.int32), cc["logits"].view(np.int32))
    assert np.array_equal(tc["loss"].view(np.int32), cc["loss"].view(np.int32))
    worst = 0.0
    for off, n in zip(tc["offsets"], tc["sizes"]):
        a, b = tc["grad"][off:off + n].astype(np.float64), cc["grad"][off:off + n].astype(np.float64)
        if np.linalg.norm(b) > 0:
            e = np.linalg.norm(a - b) / np.linalg.norm(b)
            worst = max(worst, e)
            assert e < 2e-5, (int(off), int(n), e)
    assert worst > 0.0          # the two paths really differ (different summation orders)
