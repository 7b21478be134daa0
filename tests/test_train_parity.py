"""GPU: training mode (dropout p = 0.2, the configuration bench.py measures) against a float64 oracle that replays
the kernels' own dropout masks.

The masks cannot match torch's RNG, and they do not need to: every dropout decision of the CUDA path is a documented
function of (seed, step counter, site, element index) -- Philox4x32-10, rd_common.cuh -- which
oracle/dropout_masks.py restates in numpy.  A test reads the (seed, step) a forward captured (WS_RNG), rebuilds every
mask of that forward (lift, and per encoder layer: attention probabilities, dropout1, the FFN dropout, dropout2), runs
RaindropV2Oracle.forward_dense(masks=...) in float64 and so gets the exact train-mode logits and gradients the kernels
should have produced.  That reaches every piece of machinery that exists only because of dropout: the keep bits the
tensor-core GEMM epilogue stores for the LayerNorm backward (and the Philox regeneration used when the forward GEMM ran
on the CUDA cores), the FFN mask the backward infers from the saved activation, the attention mask that the fused
kernels regenerate and the batched path stores, and the lift mask the input gradient replays.

The oracle also replays the kernels' ReLU decisions (forward_dense(gates=...), read from the workspace: H1, the obs
columns of the encoder input, each layer's FFN activation and the head's hidden activation).  A pre-activation within
rounding distance of zero can otherwise land on the other side of its ReLU and move a gradient by up to 10 % (at PAM
B = 2 one of 81600 layer-2 ob-prop pre-activations lies within 1e-6 of zero).  Around the GPU's decisions the model is
smooth, so only rounding separates the two results.  The gates where the GPU disagrees with the oracle's own sign are
counted per site and bounded, so replay cannot hide a wrong forward.

Bounds (normwise = max|delta| / max|ref|, every tensor):
  * error-compensated ob-prop mode: TIGHT against the float64 oracle.
  * single-pass TF32 mode: against the float64 oracle under the kernels' TF32 rounding model (`tf32_model=True`) with
    the GPU's rounded layer-1 output fed to layer 2 (`h1_value`): every tensor TIGHT except the ob-prop backward's
    (lin_value gradients, d_src), FAST_TOL.  The fed H1 is itself held against the rounding model's own (H1_ULP_RATE);
    against the plain float64 oracle, logits and the encoder input normwise FWD_SANITY, gradients relative L2
    FAST_SANITY.  Where C % 4 != 0 or C < 16 the ob-prop runs on the CUDA cores in fp32 in both modes, and single-pass
    mode is held as error-compensated mode.
Measured on an H100 80GB HBM3 at 700 W: error-compensated mode at most 4.3e-6 in every case; single-pass mode up to
3.9e-4 against the rounding model (gradients) and 4.9e-4 relative L2 against plain float64.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import re

from helpers import (GATE_SITES, build_dropin, gate_disagreements, h1_ulp_ok, normwise, random_shape_case, read_gpu,
                     rel_l2, tf32_ulp_distance, to_dev)
from oracle import dropout_masks as DM
from raindrop_b200.synth import make_batch, model_config, synth_weights, used_param_keys

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXACT, FAST = 2, 1
P = 0.2
# seed and step counter with both 32-bit halves non-zero: every word of the Philox key and counter takes part
RNG0 = (0x2B7E151628AED2A6, (1 << 32) + 7)
TIGHT = 1e-4
# single-pass TF32 mode, gradients against the rounding model: measured up to 3.9e-4 (tiny_b6_len1, d_src; the backward's
# TF32 roundings of fp32 gradients land on other sides of rounding boundaries than the float64 ones)
FAST_TOL = 4e-3
FAST_TOL_TENSORS = r"(lin_value\.(weight|bias)|d_src)$"   # the ob-prop backward, where those TF32 roundings sit
FAST_SANITY = 5e-3            # single-pass TF32 mode against the plain float64 oracle, relative L2
FWD_SANITY = 1e-3             # ... and normwise on the logits and the encoder input
# single-pass mode: rates of layer-1 outputs one, and more than one, TF32 ulp from the rounding model's; 3x the worst
# measured (PAM, C = 2400: 1.1e-2 and 1.1e-3).  An output that is off by more than an ulp is a small one, computed with
# cancellation: its fp32 accumulation error is large next to its own ulp.
H1_ULP_RATE = (3.5e-2, 3.5e-3)
GATE_RATE = {EXACT: 1e-4, FAST: 2e-5}     # ReLU gates per site allowed to differ from the oracle's own sign

# name -> (config, B, make_batch options); each reaches a different dropout code path
CASES = {
    "tiny_b6_len1": ("TINY", 6, {}),            # hd = 18: attn_small; lengths[0] = 1
    "tiny8_b9": ("TINY8", 9, {}),               # attn_tc, no statics, 8 classes
    "p19_b37": ("P19", 37, {}),                 # attn_tc, D = 152: the last keep-bit word of a row is partial
    "p19_b5_t0": ("P19", 5, {"first_time_zero": True}),
    "p12_b3": ("P12", 3, {}),                   # T = 215: batched attention, stored dropped probabilities
    "pam_b2": ("PAM", 2, {}),                   # T = 600, C = 2400
    "large_b2": ("LARGE", 2, {}),               # hd = 264, C = 1024
    "p19_b9": ("P19", 9, {}),
}
RANDOM_SEEDS = range(6)
FALLBACK_CASES = ("p19_b9", "tiny8_b9")


def case_setup(name):
    """(cfg, batch, weight seed) of a named case or of `rnd<seed>` (the test_random_shapes_against_oracle generator)."""
    if name.startswith("rnd"):
        return random_shape_case(int(name[3:]))
    cfg_name, B, opts = CASES[name]
    cfg = model_config(cfg_name, dropout=P)
    batch = make_batch(cfg, B, seed=200 + B, **opts)
    if name == "tiny_b6_len1":
        batch["lengths"][0] = 1
        batch["times"][1:, 0] = 0
        batch["src"][1:, 0, :] = 0
    return cfg, batch, 21


def _ws_rng(dims, ws):
    """The (seed, step) a forward captured into its workspace (WS_RNG)."""
    from raindrop_b200 import lib as L
    n = C.c_int64(0)
    off = L.load().rd_workspace_offset(C.byref(dims), L.WS_RNG, C.byref(n))
    assert off >= 0 and off % 8 == 0 and n.value == 4
    return tuple(ws[off // 4: off // 4 + 4].view(torch.int64)[:2].tolist())


def check_masks(masks, p):
    """The masks really drop: values in {0, 1/(1-p)}, zeros in every mask large enough to have them for sure, and a
    keep rate near 1 - p overall (a test that silently ran at p = 0 would pass against all-ones masks)."""
    flat = [masks["lift"]] + [m for layer in masks["layers"] for m in layer.values()]
    inv_keep = np.float32(1) / (np.float32(1) - np.float32(p))
    for m in flat:
        assert np.all((m == 0) | (m == inv_keep))
        if m.size >= 256:
            assert (m == 0).any()
    n = sum(m.size for m in flat)
    kept = sum(int((m > 0).sum()) for m in flat) / n
    assert abs(kept - (1 - p)) < 6 * (p * (1 - p) / n) ** 0.5, kept


def oracle_train(cfg, batch, weight_seed, rng, p=P, params=None, gates=None, tf32_model=False, h1_value=None):
    """float64 train-mode reference under the masks of (seed, step) = rng and the given ReLU gates (forward_dense;
    tf32_model: under the kernels' TF32 rounding model).  `params` ({key: tensor}) overrides the synthetic weights.
    Returns (reference dict, masks); with gates, reference["gate_dis"] counts the GPU's gates that disagree with the
    oracle's own sign per site (helpers.gate_disagreements)."""
    from oracle.raindrop_oracle import build_oracle_model
    B = batch["src"].shape[1]
    masks = DM.model_masks(rng, p, cfg, B)
    oracle = build_oracle_model(cfg).eval()            # eval: the masks are the only dropout
    synth_weights(oracle, cfg, seed=weight_seed)
    if params is not None:
        missing, _ = oracle.load_state_dict(params, strict=False)
        assert not set(params) & set(missing)
    oracle.double()
    src = batch["src"].double().requires_grad_(True)
    times = batch["times"].double().requires_grad_(True)
    static = None if batch["static"] is None else batch["static"].double().requires_grad_(True)
    stages = {}
    logits, _, _ = oracle.forward_dense(src, static, times, batch["lengths"], stages=stages, masks=masks, gates=gates,
                                        tf32_model=tf32_model, h1_value=None if h1_value is None else h1_value.cpu())
    loss = F.cross_entropy(logits, batch["y"])
    loss.backward()
    go = dict(oracle.named_parameters())
    ref = dict(logits=logits.detach(), loss=loss.item(), obs=stages["obs"].detach(), pe=stages["pe"].detach(),
               enc=stages["enc"].detach(), h1_own=stages["h1_own"], grads={k: go[k].grad for k in used_param_keys(cfg)},
               d_src=src.grad, d_times=times.grad, d_static=None if static is None else static.grad)
    if gates is not None:
        ref["gate_dis"] = gate_disagreements(cfg, gates, stages, masks, slice(0, B), B, {s: [0, 0] for s in GATE_SITES})
    return ref, masks


def gpu_train(cfg, batch, weight_seed, mode, rng=RNG0):
    """One training forward + cross-entropy + backward of the drop-in with parameter and input gradients."""
    model = build_dropin(cfg, weight_seed).train()
    d = to_dev(batch)
    plan = model._prepare(d["src"].device)
    plan.rng_state.copy_(torch.tensor(rng, dtype=torch.int64))
    plan.debug_keep_workspace = True
    plan.obprop_mode = mode
    src = d["src"].clone().requires_grad_(True)
    times = d["times"].clone().requires_grad_(True)
    static = None if d["static"] is None else d["static"].clone().requires_grad_(True)
    before = tuple(plan.rng_state.tolist())
    logits, _, _ = model.forward(src, static, times, d["lengths"])
    loss = F.cross_entropy(logits, d["y"])
    loss.backward()
    assert _ws_rng(plan.last_dims, plan.last_workspace) == before == tuple(rng)    # the masks the forward drew
    assert tuple(plan.rng_state.tolist()) == (rng[0], rng[1] + 1)                 # one step consumed
    gp = dict(model.named_parameters())
    got = read_gpu(cfg, plan.last_dims, plan.last_workspace)
    got.update(logits=logits.detach(), loss=loss.item(), grads={k: gp[k].grad for k in used_param_keys(cfg)},
               d_src=src.grad, d_times=times.grad, d_static=None if static is None else static.grad)
    return got


def compare(cfg, batch, got, ref, mode, plain=None):
    """Errors of one GPU training step (gpu_train) against the gate-replaying oracle (oracle_train with got["gates"]):
    returns ({tensor: error}, [(tensor, error, bound) out of bounds]).  `ref` is the plain float64 oracle in
    error-compensated mode and the TF32 rounding model in single-pass mode; there `plain` is the plain one."""
    errs, bad = {}, []

    def chk(name, e, tol):
        errs[name] = e
        if not e < tol:
            bad.append((name, e, tol))

    N, D4 = cfg["d_inp"], cfg["d_inp"] * cfg["d_ob"]
    gtol = lambda k: FAST_TOL if mode == FAST and re.search(FAST_TOL_TENSORS, k) else TIGHT
    valid = (torch.arange(cfg["max_len"])[:, None] < batch["lengths"][None, :])
    chk("logits", normwise(got["logits"], ref["logits"]), TIGHT)
    chk("loss", abs(got["loss"] - ref["loss"]) / max(1.0, abs(ref["loss"])), TIGHT)
    chk("obs", normwise(got["enc_in"][:, :, :D4], ref["obs"]), TIGHT)
    chk("pe", normwise(got["enc_in"][:, :, D4:], ref["pe"]), 1e-5)
    chk("enc_out", normwise(got["enc_out"].cpu() * valid[:, :, None], ref["enc"] * valid[:, :, None]), TIGHT)
    if plain is None:
        chk("h1", normwise(got["h1"], ref["h1_own"]), TIGHT)
    else:
        # layer 2 took the GPU's H1: hold H1 itself against the rounding model's own, to one TF32 ulp
        ulp = tf32_ulp_distance(got["h1"], ref["h1_own"], [0, 0, 0, 0])
        if not h1_ulp_ok(ulp, H1_ULP_RATE):
            bad.append(("H1 TF32 ulp", ulp))
        chk("logits (plain float64)", normwise(got["logits"], plain["logits"]), FWD_SANITY)
        chk("obs (plain float64)", normwise(got["enc_in"][:, :, :D4], plain["obs"]), FWD_SANITY)
    for site, (n, gates) in ref["gate_dis"].items():
        if n > max(1, GATE_RATE[mode] * gates):
            bad.append(("gate disagreements " + site, n, gates))
    for k in used_param_keys(cfg):
        assert got["grads"][k] is not None, k
        chk(k, normwise(got["grads"][k], ref["grads"][k]), gtol(k))
        if plain is not None:
            chk(k + " (plain float64, rel L2)", rel_l2(got["grads"][k], plain["grads"][k]), FAST_SANITY)
    assert torch.all(got["d_src"][:, :, N:] == 0)
    vd = valid.to(got["d_times"].device)
    chk("d_src", normwise(got["d_src"][:, :, :N], ref["d_src"][:, :, :N]), gtol("d_src"))
    chk("d_times", normwise(got["d_times"] * vd, ref["d_times"] * valid), gtol("d_times"))
    if ref["d_static"] is not None:
        chk("d_static", normwise(got["d_static"], ref["d_static"]), gtol("d_static"))
    return errs, bad


def check_train_case(name, modes=(EXACT, FAST), setup=None):
    """One training step per ob-prop mode against the mask- and gate-replaying oracle (compare); `setup` = (cfg, batch,
    weight seed), default case_setup(name)."""
    cfg, batch, wseed = setup or case_setup(name)
    bad = []
    C_ = cfg["max_len"] * cfg["d_ob"]
    for mode in modes:
        got = gpu_train(cfg, batch, wseed, mode)
        gates = got["gates"]
        # where the ob-prop tensor-core kernel does not take C, both modes run the fp32 CUDA-core GEMMs
        held = EXACT if (C_ % 4 or C_ < 16) else mode
        if held == EXACT:
            ref, masks = oracle_train(cfg, batch, wseed, RNG0, gates=gates)
            plain = None
        else:
            ref, masks = oracle_train(cfg, batch, wseed, RNG0, gates=gates, tf32_model=True, h1_value=got["h1"])
            plain, _ = oracle_train(cfg, batch, wseed, RNG0, gates=gates)
        check_masks(masks, P)
        errs, b = compare(cfg, batch, got, ref, held, plain)
        top = sorted(errs.items(), key=lambda kv: -kv[1])[:5]
        tag = "exact" if mode == EXACT else "fast"
        print("train-mode parity %-12s %s B=%d mode=%s worst %s, gate disagreements %s" %
              (name, cfg["name"], batch["src"].shape[1], tag, ", ".join("%s %.2e" % kv for kv in top),
               " ".join("%s %d/%d" % (s_, n, g) for s_, (n, g) in ref["gate_dis"].items())))
        bad += [(tag,) + x for x in b]
    assert not bad, (name, bad)


# ---- 1. the mask stream itself --------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [0.1, 0.2, 0.5])
def test_debug_mask_stream_matches_numpy(p):
    """rd_debug_dropout_mask == oracle/dropout_masks.py bitwise, every site id, lengths that are not a multiple of 4,
    seeds and step counters >= 2^32 (the key word seed hi ^ step hi)."""
    from raindrop_b200 import lib as L
    lib = L.load()
    sites = [DM.SITE_LIFT] + [base + l for base in (DM.SITE_ATTN, DM.SITE_RESID1, DM.SITE_FFN, DM.SITE_RESID2)
                              for l in range(3)]
    for rng in ((1, 0), RNG0, (0x7FFFFFFF00000001, (0xABCD << 32) | 0xFFFFFFFF)):
        r = torch.tensor(rng, dtype=torch.int64, device="cuda")
        for site in sites:
            for n in (1, 7, 4099, 65537):
                out = torch.empty(n, device="cuda")
                L.check(lib.rd_debug_dropout_mask(r.data_ptr(), site, n, C.c_float(p), out.data_ptr(), L.stream_ptr()),
                        "rd_debug_dropout_mask")
                ref = DM.dropout_mask(rng[0], rng[1], site, n, p)
                assert np.array_equal(out.cpu().numpy().view(np.uint32), ref.view(np.uint32)), (rng, site, n, p)


# ---- 2. the whole model in training mode ----------------------------------------------------------------------------
@pytest.mark.parametrize("name", [n for n in CASES if n != "p19_b9"] + ["rnd%d" % s for s in RANDOM_SEEDS])
def test_train_mode_against_masked_oracle(name):
    """Logits, loss, encoder input, all parameter gradients and the input gradients of one training step (p = 0.2)
    against the float64 oracle under the same masks, in both ob-prop arithmetic modes."""
    check_train_case(name)


# ---- 3. the CUDA-core fallbacks (the switches are read once per process) ---------------------------------------------
@pytest.mark.parametrize("env", [{"RD_TC_GEMM": "0"}, {"RD_ATTN_TC": "0"}, {"RD_ATTN_TC": "0", "RD_ATTN_SMALL": "0"}],
                         ids=["cuda_core_gemm", "attn_small", "batched_attention"])
def test_cuda_core_fallbacks_against_masked_oracle(env):
    """RD_TC_GEMM=0: dropout in the CUDA-core GEMM epilogue and the LayerNorm backward regenerating the residual
    dropout decisions from Philox (no stored keep bits); RD_ATTN_TC=0: the CUDA-core fused attention at hd = 76;
    RD_ATTN_TC=0 RD_ATTN_SMALL=0: the batched attention path (stored dropped probabilities) at T <= 64."""
    code = ("import sys\nsys.path[:0] = [%r, %r]\nimport test_train_parity as t\n"
            "for name in t.FALLBACK_CASES:\n    t.check_train_case(name)\nprint('FALLBACK_OK')\n"
            % (os.path.join(ROOT, "tests"), ROOT))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, **env),
                       cwd=ROOT, timeout=900)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "FALLBACK_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


# ---- 4. TrainStep under CUDA-graph replay (what bench.py times) ----------------------------------------------------
def test_train_step_graph_replay_against_masked_oracle():
    """TrainStep (fused loss, flat gradient bucket, one CUDA graph per step) at p = 0.2: every step consumes exactly one
    counter value, draws new masks, and its gradient bucket and loss equal the float64 oracle at the pre-step
    parameters under that step's masks and gates."""
    from raindrop_b200.train import TrainStep
    cfg = model_config("P19", dropout=P)
    B = 16
    model = build_dropin(cfg, 4).train()
    model._prepare(torch.device("cuda")).obprop_mode = EXACT
    ts = TrainStep(model, B, lr=1e-3, use_graph=True)
    plan = ts.plan
    keys = [k for k, _ in plan.fields]
    params = model.used_parameters()
    prev = None
    for it in range(4):
        batch = make_batch(cfg, B, seed=30 + it)
        ts.load_batch(to_dev(batch))
        p_before = ts.flat_p.clone()
        rng = tuple(plan.rng_state.tolist())
        ts.step()
        torch.cuda.synchronize()
        assert ts.graph is not None
        assert tuple(plan.rng_state.tolist()) == (rng[0], rng[1] + 1), (it, rng, plan.rng_state.tolist())
        assert _ws_rng(ts.dims, ts.ws) == rng
        sd = {k: p_before[off:off + p.numel()].view(p.shape).cpu() for k, p, off in zip(keys, params, ts.offsets)}
        ref, masks = oracle_train(cfg, batch, 4, rng, params=sd, gates=read_gpu(cfg, ts.dims, ts.ws)["gates"])
        check_masks(masks, P)
        assert all(n <= max(1, GATE_RATE[EXACT] * g) for n, g in ref["gate_dis"].values()), ref["gate_dis"]
        if prev is not None:
            assert not np.array_equal(masks["lift"], prev["lift"])
            assert not np.array_equal(masks["layers"][0]["attn"], prev["layers"][0]["attn"])
        prev = masks
        errs = {"loss": abs(ts.loss.item() - ref["loss"]) / max(1.0, abs(ref["loss"]))}
        assert errs["loss"] < TIGHT, (it, ts.loss.item(), ref["loss"])
        for k, p, off in zip(keys, params, ts.offsets):
            errs[k] = normwise(ts.flat_g[off:off + p.numel()].view(p.shape), ref["grads"][k])
            assert errs[k] < TIGHT, (it, k, errs[k])
        print("TrainStep step", it, "rng", rng, "worst", max(errs.items(), key=lambda kv: kv[1]))
