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

Bounds (normwise = max|delta| / max|ref|, as in test_gpu_parity.py):
  * error-compensated ob-prop mode: the eval-mode bounds, every tensor normwise (gradients 2e-3, 1e-2 for C >= 1024).
    Measured on an H100: 2e-6 .. 1e-5 in every case but two.  At PAM B = 2 one of 81600 layer-2 ob-prop
    pre-activations lies within 1e-6 of zero and rounds to the other side of the ReLU (fp64 1.0e-6, kernel 0); with 34
    rows that one gate moves the layer-2 lin_value gradient by 9e-2 normwise, 4.5e-3 in relative L2 (LARGE B = 2, also
    one gate: 9.5e-3 normwise, 1.9e-3 relative L2).  So the test counts the ob-prop
    gates whose state differs from the float64 oracle (read from H1 and the encoder input); where there are any, the
    four lin_value gradients and d_src are held in relative L2 to the same bound, and the count itself is bounded.
  * single-pass TF32 mode: relative L2 5e-2 against the float64 oracle, and normwise 5e-3 (lin_value: relative L2 5e-2)
    against the oracle evaluated under the kernels' TF32 rounding model with the same masks (`tf32_model=True`), as
    test_against_oracle does in eval mode.  The eval-mode normwise 2e-2 against fp32 is not used: with dropout, the
    encoder's first FFN gate flips that the forward's TF32 error causes show up as 2.5e-2 .. 4.8e-2 normwise in
    linear1 (TINY8 B = 9, LARGE B = 2, random shape 0) while the same gradients agree with the rounding model to
    3e-6 .. 3.4e-3.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import build_dropin, normwise, random_shape_case, rel_l2, to_dev
from oracle import dropout_masks as DM
from raindrop_b200.synth import make_batch, model_config, synth_weights, used_param_keys

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXACT, FAST = 2, 1
P = 0.2
# seed and step counter with both 32-bit halves non-zero: every word of the Philox key and counter takes part
RNG0 = (0x2B7E151628AED2A6, (1 << 32) + 7)
LOGIT_TOL_EXACT, FWD_TOL = 1e-4, 1e-3
GRAD_TOL_EXACT, GRAD_TOL_EXACT_WIDE = 2e-3, 1e-2
GRAD_TOL, L2_TOL_FAST = 2e-2, 5e-2
MODEL_TOL = 5e-3              # single-pass TF32 mode vs the oracle under the kernels' rounding model
MAX_GATE_FLIP_RATE = 1e-4     # ob-prop ReLU gates allowed to differ from the float64 oracle (error-compensated mode)

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


def _exact_tol(cfg):
    return GRAD_TOL_EXACT_WIDE if cfg["max_len"] * cfg["d_ob"] >= 1024 else GRAD_TOL_EXACT


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


def oracle_train(cfg, batch, weight_seed, rng, p=P, params=None):
    """float64 train-mode reference under the masks of (seed, step) = rng.  `params` ({key: tensor}) overrides the
    synthetic weights.  Returns (reference dict, masks)."""
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
    logits, _, _ = oracle.forward_dense(src, static, times, batch["lengths"], stages=stages, masks=masks)
    loss = F.cross_entropy(logits, batch["y"])
    loss.backward()
    go = dict(oracle.named_parameters())
    ref = dict(logits=logits.detach(), loss=loss.item(), obs=stages["obs"].detach(), pe=stages["pe"].detach(),
               h1=stages["h1"].detach(), grads={k: go[k].grad for k in used_param_keys(cfg)}, d_src=src.grad,
               d_times=times.grad, d_static=None if static is None else static.grad)
    return ref, masks


def oracle_tf32_grads(cfg, batch, weight_seed, masks):
    """Parameter gradients of the fp32 oracle under the kernels' TF32 rounding model (single-pass ob-prop mode)."""
    from oracle.raindrop_oracle import build_oracle_model
    oracle = build_oracle_model(cfg).eval()
    synth_weights(oracle, cfg, seed=weight_seed)
    logits, _, _ = oracle.forward_dense(batch["src"], batch["static"], batch["times"], batch["lengths"], tf32_model=True,
                                        masks=masks)
    F.cross_entropy(logits, batch["y"]).backward()
    go = dict(oracle.named_parameters())
    return {k: go[k].grad for k in used_param_keys(cfg)}


def gpu_train(cfg, batch, weight_seed, mode, rng=RNG0):
    """One training forward + cross-entropy + backward of the drop-in with parameter and input gradients."""
    from raindrop_b200 import functional as RF
    from raindrop_b200 import lib as L
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
    T, B, N = src.shape[0], src.shape[1], cfg["d_inp"]
    D = N * cfg["d_ob"] + 16
    gp = dict(model.named_parameters())
    return dict(logits=logits.detach(), loss=loss.item(), enc_in=RF.workspace_view(plan, L.WS_ENC_IN).view(T, B, D),
                h1=RF.workspace_view(plan, L.WS_H1).view(B, N, -1), grads={k: gp[k].grad for k in used_param_keys(cfg)},
                d_src=src.grad, d_times=times.grad, d_static=None if static is None else static.grad)


def gate_flips(cfg, got, ref):
    """(number of ob-prop ReLU gates, layer 1 and 2, whose state differs from the oracle, number of gates)."""
    D4 = cfg["d_inp"] * cfg["d_ob"]
    h1, obs = got["h1"].cpu(), got["enc_in"][:, :, :D4].cpu()
    n = int(((h1 == 0) != (ref["h1"] == 0)).sum()) + int(((obs == 0) != (ref["obs"] == 0)).sum())
    return n, h1.numel() + obs.numel()


def compare(cfg, batch, got, ref, mode, ref_tf32=None):
    """Errors under the bounds of the module docstring: returns ({tensor: error}, [(tensor, error, bound) out of
    bounds]).  `ref_tf32` = oracle_tf32_grads (single-pass TF32 mode)."""
    exact = mode == EXACT
    errs, bad = {}, []

    def chk(name, e, tol):
        errs[name] = e
        if not e < tol:
            bad.append((name, e, tol))

    N, D4 = cfg["d_inp"], cfg["d_inp"] * cfg["d_ob"]
    chk("logits", normwise(got["logits"], ref["logits"]), LOGIT_TOL_EXACT if exact else FWD_TOL)
    chk("loss", abs(got["loss"] - ref["loss"]) / max(1.0, abs(ref["loss"])), LOGIT_TOL_EXACT if exact else FWD_TOL)
    chk("obs", normwise(got["enc_in"][:, :, :D4], ref["obs"]), 1e-4 if exact else FWD_TOL)
    chk("pe", normwise(got["enc_in"][:, :, D4:], ref["pe"]), 1e-5)
    flips, gates = gate_flips(cfg, got, ref)
    if exact and flips > max(1, MAX_GATE_FLIP_RATE * gates):
        bad.append(("ob-prop gate flips", flips, gates))
    # a flipped ob-prop gate moves whole rows of the lin_value gradients and of d_src: relative L2 there
    flipped = exact and flips > 0
    metric = rel_l2 if flipped else normwise
    for k in used_param_keys(cfg):
        g, r = got["grads"][k], ref["grads"][k]
        assert g is not None, k
        if exact:
            chk(k, (metric if "lin_value" in k else normwise)(g, r), _exact_tol(cfg))
        else:
            chk(k, rel_l2(g, r), L2_TOL_FAST)
            if "lin_value" in k:
                chk(k + " (tf32 model)", rel_l2(g, ref_tf32[k]), L2_TOL_FAST)
            else:
                chk(k + " (tf32 model)", normwise(g, ref_tf32[k]), MODEL_TOL)
    assert torch.all(got["d_src"][:, :, N:] == 0)
    valid = (torch.arange(cfg["max_len"])[:, None] < batch["lengths"][None, :]).to(got["d_times"].device)
    d_times, d_times_ref = got["d_times"] * valid, ref["d_times"] * valid.cpu()
    if exact:
        chk("d_src", metric(got["d_src"][:, :, :N], ref["d_src"][:, :, :N]), _exact_tol(cfg))
        chk("d_times", normwise(d_times, d_times_ref), _exact_tol(cfg))
    else:
        chk("d_src", rel_l2(got["d_src"][:, :, :N], ref["d_src"][:, :, :N]), L2_TOL_FAST)
        chk("d_times", rel_l2(d_times, d_times_ref), L2_TOL_FAST)
    if ref["d_static"] is not None:
        chk("d_static", normwise(got["d_static"], ref["d_static"]), _exact_tol(cfg) if exact else GRAD_TOL)
    return errs, bad


def check_train_case(name, modes=(EXACT, FAST)):
    cfg, batch, wseed = case_setup(name)
    ref, masks = oracle_train(cfg, batch, wseed, RNG0)
    check_masks(masks, P)
    ref_tf32 = oracle_tf32_grads(cfg, batch, wseed, masks) if FAST in modes else None
    bad = []
    for mode in modes:
        got = gpu_train(cfg, batch, wseed, mode)
        errs, b = compare(cfg, batch, got, ref, mode, ref_tf32)
        worst = max(errs.items(), key=lambda kv: kv[1])
        tag = "exact" if mode == EXACT else "fast"
        print("train-mode parity %-12s %s B=%d mode=%s worst %s %.3e, ob-prop gate flips %d of %d" %
              ((name, cfg["name"], batch["src"].shape[1], tag) + worst + gate_flips(cfg, got, ref)))
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
    parameters under that step's masks."""
    from raindrop_b200.train import TrainStep
    cfg = model_config("P19", dropout=P)
    B = 16
    model = build_dropin(cfg, 4).train()
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
        ref, masks = oracle_train(cfg, batch, 4, rng, params=sd)
        check_masks(masks, P)
        if prev is not None:
            assert not np.array_equal(masks["lift"], prev["lift"])
            assert not np.array_equal(masks["layers"][0]["attn"], prev["layers"][0]["attn"])
        prev = masks
        errs = {"loss": abs(ts.loss.item() - ref["loss"]) / max(1.0, abs(ref["loss"]))}
        assert errs["loss"] < LOGIT_TOL_EXACT, (it, ts.loss.item(), ref["loss"])
        for k, p, off in zip(keys, params, ts.offsets):
            errs[k] = normwise(ts.flat_g[off:off + p.numel()].view(p.shape), ref["grads"][k])
            assert errs[k] < GRAD_TOL_EXACT, (it, k, errs[k])
        print("TrainStep step", it, "rng", rng, "worst", max(errs.items(), key=lambda kv: kv[1]))
