"""GPU: the training step at the production batch sizes -- the P19 step bench.py times (B = 128, dropout 0.2, TrainStep's
CUDA graph), P12 B = 32, PAM B = 256 and LARGE B = 512 -- against a float64 oracle that replays both the kernels'
dropout masks and their ReLU decisions.

A pre-activation within rounding distance of zero can land on either side of its ReLU, and one such gate moves a
gradient by up to 10 % normwise.  A full-size batch has millions of gates, so some always lie that close.  The oracle
therefore takes the GPU's own decisions (RaindropV2Oracle.forward_dense(gates=...)), read from the workspace after the
step: H1 > 0 (ob-prop layer 1), the obs columns of the encoder input > 0 (layer 2), each layer's FFN activation
RD_WS_FFN + l > 0, and the head's hidden activation RD_WS_HEAD_HIDDEN > 0.  Around those decisions the model is a
smooth function, so only rounding separates the two results and every tensor is held near fp32 accuracy.  Replay cannot
hide a wrong forward: at each site the gates where the GPU disagrees with the oracle's own sign are counted and bounded.

The masks are built on the device (rd_debug_dropout_mask, pinned bitwise to oracle/dropout_masks.py by
test_train_parity) and spot-checked against numpy at 10^4 indices per site, the last index included.  The oracle runs in
float64 on the GPU, a chunk of samples at a time.

Bounds (normwise = max|delta| / max|ref|, per tensor), measured on an H100 80GB HBM3 at 700 W:
  * every tensor TIGHT (1e-4): logits, loss, H1 (exact mode), the encoder input and output, every parameter gradient
    and the input gradients.  Measured at most 1.0e-5 at P19 and P12 and 3.5e-5 at PAM, except the tensors WIDE
    names, whose reductions are long; their bound is about 10x the worst of the class:
      - LARGE, both modes, the encoder and ob-prop parameter gradients: sums over T*B = 131072 tokens or B*N = 65536
        rows in fp32 accumulators (grouped weight-gradient kernel: about 26k rows per split).  Measured 2.9e-4
        (in_proj_weight), 1.6e-4 (linear2.weight), 1.05e-4 (layer-1 lin_value.weight).  The head gradients (sums over
        B = 512), logits, loss and input gradients stay TIGHT.
      - PAM, exact mode, the ob-prop lin_value gradients (C = 2400): 3.5e-5.
      - single-pass mode, the ob-prop backward (lin_value gradients, d_src): it rounds fp32 gradients to TF32, and some
        land on the other side of a rounding boundary than the float64 ones.  Measured P19 1.9e-4, P12 9.3e-5, PAM
        1.2e-4, LARGE 4.4e-4 (all d_src).
  * single-pass mode is held against the float64 TF32 rounding model (oracle `tf32_model=True`) with the gates replayed
    and the GPU's rounded layer-1 output fed to layer 2 (`h1_value`).  That H1 is itself checked against the rounding
    model's own (`stages["h1_own"]`): every GPU value TF32-representable, and at most H1_ULP_RATE of the elements one,
    and more than one, TF32 ulp away (3x the worst measured, PAM: 1.1e-2 and 1.1e-3; P19 4e-4 and 7e-5; an element
    more than an ulp off is a small output computed with cancellation).  Against plain float64: logits and the encoder
    input normwise FWD_SANITY (measured 4.2e-4), logits and gradients relative L2 FAST_SANITY (measured 4.2e-4).
  * Adam: element-wise against float64 Adam with the kernel's fp32 constants applied to the GPU's own gradient, to a few
    fp32 spacings.
  * gate disagreements per site: GATE_RATE_EXACT (1e-4) in exact mode, GATE_RATE_FAST in single-pass mode.  Worst
    measured rate: exact 3.0e-6 (LARGE, FFN: 644 of 2.1e8), single-pass 1.8e-6 (LARGE, FFN: 396 of 2.1e8); the bound
    allows one disagreement per site whatever the rate.
  * DP-SGD at P19 B = 128 (measured 8.6e-6 on the norms, 8.9e-6 on the bucket): TIGHT.  The B = 3880 eval forward
    (logits, H1 or its ulp rates, encoder input; measured at most 2.8e-6): EVAL_BOUND, and its gate disagreements at
    all four sites.
The whole file takes about 70 s on that GPU.  The float64 oracle runs a chunk of samples at a time and peaks at
1.8 GB above what the step and its masks hold (17 GB at LARGE B = 512).
"""
import ctypes as C
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import re

from helpers import (GATE_SITES, build_dropin, gate_disagreements, h1_ulp_ok, normwise, read_gpu, rel_l2,
                     tf32_ulp_distance, to_dev, ws_view)
from oracle import dropout_masks as DM
from raindrop_b200 import lib as L
from raindrop_b200.synth import make_batch, model_config, synth_weights, used_param_keys

pytestmark = pytest.mark.gpu
torch.backends.cuda.matmul.allow_tf32 = False     # the float64 oracle must not pick up TF32 anywhere

EXACT, FAST = 2, 1
MODES = {EXACT: "exact", FAST: "fast"}
P = 0.2
RNG0 = (0x2B7E151628AED2A6, (1 << 32) + 7)
WSEED = 4
TIGHT = 1e-4
# Every tensor is held to TIGHT except these, whose reductions are long (module docstring): (configs, modes, tensor
# name pattern, bound), about 10x the worst measured
LONG_PARAM_GRADS = r"^(transformer_encoder|ob_propagation)"
OBPROP_BWD = r"(lin_value\.(weight|bias)|d_src)$"
WIDE = [
    (("LARGE",), (EXACT, FAST), LONG_PARAM_GRADS, 3e-3),
    (("PAM",), (EXACT,), r"lin_value\.(weight|bias)$", 4e-4),
    (("P19",), (FAST,), OBPROP_BWD, 2e-3),
    (("P12",), (FAST,), OBPROP_BWD, 1e-3),
    (("PAM",), (FAST,), OBPROP_BWD, 1.5e-3),
    (("LARGE",), (FAST,), OBPROP_BWD, 5e-3),
]
EVAL_BOUND = 3e-5
FAST_SANITY = 5e-3            # single-pass mode against plain float64, relative L2
FWD_SANITY = 1e-3             # single-pass mode against plain float64, normwise: logits and the encoder input
# single-pass mode: rates of layer-1 outputs one, and more than one, TF32 ulp from the rounding model's (module docstring)
H1_ULP_RATE = (3.5e-2, 3.5e-3)
GATE_RATE_EXACT = 1e-4
GATE_RATE_FAST = 2e-5         # about 10x the worst measured, 1.8e-6
STEPS = 3
SPOT = 10000

# name -> (config, B, first_time_zero, samples per oracle chunk)
CASES = {
    "p19_b128": ("P19", 128, False, 128),
    "p19_b129_t0": ("P19", 129, True, 129),     # last M tile of every token-major GEMM ragged; first timestamp 0
    "p12_b32": ("P12", 32, False, 32),
    "pam_b256": ("PAM", 256, False, 8),
    "large_b512": ("LARGE", 512, False, 16),
}


def case_batch(name):
    cfg_name, B, t0, _ = CASES[name]
    cfg = model_config(cfg_name, dropout=P)
    if cfg_name != "P19":
        return cfg, make_batch(cfg, B, seed=500 + B)
    batch = make_batch(cfg, B, seed=500 + B, first_time_zero=t0, zero_sensors=3)
    full = make_batch(cfg, 1, seed=7, full_length=True)
    for k in ("src", "times"):
        batch[k][:, 5] = full[k][:, 0]
    batch["lengths"][5] = full["lengths"][0]
    assert batch["lengths"][5] == cfg["max_len"]
    for b in (0, 17, B - 1):                     # samples of length 1
        batch["lengths"][b] = 1
        batch["times"][1:, b] = 0
        batch["src"][1:, b] = 0
    return cfg, batch


# ---- masks and gates ------------------------------------------------------------------------------------------------
def device_masks(rng, cfg, B):
    """Every mask of one training forward (model_masks layout, float32 on the device) from rd_debug_dropout_mask, each
    site spot-checked against the numpy stream at SPOT indices including its last."""
    lib = L.load()
    r = torch.tensor(rng, dtype=torch.int64, device="cuda")
    gen = np.random.default_rng(B)

    def site(s, n):
        out = torch.empty(n, device="cuda")
        L.check(lib.rd_debug_dropout_mask(r.data_ptr(), s, n, C.c_float(P), out.data_ptr(), L.stream_ptr()),
                "rd_debug_dropout_mask")
        idx = np.concatenate([gen.integers(0, n, SPOT - 1), [n - 1]])
        got = out[torch.from_numpy(idx).cuda()].cpu().numpy()
        assert np.array_equal(got.view(np.uint32), DM.dropout_mask_at(rng[0], rng[1], s, idx, P).view(np.uint32)), s
        return out

    T, N, d_ob, H, nhid = cfg["max_len"], cfg["d_inp"], cfg["d_ob"], cfg["nhead"], cfg["nhid"]
    D, rows = N * d_ob + 16, T * B
    layers = [dict(attn=site(DM.SITE_ATTN + l, B * H * T * T).view(B, H, T, T),
                   resid1=site(DM.SITE_RESID1 + l, rows * D).view(rows, D),
                   ffn=site(DM.SITE_FFN + l, rows * nhid).view(rows, nhid),
                   resid2=site(DM.SITE_RESID2 + l, rows * D).view(rows, D)) for l in range(cfg["nlayers"])]
    return dict(lift=site(DM.SITE_LIFT, rows * N * d_ob).view(T, B, N * d_ob), layers=layers)


def ws_rng(dims, ws):
    return tuple(ws_view(dims, ws, L.WS_RNG).view(torch.int64)[:2].tolist())


def oracle_model(cfg, params=None):
    from oracle.raindrop_oracle import build_oracle_model
    m = build_oracle_model(cfg).eval()              # eval: the replayed masks are the only dropout
    synth_weights(m, cfg, seed=WSEED)
    if params is not None:
        missing, _ = m.load_state_dict(params, strict=False)
        assert not set(params) & set(missing)
    return m.double().cuda()


class Errs:
    """Normwise errors accumulated over chunks (max |delta| and max |ref| per tensor) and bound checks."""

    def __init__(self):
        self.num, self.den, self.direct = {}, {}, {}

    def add(self, name, got, ref):
        got, ref = got.double(), ref.double()
        self.num[name] = max(self.num.get(name, 0.0), float((got - ref).abs().max()))
        self.den[name] = max(self.den.get(name, 0.0), float(ref.abs().max()))

    def set(self, name, e):
        self.direct[name] = e

    def all(self):
        out = {k: self.num[k] / (self.den[k] + 1e-30) for k in self.num}
        out.update(self.direct)
        return out


def tensor_bound(cfg, mode, name):
    for cfgs, modes, pattern, bound in WIDE:
        if cfg["name"] in cfgs and mode in modes and re.search(pattern, name):
            return bound
    return TIGHT


def compare_step(cfg, batch, gpu, params, masks, mode, chunk, gpu_grads, input_grads=None):
    """The oracle at `params` under `masks` with the GPU's gates against one GPU forward / backward: logits, loss, the
    layer-1 output, the encoder input (obs and pe columns) and output (valid positions), every parameter gradient
    (gpu_grads {key: tensor}) and, given input_grads {d_src, d_times, d_static}, the input gradients.  Returns (errors
    {tensor: normwise} of the tight comparison, sanity errors {tensor: (error, bound)} against plain float64 (fast
    mode), gate disagreements {site: (count, gates)}, [H1 elements, 1 TF32 ulp off, more than 1 ulp off] (fast mode))."""
    from oracle.raindrop_oracle import dense_train_chunked
    T, B, N, d_ob = cfg["max_len"], batch["src"].shape[1], cfg["d_inp"], cfg["d_ob"]
    Dm = N * d_ob
    d = to_dev(batch)
    valid = (torch.arange(T, device="cuda")[:, None] < d["lengths"][None, :])          # [T, B]
    errs, dis, ulp, plain_fwd = Errs(), {s: [0, 0] for s in GATE_SITES}, [0, 0, 0, 0], Errs()
    want_in = input_grads is not None

    def on_chunk(sl, st, logits):
        # single-pass mode: layer 2 takes the GPU's H1, so H1 itself is held against the rounding model's own
        if mode == FAST:
            tf32_ulp_distance(gpu["h1"][sl], st["h1_own"], ulp)
        else:
            errs.add("h1", gpu["h1"][sl], st["h1_own"])
        errs.add("obs", gpu["enc_in"][:, sl, :Dm], st["obs"])
        errs.add("pe", gpu["enc_in"][:, sl, Dm:], st["pe"])
        v = valid[:, sl, None]
        errs.add("enc_out", gpu["enc_out"][:, sl] * v, st["enc"] * v)
        gate_disagreements(cfg, gpu["gates"], st, masks, sl, B, dis)

    def run(tf32_model, h1_value=None, cb=None):
        m = oracle_model(cfg, params)
        out = dense_train_chunked(m, d, masks=masks, gates=gpu["gates"], chunk=chunk, tf32_model=tf32_model,
                                  input_grads=want_in, on_chunk=cb, h1_value=h1_value)
        gm = dict(m.named_parameters())
        out["grads"] = {k: gm[k].grad for k in used_param_keys(cfg)}
        return out

    # the tight reference: plain float64 (exact mode) or the float64 TF32 rounding model fed the GPU's rounded H1
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ref = run(mode == FAST, gpu["h1"] if mode == FAST else None, on_chunk)
    print("oracle peak device memory above the GPU step's %.2f GB: %.2f GB" % (
        base / 2 ** 30, (torch.cuda.max_memory_allocated() - base) / 2 ** 30))
    errs.add("logits", gpu["logits"], ref["logits"])
    errs.set("loss", abs(gpu["loss"] - ref["loss"]) / max(1.0, abs(ref["loss"])))
    for k in used_param_keys(cfg):
        errs.add(k, gpu_grads[k], ref["grads"][k])
    if want_in:
        v = valid.double()
        assert torch.all(input_grads["d_src"][:, :, N:] == 0)
        errs.add("d_src", input_grads["d_src"][:, :, :N], ref["d_src"][:, :, :N])
        errs.add("d_times", input_grads["d_times"] * v, ref["d_times"] * v)
        if ref["d_static"] is not None:
            errs.add("d_static", input_grads["d_static"], ref["d_static"])
    sanity = {}
    if mode == FAST:
        plain = run(False, cb=lambda sl, st, lg: plain_fwd.add("obs", gpu["enc_in"][:, sl, :Dm], st["obs"]))
        plain_fwd.add("logits", gpu["logits"], plain["logits"])
        sanity.update({k + " (normwise)": (e, FWD_SANITY) for k, e in plain_fwd.all().items()})
        sanity["logits"] = (rel_l2(gpu["logits"], plain["logits"]), FAST_SANITY)
        sanity.update({k: (rel_l2(gpu_grads[k], plain["grads"][k]), FAST_SANITY) for k in used_param_keys(cfg)})
        if want_in:
            sanity["d_src"] = (rel_l2(input_grads["d_src"][:, :, :N], plain["d_src"][:, :, :N]), FAST_SANITY)
    return errs.all(), sanity, {s: tuple(v) for s, v in dis.items()}, ulp


def check_bounds(tag, cfg, errs, sanity, dis, ulp, mode, bad):
    rate = GATE_RATE_EXACT if mode == EXACT else GATE_RATE_FAST
    top = sorted(errs.items(), key=lambda kv: -kv[1])[:6]
    print("%s mode=%s worst %s%s gate disagreements %s%s" % (
        tag, MODES[mode], ", ".join("%s %.2e" % kv for kv in top),
        (", sanity worst %s %.3e" % max(((k, e) for k, (e, _) in sanity.items()), key=lambda kv: kv[1])) if sanity else "",
        " ".join("%s %d/%d" % (s, n, g) for s, (n, g) in dis.items()),
        (", H1 TF32 ulp off: 1 ulp %d, more %d of %d, not TF32 %d" % (ulp[1], ulp[2], ulp[0], ulp[3]))
        if mode == FAST else ""))
    bad += [(tag, MODES[mode], k, e) for k, e in errs.items() if not e < tensor_bound(cfg, mode, k)]
    bad += [(tag, MODES[mode], "sanity " + k, e) for k, (e, tol) in sanity.items() if not e < tol]
    bad += [(tag, MODES[mode], "gates " + s, n, g) for s, (n, g) in dis.items() if n > max(1, rate * g)]
    if mode == FAST and not h1_ulp_ok(ulp, H1_ULP_RATE):
        bad.append((tag, MODES[mode], "H1 TF32 ulp", ulp))


# ---- 1. the bench path: TrainStep under CUDA-graph replay -----------------------------------------------------------
def train_step_case(name, mode):
    from raindrop_b200.train import TrainStep
    cfg, batch = case_batch(name)
    chunk = CASES[name][3]
    B = batch["src"].shape[1]
    model = build_dropin(cfg, WSEED).train()
    plan = model._prepare(torch.device("cuda"))
    plan.obprop_mode = mode
    plan.rng_state.copy_(torch.tensor(RNG0, dtype=torch.int64))
    lr, (b1, b2), eps = 1e-3, (0.9, 0.999), 1e-8
    ts = TrainStep(model, B, lr=lr, betas=(b1, b2), eps=eps, use_graph=True)
    keys = [k for k, _ in ts.plan.fields]
    params = model.used_parameters()
    ts.load_batch(to_dev(batch))
    bad = []
    for it in range(STEPS):
        p0, m0, v0 = ts.flat_p.clone(), ts.exp_avg.clone(), ts.exp_avg_sq.clone()
        t = int(ts.step_count[0]) + 1
        rng = tuple(plan.rng_state.tolist())
        ts.step()
        torch.cuda.synchronize()
        assert ts.graph is not None and ws_rng(ts.dims, ts.ws) == rng
        assert tuple(plan.rng_state.tolist()) == (rng[0], rng[1] + 1)
        gpu = read_gpu(cfg, ts.dims, ts.ws)
        gpu.update(logits=ts.logits.clone(), loss=ts.loss.item())
        grads = {k: ts.flat_g[off:off + p.numel()].view(p.shape) for k, p, off in zip(keys, params, ts.offsets)}
        sd = {k: p0[off:off + p.numel()].view(p.shape).cpu() for k, p, off in zip(keys, params, ts.offsets)}
        masks = device_masks(rng, cfg, B)
        errs, sanity, dis, ulp = compare_step(cfg, batch, gpu, sd, masks, mode, chunk, grads)
        del masks
        check_bounds("TrainStep %s step %d" % (name, it), cfg, errs, sanity, dis, ulp, mode, bad)
        # Adam, element-wise: float64 arithmetic on the GPU's own gradient from the pre-step state, with the kernel's fp32
        # constants; the parameter update from the GPU's own new moments
        f32 = np.float32
        b1f, b2f, epsf, lrf = (float(f32(x)) for x in (b1, b2, eps, lr))
        bc1, bc2s = float(f32(1 - b1f ** t)), float(f32((1 - b2f ** t) ** 0.5))
        g = ts.flat_g.double()
        m = b1f * m0.double() + float(f32(1) - f32(b1)) * g
        v = b2f * v0.double() + float(f32(1) - f32(b2)) * g * g
        upd = (lrf / bc1) * ts.exp_avg.double() / (ts.exp_avg_sq.double().sqrt() / bc2s + epsf)
        spacing = lambda x: torch.from_numpy(np.spacing(np.abs(x.float().cpu().numpy()))).cuda().double()
        # one fp32 spacing per rounding of the largest term of each expression
        checks = (("exp_avg", ts.exp_avg, m, 2 * spacing(b1f * m0.double().abs() + (1 - b1f) * g.abs())),
                  ("exp_avg_sq", ts.exp_avg_sq, v, 3 * spacing(b2f * v0.double() + (1 - b2f) * g * g)),
                  ("param", ts.flat_p, p0.double() - upd, spacing(p0.double().abs() + upd.abs()) + 8 * spacing(upd)))
        for what, got, want, tol in checks:
            n_out = int(((got.double() - want).abs() > tol).sum())
            if n_out:
                bad.append(("TrainStep %s step %d" % (name, it), MODES[mode], "adam " + what, n_out))
    return bad


@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
@pytest.mark.parametrize("name", list(CASES))
def test_train_step_against_gate_replaying_oracle(name, mode):
    """Three CUDA-graph replays of TrainStep: logits, loss, encoder input and output, every field of the gradient bucket
    against the oracle at the pre-step parameters with that step's masks and gates; the Adam update element-wise."""
    t0 = time.time()
    bad = train_step_case(name, mode)
    print("%s %s: %.1f s, peak device memory %.2f GB" % (name, MODES[mode], time.time() - t0,
                                                         torch.cuda.max_memory_allocated() / 2 ** 30))
    assert not bad, bad


# ---- 2. input gradients through the module's autograd path ----------------------------------------------------------
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
@pytest.mark.parametrize("name", ["p19_b128", "p12_b32", "pam_b256", "large_b512"])
def test_input_grads_against_gate_replaying_oracle(name, mode):
    """One training forward / backward of the module with src, times and static requiring grad: d_src (value half),
    d_times (valid rows) and d_static, with the parameter gradients, against the gate-replaying oracle."""
    cfg, batch = case_batch(name)
    B = batch["src"].shape[1]
    model = build_dropin(cfg, WSEED).train()
    plan = model._prepare(torch.device("cuda"))
    plan.obprop_mode = mode
    plan.rng_state.copy_(torch.tensor(RNG0, dtype=torch.int64))
    plan.debug_keep_workspace = True
    d = to_dev(batch)
    src = d["src"].clone().requires_grad_(True)
    times = d["times"].clone().requires_grad_(True)
    static = None if d["static"] is None else d["static"].clone().requires_grad_(True)
    logits, _, _ = model.forward(src, static, times, d["lengths"])
    loss = F.cross_entropy(logits, d["y"])
    loss.backward()
    torch.cuda.synchronize()
    assert ws_rng(plan.last_dims, plan.last_workspace) == RNG0
    gpu = read_gpu(cfg, plan.last_dims, plan.last_workspace)
    gpu.update(logits=logits.detach(), loss=loss.item())
    gp = dict(model.named_parameters())
    masks = device_masks(RNG0, cfg, B)
    errs, sanity, dis, ulp = compare_step(cfg, batch, gpu, None, masks, mode, CASES[name][3],
                                     {k: gp[k].grad for k in used_param_keys(cfg)},
                                     dict(d_src=src.grad, d_times=times.grad, d_static=None if static is None else static.grad))
    bad = []
    check_bounds("module %s" % name, cfg, errs, sanity, dis, ulp, mode, bad)
    assert not bad, bad


# ---- 3. DP-SGD at the size its timings were taken -------------------------------------------------------------------
def test_dp_sgd_at_p19_b128_against_gate_replaying_oracle():
    """per_sample_grad_sqnorms against the float64 per-sample gradient norms under replayed masks and gates, per entry
    to TIGHT relative; DPTrainStep's clipped bucket (noise 0) against sum_b c_b g_b / L."""
    from raindrop_b200 import privacy as PV
    cfg, batch = case_batch("p19_b128")
    B = batch["src"].shape[1]
    d = to_dev(batch)

    def fresh():
        model = build_dropin(cfg, WSEED).train()
        plan = model._prepare(torch.device("cuda"))
        plan.obprop_mode = EXACT
        plan.rng_state.copy_(torch.tensor(RNG0, dtype=torch.int64))
        return model, plan

    # the gates: a training forward at the same (seed, step), dims and arithmetic as the norm pass's, so bitwise the same
    model, plan = fresh()
    plan.debug_keep_workspace = True
    with torch.no_grad():
        model.forward(d["src"], d["static"], d["times"], d["lengths"])
    torch.cuda.synchronize()
    gates = read_gpu(cfg, plan.last_dims, plan.last_workspace)["gates"]
    model, plan = fresh()
    sq = PV.per_sample_grad_sqnorms(model, d["src"], d["static"], d["times"], d["lengths"], d["y"]).double().cpu().numpy()
    keys = PV.sqnorm_fields(model)
    # float64 per-sample gradients under the same masks and gates
    oracle = oracle_model(cfg)
    masks = device_masks(RNG0, cfg, B)
    st = None if d["static"] is None else d["static"].double()
    logits, _, _ = oracle.forward_dense(d["src"].double(), st, d["times"].double(), d["lengths"], masks=masks, gates=gates)
    prm = dict(oracle.named_parameters())
    ref_sq, ref_g = np.empty((B, len(keys))), []
    for b in range(B):
        gs = torch.autograd.grad(F.cross_entropy(logits[b:b + 1], d["y"][b:b + 1]), [prm[k] for k in keys],
                                 retain_graph=True)
        ref_sq[b] = [float(g.pow(2).sum()) for g in gs]
        ref_g.append(gs)
    rel = np.abs(sq - ref_sq) / np.maximum(ref_sq, 1e-300)
    worst = np.unravel_index(np.argmax(rel), rel.shape)
    print("dp p19_b128 sqnorms worst relative %.3e (sample %d, %s)" % (rel[worst], worst[0], keys[worst[1]]))
    bad = [(b, keys[f], sq[b, f], ref_sq[b, f]) for b, f in zip(*np.nonzero(~(rel <= TIGHT)))][:10]
    # the clipped bucket
    norms = np.sqrt(ref_sq.sum(1))
    Cn = float(np.median(norms)) * 0.5
    L_ = float(B) + 3.0
    model, plan = fresh()
    step = PV.DPTrainStep(model, B, max_grad_norm=Cn, noise_multiplier=0.0, expected_batch_size=L_, use_graph=False)
    step.load_batch(d)
    step.step()
    torch.cuda.synchronize()
    c = np.minimum(1.0, Cn / (norms + 1e-6))
    np.testing.assert_allclose(step.clip_factors.cpu().numpy(), c, rtol=TIGHT)
    errs = {}
    for i, k in enumerate(keys):
        ref = sum(float(c[b]) * ref_g[b][i] for b in range(B)) / L_
        off = step.offsets[i]
        errs[k] = normwise(step.flat_g[off:off + ref.numel()].view(ref.shape), ref)
    w = max(errs.items(), key=lambda kv: kv[1])
    print("dp p19_b128 clipped bucket worst %s %.3e" % w)
    bad += [(k, e) for k, e in errs.items() if not e < TIGHT]
    assert not bad, bad


# ---- 4. the whole validation set in one eval forward ----------------------------------------------------------------
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
def test_whole_validation_set_logits_against_oracle(mode):
    """evaluate_standard's one batch of B = 3880 (P19): logits, the layer-1 output and the encoder input against the
    oracle with the GPU's gates (plain float64 in exact mode, the TF32 rounding model in single-pass mode), and the gate
    disagreements of all four sites (every FFN gate counts: eval has no mask)."""
    cfg = model_config("P19", dropout=P)
    B, T, Dm = 3880, cfg["max_len"], cfg["d_inp"] * cfg["d_ob"]
    batch = make_batch(cfg, B, seed=9)
    d = to_dev(batch)
    model = build_dropin(cfg, WSEED).eval()
    model._plan.obprop_mode = mode
    model._plan.debug_keep_workspace = True
    with torch.no_grad():
        logits, _, _ = model.forward(d["src"], d["static"], d["times"], d["lengths"])
    gpu = read_gpu(cfg, model._plan.last_dims, model._plan.last_workspace)
    oracle = oracle_model(cfg)
    no_masks = dict(lift=None, layers=[{} for _ in range(cfg["nlayers"])])       # eval: written-out layers, no dropout
    errs, dis, ulp = Errs(), {s: [0, 0] for s in GATE_SITES}, [0, 0, 0, 0]
    with torch.no_grad():
        for b0 in range(0, B, 1024):
            sl = slice(b0, min(B, b0 + 1024))
            g = dict(h1=gpu["gates"]["h1"][sl], obs=gpu["gates"]["obs"][:, sl], head=gpu["gates"]["head"][sl],
                     ffn=[f.view(T, B, -1)[:, sl].reshape(-1, f.shape[-1]) for f in gpu["gates"]["ffn"]])
            st = {}
            out, _, _ = oracle.forward_dense(d["src"][:, sl].double(), d["static"][sl].double(), d["times"][:, sl].double(),
                                             d["lengths"][sl], stages=st, tf32_model=mode == FAST, masks=no_masks, gates=g,
                                             h1_value=gpu["h1"][sl] if mode == FAST else None)
            errs.add("logits", logits[sl], out)
            errs.add("obs", gpu["enc_in"][:, sl, :Dm], st["obs"])
            errs.add("pe", gpu["enc_in"][:, sl, Dm:], st["pe"])
            if mode == FAST:
                tf32_ulp_distance(gpu["h1"][sl], st["h1_own"], ulp)
            else:
                errs.add("h1", gpu["h1"][sl], st["h1_own"])
            gate_disagreements(cfg, gpu["gates"], st, no_masks, sl, B, dis)
    e = errs.all()
    print("eval B=3880 mode=%s %s gate disagreements %s H1 TF32 ulp off %s" % (
        MODES[mode], ", ".join("%s %.2e" % kv for kv in e.items()), dis, ulp if mode == FAST else "-"))
    rate = GATE_RATE_EXACT if mode == EXACT else GATE_RATE_FAST
    assert all(v < EVAL_BOUND for v in e.values()), e
    assert all(n <= max(1, rate * g) for n, g in dis.values()), dis
    assert mode == EXACT or h1_ulp_ok(ulp, H1_ULP_RATE), ulp
