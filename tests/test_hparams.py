"""Raindrop_v2 across its constructor's hyper-parameters: d_ob, nhead, nhid and up to RD_MAX_LAYERS = 8 encoder layers.

Every other parity test builds d_ob = 4, nhead = 2, nhid = 2 d_model and at most 3 layers, so D = N d_ob + 16 and nhid
are always multiples of 4.  Many dispatch decisions of the CUDA path depend on exactly these four numbers.  The named
cases below each reach a distinct set of kernels; `test_kernel_coverage` asserts that they still do.

  case  N, d_ob -> D   nhead (hd)  nhid  layers  T    statics, classes, B   reaches
  A     12, 3 -> 52    4 (13)      50    5       40   4, 3, 9               attn_small with D % 4 == 0 but hd odd;
        linear1/2 on the CUDA cores next to tensor-core in/out_proj (dropout1 keep bits and dropout2 from Philox in one
        layer's LayerNorm backward); CUDA-core and grouped weight gradients together; two weight-prep launches; ob-prop
        layer 2 on the CUDA cores (permuted store) and the generic-d_ob lift and obprop_out_grad
  B     8, 2 -> 32     8 (4)       64    8       48   -, 2, 6               attn_tc at hd = 4; 32 grouped weight gradients
        (flushes in the middle of the encoder); three weight-prep launches
  C     10, 1 -> 26    2 (13)      37    3       130  2, 4, 3               D % 4 != 0: scalar LayerNorm, every encoder GEMM
        on the CUDA cores, the head's scalar masked mean; C = 130, so the whole ob-prop runs on the CUDA cores; batched
        attention
  D     40, 16 -> 656  4 (164)     100   1       20   3, 2, 4               D > 640: the non-fused LayerNorm with tensor-core
        keep bits; batched attention at short T (hd > 96); Df = 696, close to the head backward's 722
  E     20, 4 -> 96    1 (96)      200   4       64   5, 5, 5               attn_tc at hd = 96 and T = 64 together; grouped
        weight-gradient flush with d_ob = 4
  F     11, 4 -> 60    3 (20)      30    2       65   -, 7, 4               T = 65, one past the fused attention;
        nhid % 4 != 0 with the standard ob-prop

A, B and C are also pinned to the reference's own outputs (tests/golden/hparams_<case>.npz, oracle/make_golden.py).

Bounds are those of test_gpu_parity.test_against_oracle (eval) and test_train_parity.compare (train): a training step
replays the kernels' dropout masks and ReLU decisions, so every tensor is held to test_train_parity.TIGHT.
"""
import collections
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import build_dropin, check_against_golden, load_golden, normwise, rel_l2, to_dev
from oracle.make_golden import HPARAM_CASES, hparam_config
from raindrop_b200 import lib as L
from raindrop_b200.synth import make_batch, synth_weights, used_param_keys

EXACT, FAST = 2, 1
P = 0.2
FWD_TOL, GRAD_TOL_EXACT, GRAD_TOL, OBPROP_GRAD_L2, MODEL_TOL = 1e-3, 2e-3, 2e-2, 5e-2, 5e-3
HEAD_BWD_MAX_DF = 722       # (1 + 16 warps) * Df floats of shared memory <= 48 KB (rd_head.cu)

# name -> (hyper-parameters, B, data seed, weight seed)
CASES = dict(HPARAM_CASES)
CASES.update({
    "D": (dict(d_inp=40, d_ob=16, nhead=4, nhid=100, nlayers=1, max_len=20, d_static=3, n_classes=2), 4, 34, 44),
    "E": (dict(d_inp=20, d_ob=4, nhead=1, nhid=200, nlayers=4, max_len=64, d_static=5, n_classes=5), 5, 35, 45),
    "F": (dict(d_inp=11, d_ob=4, nhead=3, nhid=30, nlayers=2, max_len=65, d_static=0, n_classes=7), 4, 96, 46),
})
FIXTURE_CASES = sorted(HPARAM_CASES)


def case_setup(name):
    """(cfg, batch, weight seed) of a named case or of `rnd<seed>` (random_case)."""
    if name.startswith("rnd"):
        return random_case(int(name[3:]))
    hp, B, dseed, wseed = CASES[name]
    cfg = hparam_config(name, hp)
    return cfg, make_batch(cfg, B, seed=dseed), wseed


def random_case(seed):
    """A seeded model drawn wider than helpers.random_shape_case: d_ob 1..5, N 1..40, nhead a random divisor of D,
    nhid 4..3D, 1..8 layers, T 2..200 (above 64 for at least a third of the seeds).  Draws whose training the head
    backward cannot hold (Df > 722) are redrawn."""
    g = torch.Generator().manual_seed(5000 + seed)
    ri = lambda lo, hi: int(torch.randint(lo, hi + 1, (1,), generator=g))
    while True:
        d_ob, N = ri(1, 5), ri(1, 40)
        D = N * d_ob + 16
        divisors = [h for h in range(1, D + 1) if D % h == 0]
        nhead = divisors[ri(0, len(divisors) - 1)]
        static = bool(ri(0, 1))
        ds = ri(1, 6) if static else 0
        if D + (N if static else 0) <= HEAD_BWD_MAX_DF:
            break
    T = ri(65, 200) if seed % 3 == 0 else ri(2, 200)
    B = [1, 2, 3, 4, 5, 7][ri(0, 5)]
    hp = dict(d_inp=N, d_ob=d_ob, nhead=nhead, nhid=ri(4, 3 * D), nlayers=ri(1, 8), max_len=T, d_static=ds,
              n_classes=ri(2, 6))
    cfg = hparam_config("R%d" % seed, hp)
    if ri(0, 1):
        cfg["global_structure"] = (torch.rand(N, N, generator=g) < 0.4).float() * torch.rand(N, N, generator=g)
    return cfg, make_batch(cfg, B, seed=seed, first_time_zero=bool(ri(0, 1))), 60 + seed


RANDOM = ["rnd%d" % s for s in range(12)]


def _oracle(cfg, wseed, dtype=torch.float32):
    from oracle.raindrop_oracle import build_oracle_model
    m = build_oracle_model(cfg).eval()
    synth_weights(m, cfg, seed=wseed)
    return m.to(dtype)


# ---- CPU: the oracle against the reference's own outputs ------------------------------------------------------------
def test_random_cases_are_inside_the_envelope():
    """The sweep really is wide: hyper-parameters the fixed-config tests never build, T > 64 for a third of the seeds."""
    cfgs = [random_case(s)[0] for s in range(12)]
    assert sum(c["max_len"] > 64 for c in cfgs) >= 4
    assert {c["d_ob"] for c in cfgs} != {4} and any((c["d_inp"] * c["d_ob"] + 16) % 4 for c in cfgs)
    assert any(c["nhead"] != 2 for c in cfgs) and any(c["nlayers"] > 3 for c in cfgs) and any(c["nhid"] % 4 for c in cfgs)
    for c in cfgs:
        D = c["d_inp"] * c["d_ob"] + 16
        assert D % c["nhead"] == 0 and 1 <= c["nlayers"] <= 8 and D + (c["d_inp"] if c["static"] else 0) <= HEAD_BWD_MAX_DF


@pytest.mark.parametrize("name", FIXTURE_CASES)
@pytest.mark.parametrize("mode", ["edgewise", "dense"])
def test_oracle_matches_reference_at_hparams(golden_dir, name, mode):
    """oracle/raindrop_oracle.py (the reference the GPU tests below use) equals the reference's own Raindrop_v2 at
    d_ob 1..3, nhead 2..8, nhid not a multiple of 4 and up to 8 layers: bounds of test_oracle_golden.py."""
    z, meta = load_golden(golden_dir, "hparams_" + name)
    cfg, batch, wseed = case_setup(name)
    assert meta["cfg"] == cfg and meta["weight_seed"] == wseed and meta["batch"] == batch["src"].shape[1]
    torch.set_num_threads(8)
    model = _oracle(cfg, wseed)
    stages = {}
    fwd = model.forward if mode == "edgewise" else model.forward_dense
    logits, distance, _ = fwd(batch["src"], batch["static"], batch["times"], batch["lengths"], stages=stages)
    loss = F.cross_entropy(logits, batch["y"])
    loss.backward()
    tol = 1e-6 if mode == "edgewise" else 2e-5
    errs = {}
    assert normwise(logits, z["logits"]) < tol
    assert abs(loss.item() - float(z["loss"])) < tol * max(1.0, abs(float(z["loss"])))
    assert float(distance) == float(z["distance"])
    check_against_golden(z, "obs" in z.files, "obs", stages["obs"], tol, errs)
    check_against_golden(z, "pe" in z.files, "pe", stages["pe"], 1e-7, errs)
    check_against_golden(z, "enc" in z.files, "enc", stages["enc"], tol, errs)
    params = dict(model.named_parameters())
    for k in used_param_keys(cfg):
        check_against_golden(z, "grad." + k in z.files, "grad." + k, params[k].grad, 10 * tol, errs)
    assert sorted(k for k, p in params.items() if p.grad is not None) == sorted(used_param_keys(cfg))
    print(name, mode, "worst", max(errs.items(), key=lambda kv: kv[1]))


def test_more_than_eight_layers_is_refused_on_the_host():
    """RD_MAX_LAYERS = 8: the workspace query (pure host code) refuses 9 layers with a message, so no forward runs."""
    from raindrop_b200 import functional as RF
    lib = L.load()
    ok = RF.Plan(8, 2, 8, 64, 8, 0, 2, 48, 0.2, False).dims(6, True)
    assert lib.rd_workspace_bytes(C.byref(ok)) > 0
    bad = RF.Plan(8, 2, 8, 64, 9, 0, 2, 48, 0.2, False).dims(6, True)
    assert lib.rd_workspace_bytes(C.byref(bad)) == 0
    assert b"nlayers=9" in lib.rd_last_error_string()


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _kernel_counts(step, cycles=2):
    """[{short kernel name: launches}] of `cycles` profiled calls of `step()`, from torch.profiler's CUDA activity.

    A trace can miss records, most of all those at the very start of a profiling session, where this step launches its
    weight-prep kernels.  So each profiled call follows a discarded warm-up call in the same session (the profiler's
    documented warm-up phase), and this is done for `cycles` calls; the caller takes the largest count of each."""
    import json
    import os
    import sys
    import tempfile
    from torch.profiler import ProfilerActivity, profile, schedule
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    from step_kernel_times import short_name
    counts = []

    def ready(prof):
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "trace.json")
            prof.export_chrome_trace(path)
            with open(path) as f:
                evs = json.load(f).get("traceEvents", [])
        counts.append(collections.Counter(short_name(e["name"]) for e in evs
                                          if e.get("cat") == "kernel" and e.get("ph") == "X"))

    with profile(activities=[ProfilerActivity.CUDA], schedule=schedule(wait=0, warmup=1, active=1, repeat=cycles),
                 on_trace_ready=ready) as prof:
        for _ in range(2 * cycles):
            step()
            torch.cuda.synchronize()
            prof.step()
    assert len(counts) == cycles, len(counts)
    return counts


# case -> (kernels that must run, kernels that must not run, {kernel: minimum launches}) in one eager training step
COVERAGE = {
    "A": (["attn_small_fwd_kernel", "attn_small_bwd_kernel", "gemm_f32_kernel", "tc_nt_kernel", "tc_wgrad_kernel",
           "obprop_out_grad_kernel", "lift_posenc_kernel", "layernorm_fwd_vec_kernel", "layernorm_bwd_fused_kernel",
           "head_fwd_kernel<true>"],
          ["attn_tc_fwd_kernel", "obprop_out_grad_vec4_kernel", "layernorm_fwd_kernel"],
          # CUDA-core NT GEMMs: linear1 and linear2 of five layers and ob-prop layer 2 (d_ob = 3, permuted store)
          {"split_weights_kernel": 2, "gemm_f32_kernel<false, true>": 11}),
    "B": (["attn_tc_fwd_kernel", "attn_tc_bwd_kernel", "tc_wgrad_kernel", "tc_nt_kernel", "obprop_out_grad_kernel"],
          ["attn_small_fwd_kernel", "layernorm_fwd_kernel"],
          {"split_weights_kernel": 3, "tc_wgrad_kernel": 3}),
    "C": (["layernorm_fwd_kernel", "layernorm_bwd_dx_kernel", "layernorm_bwd_param_kernel", "gemm_f32_kernel",
           "attn_softmax_fwd_kernel", "attn_softmax_bwd_kernel", "head_fwd_kernel<false>",
           "head_bwd_sample_kernel<false>", "obprop_out_grad_kernel"],
          ["tc_nt_kernel", "tc_wgrad_kernel", "layernorm_fwd_vec_kernel", "layernorm_bwd_fused_kernel",
           "attn_tc_fwd_kernel", "attn_small_fwd_kernel", "head_fwd_kernel<true>"],
          {}),
    "D": (["layernorm_fwd_kernel", "layernorm_bwd_dx_kernel", "layernorm_bwd_param_kernel", "tc_nt_kernel",
           "attn_softmax_fwd_kernel", "head_fwd_kernel<true>", "head_bwd_sample_kernel<true>"],
          ["layernorm_fwd_vec_kernel", "layernorm_bwd_fused_kernel", "attn_tc_fwd_kernel", "attn_small_fwd_kernel"],
          {}),
    "E": (["attn_tc_fwd_kernel", "attn_tc_bwd_kernel", "tc_wgrad_kernel", "obprop_out_grad_vec4_kernel"],
          # every forward GEMM on the tensor cores
          ["gemm_f32_kernel<false, true>", "attn_small_fwd_kernel", "attn_softmax_fwd_kernel"],
          {"tc_wgrad_kernel": 2, "split_weights_kernel": 2}),
    "F": (["attn_softmax_fwd_kernel", "gemm_f32_kernel", "tc_nt_kernel", "obprop_out_grad_vec4_kernel"],
          ["attn_tc_fwd_kernel", "attn_small_fwd_kernel"],
          {}),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_kernel_coverage(name):
    """One eager training step of each case launches the kernels its row of the module docstring names."""
    from raindrop_b200.train import TrainStep
    cfg, batch, wseed = case_setup(name)
    B = batch["src"].shape[1]
    ts = TrainStep(build_dropin(cfg, wseed).train(), B, use_graph=False)
    ts.load_batch(to_dev(batch))
    ts.step()
    torch.cuda.synchronize()
    cycles = _kernel_counts(ts.step)
    names = sorted(set().union(*cycles))
    # a template argument list is optional in COVERAGE: "tc_nt_kernel" stands for every instance
    count = lambda k: max(sum(n for full, n in c.items() if k in (full, full.split("<")[0])) for c in cycles)
    print(name, [dict(sorted(c.items())) for c in cycles])
    must, must_not, at_least = COVERAGE[name]
    assert not [k for k in must if count(k) == 0], ([k for k in must if count(k) == 0], names)
    assert not [k for k in must_not if count(k) > 0], ([k for k in must_not if count(k) > 0], names)
    assert all(count(k) >= n for k, n in at_least.items()), {k: (count(k), n) for k, n in at_least.items()}


def _run_dropin(cfg, batch, wseed, mode):
    from raindrop_b200 import functional as RF
    model = build_dropin(cfg, wseed).eval()
    model._plan.debug_keep_workspace = True
    model._plan.obprop_mode = mode
    d = to_dev(batch)
    logits, _, _ = model.forward(d["src"], d["static"], d["times"], d["lengths"])
    loss = F.cross_entropy(logits, d["y"])
    loss.backward()
    T, B = d["src"].shape[0], d["src"].shape[1]
    D = cfg["d_inp"] * cfg["d_ob"] + 16
    enc_in = RF.workspace_view(model._plan, L.WS_ENC_IN).view(T, B, D)
    enc_out = RF.workspace_view(model._plan, L.WS_ENC_OUT).view(T, B, D)
    return dict(model.named_parameters()), logits.detach(), loss.item(), enc_in, enc_out


def _exact_tol(cfg):
    return 1e-2 if cfg["max_len"] * cfg["d_ob"] >= 1024 else GRAD_TOL_EXACT


def check_eval(name):
    """Eval-mode forward and parameter gradients in both ob-prop modes against the fp32 oracle (and in single-pass TF32
    mode against the oracle under the kernels' rounding model), as test_gpu_parity.test_against_oracle."""
    cfg, batch, wseed = case_setup(name)
    oracle = _oracle(cfg, wseed)
    stages = {}
    ref_logits, _, _ = oracle.forward_dense(batch["src"], batch["static"], batch["times"], batch["lengths"], stages=stages)
    F.cross_entropy(ref_logits, batch["y"]).backward()
    go = dict(oracle.named_parameters())
    ref = {k: go[k].grad.clone() for k in used_param_keys(cfg)}
    D4 = cfg["d_inp"] * cfg["d_ob"]
    C_ = cfg["max_len"] * cfg["d_ob"]
    worst = {}
    gp, logits, _, enc_in, _ = _run_dropin(cfg, batch, wseed, EXACT)
    assert normwise(enc_in[:, :, :D4], stages["obs"]) < 1e-4
    assert normwise(enc_in[:, :, D4:], stages["pe"]) < 1e-5
    assert normwise(logits, ref_logits) < 1e-4
    errs = {k: normwise(gp[k].grad, ref[k]) for k in used_param_keys(cfg)}
    worst["exact"] = max(errs.items(), key=lambda kv: kv[1])
    assert all(e < _exact_tol(cfg) for e in errs.values()), errs
    gp, logits, _, enc_in, _ = _run_dropin(cfg, batch, wseed, FAST)
    if C_ % 4 or C_ < 16:
        # the ob-prop tensor-core kernel does not take this C: both modes run the fp32 CUDA-core GEMMs, so the
        # single-pass TF32 mode is held to the error-compensated bounds
        assert normwise(enc_in[:, :, :D4], stages["obs"]) < 1e-4
        assert normwise(logits, ref_logits) < 1e-4
        errs = {k: normwise(gp[k].grad, ref[k]) for k in used_param_keys(cfg)}
        worst["fast (fp32 ob-prop)"] = max(errs.items(), key=lambda kv: kv[1])
        assert all(e < _exact_tol(cfg) for e in errs.values()), errs
        print("eval parity %-6s %s" % (name, worst))
        return
    assert normwise(enc_in[:, :, :D4], stages["obs"]) < FWD_TOL
    assert normwise(logits, ref_logits) < FWD_TOL
    for k in used_param_keys(cfg):
        if "lin_value" in k:
            assert rel_l2(gp[k].grad, ref[k]) < OBPROP_GRAD_L2, k
        else:
            assert normwise(gp[k].grad, ref[k]) < GRAD_TOL, k
    oracle.zero_grad()
    st2 = {}
    m_logits, _, _ = oracle.forward_dense(batch["src"], batch["static"], batch["times"], batch["lengths"], stages=st2,
                                          tf32_model=True)
    F.cross_entropy(m_logits, batch["y"]).backward()
    assert normwise(enc_in[:, :, :D4], st2["obs"].detach()) < 1e-4
    assert normwise(logits, m_logits.detach()) < 1e-4
    errs = {}
    for k in used_param_keys(cfg):
        if "lin_value" in k:
            errs[k] = rel_l2(gp[k].grad, go[k].grad)
            assert errs[k] < 10 * MODEL_TOL, (k, "rel_l2 vs tf32 precision model")
        else:
            errs[k] = normwise(gp[k].grad, go[k].grad)
            assert errs[k] < MODEL_TOL, (k, "vs tf32 precision model", errs[k])
    worst["fast (tf32 model)"] = max(errs.items(), key=lambda kv: kv[1])
    print("eval parity %-6s %s" % (name, worst))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES) + RANDOM)
def test_eval_against_oracle(name):
    check_eval(name)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
@pytest.mark.parametrize("name", FIXTURE_CASES)
def test_eval_against_reference_fixture(golden_dir, name, mode):
    """The CUDA path against the reference's own outputs at A, B and C (bounds of test_golden_fixture)."""
    z, _ = load_golden(golden_dir, "hparams_" + name)
    cfg, batch, wseed = case_setup(name)
    gp, logits, loss, enc_in, enc_out = _run_dropin(cfg, batch, wseed, mode)
    errs = {}
    assert normwise(logits, z["logits"]) < (1e-4 if mode == EXACT else FWD_TOL)
    assert abs(loss - float(z["loss"])) < 1e-3 * max(1.0, abs(float(z["loss"])))
    D4 = cfg["d_inp"] * cfg["d_ob"]
    check_against_golden(z, "obs" in z.files, "obs", enc_in[:, :, :D4], 1e-4 if mode == EXACT else FWD_TOL, errs)
    check_against_golden(z, "pe" in z.files, "pe", enc_in[:, :, D4:], 1e-5, errs)
    valid = (torch.arange(cfg["max_len"])[:, None] < batch["lengths"][None, :]).to(enc_out.device)[:, :, None]
    if "enc" in z.files:
        errs["enc"] = normwise(enc_out * valid, torch.from_numpy(z["enc"]).to(enc_out.device) * valid)
        assert errs["enc"] < FWD_TOL
    for k in used_param_keys(cfg):
        full = "grad." + k in z.files
        if mode == EXACT:
            check_against_golden(z, full, "grad." + k, gp[k].grad, _exact_tol(cfg), errs)
        elif "lin_value" in k:
            check_against_golden(z, full, "grad." + k, gp[k].grad, OBPROP_GRAD_L2 * (1 if full else 2), errs, metric=rel_l2)
        else:
            check_against_golden(z, full, "grad." + k, gp[k].grad, GRAD_TOL, errs)
    assert all(p.grad is None for k, p in gp.items() if k not in set(used_param_keys(cfg)))
    print(name, mode, "worst", max(errs.items(), key=lambda kv: kv[1]))


def check_train(name, modes=(EXACT, FAST)):
    """One training step with replayed masks and gates against the float64 oracle, input gradients included
    (test_train_parity.check_train_case)."""
    from test_train_parity import check_train_case
    check_train_case(name, modes, setup=case_setup(name))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_train_against_masked_oracle(name):
    check_train(name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", RANDOM)
def test_random_train_against_masked_oracle(name):
    check_train(name, modes=(EXACT,))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["A", "B"])
def test_dp_sqnorms_against_oracle(name):
    """Per-sample squared gradient norms of a training forward against the float64 oracle's per-sample gradients under
    the same masks (bounds of test_dp_sgd.test_sqnorms_train_match_oracle_under_replayed_masks)."""
    from oracle import dropout_masks as DM
    from raindrop_b200 import privacy as PV
    from test_dp_sgd import RNG0, _check_gates, _close, _gpu_gates, _oracle_per_sample
    cfg, batch, _ = case_setup(name)
    model = build_dropin(cfg, 21).train()        # _oracle_per_sample builds weight seed 21
    plan = model._prepare(torch.device("cuda"))
    plan.obprop_mode = EXACT
    d = to_dev(batch)
    gates = _gpu_gates(model, cfg, d)
    sq = PV.per_sample_grad_sqnorms(model, d["src"], d["static"], d["times"], d["lengths"], d["y"]).cpu().numpy()
    keys = PV.sqnorm_fields(model)
    assert sorted(keys) == sorted(used_param_keys(cfg))
    masks = DM.model_masks(RNG0, P, cfg, batch["src"].shape[1])
    ref, _, stages = _oracle_per_sample(cfg, batch, masks, keys, gates)
    _check_gates(cfg, gates, stages, masks, batch["src"].shape[1])
    ok = _close(sq, ref, 1e-4)
    assert ok.all(), [(b, keys[f], sq[b, f], ref[b, f]) for b, f in zip(*np.nonzero(~ok))][:10]


@pytest.mark.gpu
def test_dp_train_step_at_eight_layers():
    """DPTrainStep on B (eight layers, 104 gradient fields): without clipping or noise it is TrainStep, bitwise."""
    from raindrop_b200 import privacy as PV
    from raindrop_b200.train import TrainStep
    from test_train_parity import RNG0
    cfg, batch, wseed = case_setup("B")
    B = batch["src"].shape[1]
    out = []
    for dp in (False, True):
        model = build_dropin(cfg, wseed).train()
        plan = model._prepare(torch.device("cuda"))
        plan.obprop_mode = EXACT
        plan.rng_state.copy_(torch.tensor(RNG0, dtype=torch.int64))
        if dp:
            s = PV.DPTrainStep(model, B, max_grad_norm=1e30, noise_multiplier=0.0, expected_batch_size=B, noise_seed=9)
            assert len(s.plan.fields) == len(used_param_keys(cfg)) == 104
        else:
            s = TrainStep(model, B)
        s.load_batch(to_dev(batch))
        losses = [s.step().clone() for _ in range(2)]
        torch.cuda.synchronize()
        out.append((s.flat_p.clone(), torch.cat(losses)))
    assert torch.isfinite(out[0][0]).all()
    for a, b in zip(*out):
        assert torch.equal(a, b)
    # with clipping and noise the step still runs and moves the parameters
    model = build_dropin(cfg, wseed).train()
    s = PV.DPTrainStep(model, B, max_grad_norm=0.5, noise_multiplier=1.0, expected_batch_size=B, noise_seed=9)
    p0 = s.flat_p.clone()
    s.load_batch(to_dev(batch))
    s.step()
    torch.cuda.synchronize()
    assert torch.isfinite(s.flat_p).all() and not torch.equal(s.flat_p, p0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["A", "C"])
def test_mc_dropout_equals_module_loop(name):
    """Monte Carlo replicates equal the module's training forwards at (seed, step + m) (test_mc_dropout)."""
    from raindrop_b200 import uncertainty as U
    from test_mc_dropout import LOOP_TOL, SEED, STEP, check_stats_derived, mc, module_loop
    cfg, batch, wseed = case_setup(name)
    model = build_dropin(cfg, wseed).eval()
    d = to_dev(batch)
    B, M = batch["src"].shape[1], 4
    loop = module_loop(model, d, SEED, STEP, M, EXACT)
    res = mc(model, d, EXACT, n_samples=M, return_samples=True, internal_batch_size=3 * B)   # chunks 3, 1
    e = normwise(res.samples, loop)
    print("mc_dropout vs module loop %s normwise %.3e" % (name, e))
    assert e <= LOOP_TOL, (name, e)
    assert not torch.equal(loop[0], loop[1])
    check_stats_derived(res, U.mc_dropout_from_logits(loop), (res.samples - loop).abs().max().item(), cfg["n_classes"])


@pytest.mark.gpu
def test_integrated_gradients_at_d_mod_4():
    """Case C (D = 26): attributions equal the loop of torch.autograd.grad at the quadrature nodes, and are complete."""
    from raindrop_b200 import attribution as A
    from test_integrated_gradients import _endpoint_logits, _loop
    cfg, batch, wseed = case_setup("C")
    d = to_dev(batch)
    model = build_dropin(cfg, wseed).eval()
    model._plan.obprop_mode = EXACT
    attr_src, attr_st = A.integrated_gradients(model, d["src"], d["static"], d["times"], d["lengths"], target=d["y"],
                                               n_steps=6, internal_batch_size=2 * batch["src"].shape[1])
    ref_src, ref_st = _loop(model, d, d["y"], 6)
    e = {"attr_src": normwise(attr_src, ref_src), "attr_static": normwise(attr_st, ref_st)}
    assert max(e.values()) < 1e-5, e
    assert torch.count_nonzero(attr_src) > 0
    # completeness: sum of attributions = F(x) - F(0) up to the quadrature error
    attr_src, attr_st, delta = A.integrated_gradients(model, d["src"], d["static"], d["times"], d["lengths"],
                                                      target=d["y"], n_steps=64, return_convergence_delta=True)
    ends = _endpoint_logits(model, d, d["y"])
    f = ends.gather(2, d["y"].view(1, -1, 1).expand(2, -1, 1))[:, :, 0]
    total = attr_src.double().sum((0, 2)) + attr_st.double().sum(1)
    scale = float((f[1] - f[0]).abs().max()) + 1e-6
    assert float((total - (f[1] - f[0]).double()).abs().max()) / scale < 1e-2
    assert float(delta.abs().max()) / scale < 1e-2
    print("integrated gradients C", e, "completeness", float(delta.abs().max()) / scale)


@pytest.mark.gpu
def test_train_step_graph_replay_at_eight_layers():
    """TrainStep (CUDA graph) on B: two steps, each against the float64 oracle at the pre-step parameters under that
    step's masks and gates (test_train_parity.test_train_step_graph_replay_against_masked_oracle)."""
    from helpers import read_gpu
    from raindrop_b200.train import TrainStep
    from test_train_parity import TIGHT, _ws_rng, check_masks, oracle_train
    cfg, batch, wseed = case_setup("B")
    B = batch["src"].shape[1]
    model = build_dropin(cfg, wseed).train()
    ts = TrainStep(model, B, lr=1e-3, use_graph=True)
    keys = [k for k, _ in ts.plan.fields]
    params = model.used_parameters()
    for it in range(2):
        b = make_batch(cfg, B, seed=70 + it)
        ts.load_batch(to_dev(b))
        p_before = ts.flat_p.clone()
        rng = tuple(ts.plan.rng_state.tolist())
        ts.step()
        torch.cuda.synchronize()
        assert ts.graph is not None and _ws_rng(ts.dims, ts.ws) == rng
        sd = {k: p_before[off:off + p.numel()].view(p.shape).cpu() for k, p, off in zip(keys, params, ts.offsets)}
        ref, masks = oracle_train(cfg, b, wseed, rng, params=sd, gates=read_gpu(cfg, ts.dims, ts.ws)["gates"])
        check_masks(masks, P)
        assert all(n <= max(1, 1e-4 * g) for n, g in ref["gate_dis"].values()), ref["gate_dis"]
        assert abs(ts.loss.item() - ref["loss"]) / max(1.0, abs(ref["loss"])) < TIGHT
        errs = {k: normwise(ts.flat_g[off:off + p.numel()].view(p.shape), ref["grads"][k])
                for k, p, off in zip(keys, params, ts.offsets)}
        assert all(e < TIGHT for e in errs.values()), errs
        print("TrainStep B step", it, "worst", max(errs.items(), key=lambda kv: kv[1]))


@pytest.mark.gpu
def test_training_beyond_the_head_backward_raises():
    """Df = 736 > 722: eval runs and matches the oracle; a training forward, eager or TrainStep, raises
    RaindropB200Error before it produces any output, and no gradient is written."""
    from raindrop_b200.train import TrainStep
    hp = dict(d_inp=45, d_ob=16, nhead=4, nhid=64, nlayers=1, max_len=4, d_static=0, n_classes=2)
    cfg = hparam_config("WIDE", hp)
    batch = make_batch(cfg, 2, seed=1)
    d = to_dev(batch)
    model = build_dropin(cfg, 3)
    with torch.no_grad():
        logits = model.eval()(d["src"], d["static"], d["times"], d["lengths"])[0]
    ref, _, _ = _oracle(cfg, 3).forward_dense(batch["src"], batch["static"], batch["times"], batch["lengths"])
    assert normwise(logits, ref.detach()) < 1e-4
    model.train()
    with pytest.raises(L.RaindropB200Error, match="722"):
        model(d["src"], d["static"], d["times"], d["lengths"])
    assert all(p.grad is None for p in model.parameters())
    with pytest.raises(L.RaindropB200Error):
        ts = TrainStep(model, 2, use_graph=False)
        ts.load_batch(d)
        ts.step()
        torch.cuda.synchronize()
