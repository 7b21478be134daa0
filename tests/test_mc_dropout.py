"""Monte Carlo dropout (raindrop_b200.uncertainty): the host statistics on the CPU; on the GPU, the device call against
the loop of training-mode module forwards at rng_state = (seed, step + m), against the float64 oracle under the replayed
masks of every replicate, and its chunking, key and side-effect contract.

Every GPU test pins plan.obprop_mode: the auto mode picks the ob-prop arithmetic from the row count, so the chunking
would otherwise change the arithmetic."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import build_dropin, normwise, to_dev
from raindrop_b200 import uncertainty as U
from raindrop_b200.synth import make_batch, model_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXACT, FAST = 2, 1
SEED, STEP = 0x2B7E151628AED2A6, (1 << 32) - 2          # the step counter carries into its high word inside the call
LOOP_TOL = 1e-6
LOGIT_TOL_EXACT = 1e-4                                    # the train-parity bound against the float64 oracle
# name -> (config, B, make_batch options, n_samples); each reaches a different dropout code path
GPU_CASES = {
    "tiny_b6_len1": ("TINY", 6, {}, 5),        # attn_small (hd = 18), lengths[0] = 1
    "tiny8_b9": ("TINY8", 9, {}, 5),           # attn_tc, no statics, 8 classes
    "p19_b37": ("P19", 37, {}, 4),             # attn_tc, D = 152: partial keep-bit word
    "p12_b3": ("P12", 3, {}, 3),               # T = 215: batched attention
    "pam_b2": ("PAM", 2, {}, 3),               # T = 600, C = 2400
}
FALLBACK_CASES = ("tiny8_b9", "p19_b9")


# ---- host statistics --------------------------------------------------------------------------------------------------
def _direct(logits):
    """The statistics straight from their definitions, one replicate and one sample at a time."""
    M, B, C = logits.shape
    p = np.empty_like(logits)
    h = np.empty((M, B))
    for m in range(M):
        for b in range(B):
            e = np.exp(logits[m, b] - logits[m, b].max())
            p[m, b] = e / e.sum()
            h[m, b] = -sum(x * np.log(x) for x in p[m, b] if x > 0)
    mean = p.mean(axis=0)
    var = ((p - mean) ** 2).sum(axis=0) / (M - 1) if M > 1 else np.zeros_like(mean)
    pred = np.array([-sum(x * np.log(x) for x in mean[b] if x > 0) for b in range(B)])
    return mean, var, pred, h.mean(axis=0)


@pytest.mark.parametrize("M,C", [(1, 2), (1, 8), (7, 2), (7, 8), (30, 8)])
def test_from_logits_matches_direct_formulas(M, C):
    x = np.random.default_rng(M * 10 + C).normal(scale=3.0, size=(M, 5, C))
    r = U.mc_dropout_from_logits(torch.tensor(x))
    mean, var, pred, expected = _direct(x)
    np.testing.assert_allclose(r.mean_probs, mean, rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(r.variance, var, rtol=1e-10, atol=1e-15)
    np.testing.assert_allclose(r.predictive_entropy, pred, rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(r.expected_entropy, expected, rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(r.mutual_information, pred - expected, atol=1e-13)
    assert np.all(r.mutual_information > -1e-13)
    if M == 1:
        assert np.all(r.variance == 0) and np.all(np.abs(r.mutual_information) <= 1e-15)
    assert np.array_equal(r.samples, x)


def test_from_logits_saturated_and_identical():
    # probabilities that underflow to 0 in fp64 (0 log 0 = 0, no NaN), and identical replicates (MI = 0)
    x = np.zeros((4, 3, 8))
    x[:, 0, 3] = 2000.0
    x[:, 1, :] = np.arange(8) * 300.0
    x[:, 2, :] = np.linspace(-1, 1, 8)
    r = U.mc_dropout_from_logits(x)
    for f in (r.mean_probs, r.variance, r.predictive_entropy, r.expected_entropy, r.mutual_information):
        assert np.all(np.isfinite(f))
    assert r.mean_probs[0, 3] == 1.0 and r.predictive_entropy[0] == 0.0 and r.expected_entropy[0] == 0.0
    assert np.all(np.abs(r.mutual_information) <= 1e-15)
    assert np.all(np.abs(r.variance) <= 1e-30)
    mean, _, pred, expected = _direct(x)
    np.testing.assert_allclose(r.predictive_entropy, pred, rtol=1e-12, atol=1e-15)
    # two classes, replicates that disagree: MI > 0
    y = np.array([[[4.0, -4.0]], [[-4.0, 4.0]]])
    ry = U.mc_dropout_from_logits(y)
    assert ry.mutual_information[0] > 0.5 and abs(ry.mean_probs[0, 0] - 0.5) < 1e-15


def test_from_logits_validation():
    for bad in (np.zeros((2, 3)), np.zeros((0, 2, 2)), np.zeros((2, 0, 2)), np.full((2, 2, 2), np.nan),
                np.full((1, 1, 2), np.inf)):
        with pytest.raises(ValueError):
            U.mc_dropout_from_logits(bad)


def _cpu_model():
    cfg = model_config("TINY", dropout=0.2)
    return build_dropin(cfg, 3, device="cpu"), make_batch(cfg, 3, seed=1)


def test_argument_validation():
    model, b = _cpu_model()
    args = (b["src"], b["static"], b["times"], b["lengths"])
    for kw in (dict(n_samples=0), dict(seed=-1), dict(seed=1 << 64), dict(step=-1), dict(step=(1 << 64) - 2, n_samples=3),
               dict(internal_batch_size=0)):
        with pytest.raises(ValueError):
            U.mc_dropout(model, *args, **kw)
    with pytest.raises(ValueError):
        U.mc_dropout(model, b["src"][:, :, :3], b["static"], b["times"], b["lengths"])
    with pytest.raises(ValueError):
        U.mc_dropout(model, b["src"], None, b["times"], b["lengths"])
    with pytest.raises(TypeError):
        U.mc_dropout(torch.nn.Linear(2, 2), *args)
    from raindrop_b200.models_rd import Raindrop
    with pytest.raises(TypeError):
        U.mc_dropout(Raindrop.__new__(Raindrop), *args)


def test_no_cuda_raises(monkeypatch):
    from raindrop_b200.lib import RaindropB200Error
    model, b = _cpu_model()
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RaindropB200Error):
        U.mc_dropout(model, b["src"], b["static"], b["times"], b["lengths"], n_samples=4)


# ---- GPU --------------------------------------------------------------------------------------------------------------
def gpu_case(name):
    """(cfg, batch, weight seed, n_samples) of a named case."""
    if name == "p19_b9":
        cfg_name, B, opts, M = "P19", 9, {}, 5
    else:
        cfg_name, B, opts, M = GPU_CASES[name]
    cfg = model_config(cfg_name, dropout=0.2)
    batch = make_batch(cfg, B, seed=200 + B, **opts)
    if name == "tiny_b6_len1":
        batch["lengths"][0] = 1
        batch["times"][1:, 0] = 0
        batch["src"][1:, 0, :] = 0
    return cfg, batch, 21, M


def module_loop(model, d, seed, step, M, mode):
    """Logits [M, B, C] of M training-mode module forwards at rng_state = (seed, step + m); the model's mode and
    rng_state are restored."""
    plan = model._prepare(d["src"].device)
    plan.obprop_mode = mode
    saved, was_training = plan.rng_state.clone(), model.training
    model.train()
    out = []
    with torch.no_grad():
        for m in range(M):
            plan.rng_state.copy_(torch.tensor(np.array([seed, step + m], dtype=np.uint64).view(np.int64)))
            out.append(model(d["src"], d["static"], d["times"], d["lengths"])[0].clone())
    plan.rng_state.copy_(saved)
    model.train(was_training)
    return torch.stack(out)


def mc(model, d, mode, **kw):
    model._plan.obprop_mode = mode
    kw.setdefault("seed", SEED)
    kw.setdefault("step", STEP)
    return U.mc_dropout(model, d["src"], d["static"], d["times"], d["lengths"], **kw)


def check_stats(res, ref, tol_mean, tol_var, tol_ent):
    """Device statistics against a float64 MCDropoutResult, absolute bounds."""
    errs = dict(mean=(res.mean_probs.double().cpu() - torch.tensor(ref.mean_probs)).abs().max().item(),
                var=(res.variance.double().cpu() - torch.tensor(ref.variance)).abs().max().item())
    for k in ("predictive_entropy", "expected_entropy", "mutual_information"):
        errs[k] = (getattr(res, k).double().cpu() - torch.tensor(getattr(ref, k))).abs().max().item()
    tols = dict(mean=tol_mean, var=tol_var, predictive_entropy=tol_ent, expected_entropy=tol_ent,
                mutual_information=2 * tol_ent)
    bad = {k: (e, tols[k]) for k, e in errs.items() if not e <= tols[k]}
    assert not bad, bad
    return errs


def check_stats_derived(res, ref, e, C):
    """The statistics against float64 ones computed from logits that differ from the device's by at most e (absolute):
    softmax moves a probability by at most a factor exp(2e), so |d mean p| <= 2e, |d var| <= 8e and
    |d H| <= 2e (log C + 1), to first order; + the fp32 rounding of the outputs."""
    k = 2.0 * e * 1.01 + 1e-7
    return check_stats(res, ref, k, 4 * k + 1e-7, k * (np.log(C) + 1) + 1e-6)


def check_against_loop(name):
    cfg, batch, wseed, M = gpu_case(name)
    model = build_dropin(cfg, wseed).eval()
    d = to_dev(batch)
    B = batch["src"].shape[1]
    loop = module_loop(model, d, SEED, STEP, M, EXACT)
    res = mc(model, d, EXACT, n_samples=M, return_samples=True, internal_batch_size=2 * B)   # chunks 2, 2, .., ragged
    e = normwise(res.samples, loop)
    print("mc_dropout vs module loop %-12s B=%d M=%d normwise %.3e" % (name, B, M, e))
    assert e <= LOOP_TOL, (name, e)
    assert not torch.equal(loop[0], loop[1])                    # the replicates really differ
    check_stats_derived(res, U.mc_dropout_from_logits(loop), (res.samples - loop).abs().max().item(), cfg["n_classes"])


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GPU_CASES))
def test_equals_module_loop(name):
    check_against_loop(name)


@pytest.mark.gpu
@pytest.mark.parametrize("env", [{"RD_TC_GEMM": "0"}, {"RD_ATTN_TC": "0"}, {"RD_ATTN_TC": "0", "RD_ATTN_SMALL": "0"}],
                         ids=["cuda_core_gemm", "attn_small", "batched_attention"])
def test_cuda_core_fallbacks_equal_module_loop(env):
    """RD_TC_GEMM=0: dropout in the CUDA-core GEMM epilogue; RD_ATTN_TC=0: the CUDA-core fused attention at hd = 76;
    RD_ATTN_TC=0 RD_ATTN_SMALL=0: the batched attention path at T <= 64 (the switches are read once per process)."""
    code = ("import sys\nsys.path[:0] = [%r, %r]\nimport test_mc_dropout as t\n"
            "for name in t.FALLBACK_CASES:\n    t.check_against_loop(name)\nprint('FALLBACK_OK')\n"
            % (os.path.join(ROOT, "tests"), ROOT))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, **env),
                       cwd=ROOT, timeout=900)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "FALLBACK_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny_b6_len1", "tiny8_b9", "p12_b3"])
def test_against_float64_oracle(name):
    """Each replicate against RaindropV2Oracle.forward_dense(masks=...) in float64 under the masks of (seed, step + m)
    for the B-row problem, within the train-parity bound; the statistics against mc_dropout_from_logits of the oracle's
    logits, within the bounds check_stats_derived derives from the measured logit error."""
    from oracle import dropout_masks as DM
    from oracle.raindrop_oracle import build_oracle_model
    from raindrop_b200.synth import synth_weights
    cfg, batch, wseed, M = gpu_case(name)
    M = 3
    model = build_dropin(cfg, wseed)
    d = to_dev(batch)
    B, C = batch["src"].shape[1], cfg["n_classes"]
    res = mc(model, d, EXACT, n_samples=M, return_samples=True, internal_batch_size=2 * B)
    oracle = build_oracle_model(cfg).eval()
    synth_weights(oracle, cfg, seed=wseed)
    oracle.double()
    ref = []
    with torch.no_grad():
        for m in range(M):
            masks = DM.model_masks((SEED, STEP + m), 0.2, cfg, B)
            st = None if batch["static"] is None else batch["static"].double()
            ref.append(oracle.forward_dense(batch["src"].double(), st, batch["times"].double(), batch["lengths"],
                                            masks=masks)[0])
    ref = torch.stack(ref)
    errs = [normwise(res.samples[m], ref[m]) for m in range(M)]
    print("mc_dropout vs float64 oracle %-12s per-replicate normwise %s" % (name, ["%.2e" % x for x in errs]))
    assert max(errs) <= LOGIT_TOL_EXACT, errs
    stats = check_stats_derived(res, U.mc_dropout_from_logits(ref), (res.samples.double().cpu() - ref).abs().max().item(), C)
    print("  statistics errors", stats)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXACT, FAST])
def test_chunking_invariance(mode):
    cfg, batch, wseed, _ = gpu_case("tiny8_b9")
    model = build_dropin(cfg, wseed)
    d = to_dev(batch)
    B, M = batch["src"].shape[1], 7
    outs = [mc(model, d, mode, n_samples=M, return_samples=True, internal_batch_size=ibs) for ibs in (B, 3 * B, M * B)]
    for o in outs[1:]:
        for f in ("mean_probs", "variance", "predictive_entropy", "expected_entropy", "mutual_information", "samples"):
            assert torch.equal(getattr(o, f), getattr(outs[0], f)), (mode, f)


@pytest.mark.gpu
@pytest.mark.parametrize("training", [False, True])
def test_key_and_no_side_effects(training):
    cfg, batch, wseed, _ = gpu_case("p19_b37")
    model = build_dropin(cfg, wseed).train(training)
    d = to_dev(batch)
    plan = model._prepare(d["src"].device)
    inputs = {k: v.clone() for k, v in d.items() if v is not None}
    params = [p.detach().clone() for p in model.parameters()]
    rng = plan.rng_state.clone()
    M, k = 6, 2
    a = mc(model, d, EXACT, n_samples=M, return_samples=True, internal_batch_size=4 * 37)
    b = mc(model, d, EXACT, n_samples=M, return_samples=True, internal_batch_size=4 * 37)
    for f in ("mean_probs", "variance", "predictive_entropy", "expected_entropy", "mutual_information", "samples"):
        assert torch.equal(getattr(a, f), getattr(b, f)), f
    tail = mc(model, d, EXACT, n_samples=M - k, step=STEP + k, return_samples=True, internal_batch_size=4 * 37)
    assert torch.equal(tail.samples, a.samples[k:])
    other = mc(model, d, EXACT, n_samples=M, seed=SEED + 1, return_samples=True)
    assert not torch.equal(other.samples, a.samples)
    assert torch.equal(plan.rng_state, rng) and model.training == training
    assert all(torch.equal(p, q) for p, q in zip(model.parameters(), params))
    assert all(p.grad is None for p in model.parameters())
    assert all(torch.equal(d[k2], v) for k2, v in inputs.items())
    # seed=None: the model's own dropout seed
    own = mc(model, d, EXACT, n_samples=2, seed=None, step=0, return_samples=True)
    assert torch.equal(own.samples, mc(model, d, EXACT, n_samples=2, seed=model._seed, step=0, return_samples=True).samples)


@pytest.mark.gpu
def test_dropout_zero_equals_eval_forward():
    cfg = model_config("P19", dropout=0.0)
    batch = make_batch(cfg, 11, seed=5)
    model = build_dropin(cfg, 21).eval()
    d = to_dev(batch)
    model._plan.obprop_mode = EXACT
    with torch.no_grad():
        ref = model(d["src"], d["static"], d["times"], d["lengths"])[0]
    res = mc(model, d, EXACT, n_samples=5, return_samples=True, internal_batch_size=2 * 11)
    for m in range(5):
        assert normwise(res.samples[m], ref) <= LOOP_TOL
    assert res.mutual_information.abs().max().item() <= 1e-12
    assert res.variance.abs().max().item() <= 1e-14


@pytest.mark.gpu
def test_cuda_graph_capture_equals_eager():
    cfg, batch, wseed, _ = gpu_case("tiny8_b9")
    model = build_dropin(cfg, wseed)
    d = to_dev(batch)
    kw = dict(n_samples=7, return_samples=True, internal_batch_size=3 * 9)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eager = mc(model, d, EXACT, **kw)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = mc(model, d, EXACT, **kw)
    # a later eager call with another key and chunking replaces the cached key and scratch; the graph keeps its own
    mc(model, d, EXACT, n_samples=3, step=5, internal_batch_size=9)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        for f in ("mean_probs", "variance", "predictive_entropy", "expected_entropy", "mutual_information", "samples"):
            assert torch.equal(getattr(out, f), getattr(eager, f)), f
