"""DP-SGD (raindrop_b200.privacy): the RDP accountant and the Poisson sampler on the CPU; on the GPU, the per-sample
gradient norms against one-sample module backwards (eval) and the float64 oracle under the replayed dropout masks
(train), the DP step against TrainStep, clipping, slot weights, the noise stream and determinism.

Every GPU test pins plan.obprop_mode: the auto mode picks the ob-prop arithmetic from the row count, and a one-sample
backward has fewer rows than the batch."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import GATE_SITES, build_dropin, gate_disagreements, normwise, read_gpu, to_dev
from raindrop_b200 import lib as L
from raindrop_b200 import privacy as PV
from raindrop_b200.synth import make_batch, model_config, used_param_keys

EXACT = 2
RNG0 = (0x2B7E151628AED2A6, (1 << 32) + 7)


# ---- accountant ---------------------------------------------------------------------------------------------------------
def _quad_log_a(q, sigma, alpha):
    """log A_alpha = log E_{z ~ N(0, sigma^2)}[((1 - q) + q exp((2z - 1) / (2 sigma^2)))^alpha] by mpmath quadrature."""
    import mpmath as mp
    mp.mp.dps = 40
    q, s, a = mp.mpf(q), mp.mpf(sigma), mp.mpf(alpha)

    def f(z):
        return mp.npdf(z, 0, s) * ((1 - q) + q * mp.e ** ((2 * z - 1) / (2 * s * s))) ** a
    return float(mp.log(mp.quad(f, [-mp.inf, -10 * s, 0, 0.5, 10 * s + 1, mp.inf])))


def test_rdp_at_full_sampling_is_the_gaussian_mechanism():
    orders = np.array([1.5, 2, 3.25, 8, 64, 256])
    for sigma in (0.5, 1.0, 4.0):
        np.testing.assert_allclose(PV.rdp_sampled_gaussian(1.0, sigma, orders), orders / (2 * sigma ** 2), rtol=1e-12)


@pytest.mark.parametrize("q,sigma", [(0.01, 1.1), (0.1, 0.8), (0.3, 2.0)])
def test_rdp_integer_and_fractional_orders_match_quadrature(q, sigma):
    for a in (2, 3, 5, 12, 1.5, 2.75, 6.5):
        got = PV.rdp_sampled_gaussian(q, sigma, [a])[0] * (a - 1)
        ref = _quad_log_a(q, sigma, a)
        assert abs(got - ref) <= 1e-9 * max(abs(ref), 1e-300) + 1e-15, (a, got, ref)


def test_epsilon_monotone_and_zero_without_sampling():
    assert PV.epsilon(0.0, 1.0, 1000, 1e-5) == 0.0
    e = [PV.epsilon(0.01, 1.0, s, 1e-5) for s in (10, 100, 1000)]
    assert 0 < e[0] < e[1] < e[2]
    e = [PV.epsilon(0.01, s, 1000, 1e-5) for s in (2.0, 1.0, 0.7)]
    assert e[0] < e[1] < e[2]


def test_noise_multiplier_inverts_epsilon():
    for target in (1.0, 3.0, 8.0):
        sigma = PV.noise_multiplier_for(target, 1e-5, 0.01, 2000)
        assert abs(PV.epsilon(0.01, sigma, 2000, 1e-5) - target) <= 1e-6 * target


# ---- Poisson sampler ----------------------------------------------------------------------------------------------------
def test_poisson_sampler_shapes_rate_overflow_and_seed():
    s = PV.PoissonSampler(1000, 0.05, seed=3)
    idx, w = s.sample()
    assert idx.shape == w.shape == (s.capacity,) and idx.dtype == np.int64 and w.dtype == np.float32
    assert set(np.unique(w)) <= {0.0, 1.0} and np.all((idx >= 0) & (idx < 1000))
    sizes = np.array([s.sample()[1].sum() for _ in range(2000)])
    se = math.sqrt(1000 * 0.05 * 0.95 / len(sizes))
    assert abs(sizes.mean() - 50.0) < 4 * se
    with pytest.raises(RuntimeError):
        PV.PoissonSampler(1000, 0.5, capacity=10, seed=0).sample()
    a, b = PV.PoissonSampler(500, 0.1, seed=7), PV.PoissonSampler(500, 0.1, seed=7)
    for _ in range(5):
        (ia, wa), (ib, wb) = a.sample(), b.sample()
        assert np.array_equal(ia, ib) and np.array_equal(wa, wb)


def test_entry_points_raise_without_cuda():
    if torch.cuda.is_available():
        pytest.skip("checks the CPU-only behaviour")
    cfg = model_config("TINY", dropout=0.0)
    m = build_dropin(cfg, 21, device="cpu")
    b = make_batch(cfg, 3, seed=1)
    with pytest.raises(L.RaindropB200Error):
        PV.per_sample_grad_sqnorms(m, b["src"], b["static"], b["times"], b["lengths"], b["y"])
    with pytest.raises(L.RaindropB200Error):
        PV.DPTrainStep(m, 3, 1.0, 1.0, 3.0)


# ---- noise stream restated in numpy ---------------------------------------------------------------------------------------
def noise_normals(seed, step, n):
    """float32 [n]: xi_i of rd_dp_add_noise (site 96, Box-Muller on word pairs, fp64 then rounded)."""
    from oracle import dropout_masks as DM
    w = DM.dropout_words(seed, step, 96, (n + 3) // 4 * 4).reshape(-1, 2, 2)
    u1 = ((w[..., 0] >> np.uint32(8)).astype(np.float64) + 1.0) * 2.0 ** -24
    u2 = (w[..., 1] >> np.uint32(8)).astype(np.float64) * 2.0 ** -24
    r, t = np.sqrt(-2.0 * np.log(u1)), 6.283185307179586 * u2
    return np.stack([r * np.cos(t), r * np.sin(t)], -1).reshape(-1)[:n].astype(np.float32)


# ---- GPU -------------------------------------------------------------------------------------------------------------------
CASES = {
    "tiny_b6": ("TINY", 6),       # attn_small
    "tiny8_b9": ("TINY8", 9),     # no statics, 8 classes
    "p19_b37": ("P19", 37),       # ghost form, R <= 64
    "p12_b3": ("P12", 3),         # explicit encoder form, ghost ob-prop form
    "pam_b2": ("PAM", 2),         # explicit encoder form, ghost ob-prop form with C = 2400
    "large_b2": ("LARGE", 2),     # tiled ghost form, R = 256 and 128
}


def _setup(name, dropout=0.0):
    cfg_name, B = CASES[name]
    cfg = model_config(cfg_name, dropout=dropout)
    batch = make_batch(cfg, B, seed=300 + B)
    model = build_dropin(cfg, 21)
    model._prepare(torch.device("cuda")).obprop_mode = EXACT
    return cfg, batch, model


def _module_sqnorms(model, cfg, d, b):
    """||grad of the one-sample module loss||^2 per trained tensor (sqnorm_fields order)."""
    model.zero_grad(set_to_none=True)
    sl = slice(b, b + 1)
    st = None if d["static"] is None else d["static"][sl]
    logits, _, _ = model.forward(d["src"][:, sl], st, d["times"][:, sl], d["lengths"][sl])
    F.cross_entropy(logits, d["y"][sl]).backward()
    sd = dict(model.named_parameters())
    return [sd[k].grad.double().pow(2).sum().item() for k in PV.sqnorm_fields(model)], \
        {k: sd[k].grad.detach().clone() for k in PV.sqnorm_fields(model)}


def _close(got, ref, tol):
    got, ref = np.asarray(got), np.asarray(ref)
    floor = 1e-9 * ref.sum(axis=-1, keepdims=True)
    return np.abs(got - ref) <= tol * np.abs(ref) + floor


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_sqnorms_eval_match_one_sample_backward(name):
    cfg, batch, model = _setup(name)
    model.eval()
    d = to_dev(batch)
    sq = PV.per_sample_grad_sqnorms(model, d["src"], d["static"], d["times"], d["lengths"], d["y"]).cpu().numpy()
    B = d["src"].shape[1]
    assert sq.shape == (B, len(used_param_keys(cfg)))
    assert sorted(PV.sqnorm_fields(model)) == sorted(used_param_keys(cfg))
    ref = np.array([_module_sqnorms(model, cfg, d, b)[0] for b in range(B)])
    # at T = 600 the one-sample module backward itself sums 600 rows per weight gradient in fp32: 1e-5 is below its error
    ok = _close(sq, ref, 5e-5 if cfg["max_len"] >= 600 else 1e-5)
    assert ok.all(), [(b, PV.sqnorm_fields(model)[f], sq[b, f], ref[b, f]) for b, f in zip(*np.nonzero(~ok))][:10]


def _oracle_per_sample(cfg, batch, masks, keys, gates=None):
    """float64 oracle under the replayed masks and ReLU gates: (per-sample squared norms [B, fields], per-sample gradients
    [{key: grad}], the oracle's stages)."""
    from oracle.raindrop_oracle import build_oracle_model
    from raindrop_b200.synth import synth_weights
    oracle = build_oracle_model(cfg).eval()             # eval: the masks are the only dropout
    synth_weights(oracle, cfg, seed=21)
    oracle.double()
    st = None if batch["static"] is None else batch["static"].double()
    stages = {}
    logits, _, _ = oracle.forward_dense(batch["src"].double(), st, batch["times"].double(), batch["lengths"],
                                        stages=stages, masks=masks, gates=gates)
    params = dict(oracle.named_parameters())
    B = batch["src"].shape[1]
    sq, grads = np.empty((B, len(keys))), []
    total = 0
    for b in range(B):
        gs = torch.autograd.grad(F.cross_entropy(logits[b:b + 1], batch["y"][b:b + 1]), [params[k] for k in keys],
                                 retain_graph=True)
        sq[b] = [g.pow(2).sum().item() for g in gs]
        grads.append(dict(zip(keys, gs)))
        total = total + torch.cat([g.flatten() for g in gs])
    # the per-sample gradients sum to the batch gradient
    batch_g = torch.autograd.grad(F.cross_entropy(logits, batch["y"]) * B, [params[k] for k in keys])
    assert normwise(total, torch.cat([g.flatten() for g in batch_g])) < 1e-10
    return sq, grads, stages


def _gpu_gates(model, cfg, d):
    """The ReLU decisions of the training forward at RNG0 (helpers.read_gpu), for the oracle to replay; the rng state is
    left at RNG0."""
    plan = model._prepare(torch.device("cuda"))
    plan.rng_state.copy_(torch.tensor(RNG0, dtype=torch.int64))
    plan.debug_keep_workspace = True
    with torch.no_grad():
        model.forward(d["src"], d["static"], d["times"], d["lengths"])
    plan.debug_keep_workspace = False
    plan.rng_state.copy_(torch.tensor(RNG0, dtype=torch.int64))
    return read_gpu(cfg, plan.last_dims, plan.last_workspace)["gates"]


def _check_gates(cfg, gates, stages, masks, B):
    """The replayed gates disagree with the oracle's own signs at no more than 1e-4 of each site's gates
    (test_train_parity.GATE_RATE)."""
    dis = gate_disagreements(cfg, gates, stages, masks, slice(0, B), B, {s: [0, 0] for s in GATE_SITES})
    assert all(n <= max(1, 1e-4 * g) for n, g in dis.values()), dis


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_sqnorms_train_match_oracle_under_replayed_masks(name):
    from oracle import dropout_masks as DM
    cfg, batch, model = _setup(name, dropout=0.2)
    model.train()
    d = to_dev(batch)
    gates = _gpu_gates(model, cfg, d)
    sq = PV.per_sample_grad_sqnorms(model, d["src"], d["static"], d["times"], d["lengths"], d["y"]).cpu().numpy()
    B = batch["src"].shape[1]
    keys = PV.sqnorm_fields(model)
    masks = DM.model_masks(RNG0, 0.2, cfg, B)
    ref, _, stages = _oracle_per_sample(cfg, batch, masks, keys, gates)
    _check_gates(cfg, gates, stages, masks, B)
    # fp32 path against float64: 1e-4, widened 5x where test_train_parity.py widens the gradient bound 5x (C = T d_ob
    # >= 1024: PAM, LARGE; the long sequences' fp32 data-gradient chain, not the norm kernels, which agree with the
    # module's own backward to 5e-5 in the eval test)
    ok = _close(sq, ref, 5e-4 if cfg["max_len"] * cfg["d_ob"] >= 1024 else 1e-4)
    assert ok.all(), [(b, keys[f], sq[b, f], ref[b, f]) for b, f in zip(*np.nonzero(~ok))][:10]


def _step(model, batch, B, **kw):
    step = PV.DPTrainStep(model, B, **kw)
    step.load_batch(to_dev(batch))
    return step


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [False, True])
def test_dp_step_reduces_to_train_step_bitwise(use_graph):
    from raindrop_b200.train import TrainStep
    cfg = model_config("P19", dropout=0.2)
    B = 37
    batch = make_batch(cfg, B, seed=5)
    out = []
    for dp in (False, True):
        model = build_dropin(cfg, 21).train()
        plan = model._prepare(torch.device("cuda"))
        plan.obprop_mode = EXACT
        plan.rng_state.copy_(torch.tensor(RNG0, dtype=torch.int64))
        if dp:
            s = _step(model, batch, B, max_grad_norm=1e30, noise_multiplier=0.0, expected_batch_size=B, noise_seed=9,
                      use_graph=use_graph)
        else:
            s = TrainStep(model, B, use_graph=use_graph)
            s.load_batch(to_dev(batch))
        losses = [s.step().clone() for _ in range(3)]
        torch.cuda.synchronize()
        out.append((s.flat_p.clone(), s.exp_avg.clone(), s.exp_avg_sq.clone(), torch.cat(losses)))
    for a, b in zip(*out):
        assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny_b6", "p19_b37"])
def test_clipped_sum_matches_one_sample_gradients(name):
    cfg, batch, model = _setup(name)
    d = to_dev(batch)
    B = d["src"].shape[1]
    model.eval()
    per = [_module_sqnorms(model, cfg, d, b) for b in range(B)]
    norms = np.sqrt([sum(p[0]) for p in per])
    C = float(np.median(norms)) * 0.5
    L_ = float(B) + 3.0
    model.train()                 # dropout 0: the training forward is the eval forward
    # lr 0: the second norm pass below reads the step's parameters, which must still be those of its forward
    step = _step(model, batch, B, max_grad_norm=C, noise_multiplier=0.0, expected_batch_size=L_, use_graph=False, lr=0.0)
    step.step()
    torch.cuda.synchronize()
    keys = PV.sqnorm_fields(model)
    c = np.minimum(1.0, C / (norms + 1e-6))
    np.testing.assert_allclose(step.clip_factors.cpu().numpy(), c, rtol=1e-5)
    for i, k in enumerate(keys):
        ref = sum(c[b] * per[b][1][k].double() for b in range(B)) / L_
        off = step.offsets[i]
        got = step.flat_g[off:off + ref.numel()].view(ref.shape)
        assert normwise(got, ref) < 2e-3, k
    # a second norm pass over the clipped d_logits: every clipped sample's norm is C (B / L) at most
    lib = step.lib
    import ctypes as Cc
    sq2 = torch.empty_like(step.sqnorms)
    L.check(lib.rd_raindrop_v2_per_sample_grad_sqnorms(Cc.byref(step.dims), Cc.byref(step.P), L.ptr(step.static),
                                                       step.lengths.data_ptr(), step.plan.node_scale.data_ptr(),
                                                       step.ws.data_ptr(), step.d_logits.data_ptr(),
                                                       step.dp_scratch.data_ptr(), sq2.data_ptr(), L.stream_ptr()), "sqn")
    n2 = sq2.sum(1).sqrt().cpu().numpy() * L_     # norms of w_b c_b g_b (the clipped d_logits carry 1 / L)
    assert np.all(n2 <= C * (1 + 1e-5)), (n2, C)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny_b6", "p19_b37", "p12_b3"])
def test_clipped_sum_train_matches_oracle(name):
    """Dropout 0.2: the DP step's gradient bucket is (1/L) sum_b c_b g_b with g_b the float64 oracle's per-sample
    gradients under the step's own masks."""
    from oracle import dropout_masks as DM
    cfg, batch, model = _setup(name, dropout=0.2)
    model.train()
    B = batch["src"].shape[1]
    keys = PV.sqnorm_fields(model)
    d = to_dev(batch)
    gates = _gpu_gates(model, cfg, d)
    masks = DM.model_masks(RNG0, 0.2, cfg, B)
    ref_sq, ref_g, stages = _oracle_per_sample(cfg, batch, masks, keys, gates)
    _check_gates(cfg, gates, stages, masks, B)
    norms = np.sqrt(ref_sq.sum(1))
    C = float(np.median(norms)) * 0.5
    L_ = float(B) + 3.0
    step = _step(model, batch, B, max_grad_norm=C, noise_multiplier=0.0, expected_batch_size=L_, use_graph=False)
    step.step()
    torch.cuda.synchronize()
    c = np.minimum(1.0, C / (norms + 1e-6))
    np.testing.assert_allclose(step.clip_factors.cpu().numpy(), c, rtol=1e-4)
    for i, k in enumerate(keys):
        ref = sum(c[b] * ref_g[b][k] for b in range(B)) / L_
        off = step.offsets[i]
        got = step.flat_g[off:off + ref.numel()].view(ref.shape).double().cpu()
        assert normwise(got, ref) < 1e-4, (k, normwise(got, ref))       # test_train_parity.TIGHT


@pytest.mark.gpu
def test_zero_weight_slots_change_nothing():
    cfg = model_config("P19", dropout=0.0)
    B, keep = 12, [0, 2, 3, 7, 8, 11]
    batch = make_batch(cfg, B, seed=8)
    sub = {k: (None if v is None else (v[:, keep] if v.dim() >= 2 and k in ("src", "times") else v[keep]))
           for k, v in batch.items()}
    grads = []
    for bt, n in ((batch, B), (sub, len(keep))):
        model = build_dropin(cfg, 21).train()
        model._prepare(torch.device("cuda")).obprop_mode = EXACT
        s = _step(model, bt, n, max_grad_norm=0.05, noise_multiplier=0.0, expected_batch_size=10.0, use_graph=False)
        if n == B:
            w = torch.zeros(B)
            w[keep] = 1
            s.weight.copy_(w)
        s.step()
        torch.cuda.synchronize()
        grads.append((s.flat_g.clone(), s.loss.item()))
    assert normwise(grads[0][0], grads[1][0]) < 1e-5
    assert abs(grads[0][1] - grads[1][1]) < 1e-5 * abs(grads[1][1])


@pytest.mark.gpu
def test_noise_stream():
    cfg = model_config("P19", dropout=0.0)
    B = 8
    model = build_dropin(cfg, 21).train()
    sigma, C, L_, seed = 1.3, 0.7, 5.0, 0xDEADBEEF12345678
    s = _step(model, make_batch(cfg, B, seed=1), B, max_grad_norm=C, noise_multiplier=sigma, expected_batch_size=L_,
              noise_seed=seed, use_graph=False)
    s.weight.zero_()
    key0 = s.noise_key.clone()
    s.step()
    torch.cuda.synchronize()
    g1 = s.flat_g.cpu().numpy()
    std = np.float32(sigma * C / L_)
    used = np.zeros(g1.size, dtype=bool)
    params = model.used_parameters()
    for off, p in zip(s.offsets, params):
        used[off:off + p.numel()] = True
    xi = noise_normals(seed, 0, g1.size)
    assert np.array_equal(g1[used], (std * xi)[used])
    assert np.all(g1[~used] == 0)
    z = xi[used].astype(np.float64)
    n = z.size
    assert n > 400000
    assert abs(z.mean()) < 4 / math.sqrt(n) and abs(z.std() - 1) < 4 * math.sqrt(0.5 / n)
    assert s.noise_key.cpu().numpy().view(np.uint64)[1] == 1
    s.step()
    torch.cuda.synchronize()
    g2 = s.flat_g.cpu().numpy()
    assert not np.array_equal(g1[used], g2[used])
    s.noise_key.copy_(key0)
    s.step()
    torch.cuda.synchronize()
    assert np.array_equal(s.flat_g.cpu().numpy(), g1)


@pytest.mark.gpu
@pytest.mark.parametrize("name,widths", [("p19_b37", [None, None, 48, 152, 232]), ("pam_b2", [None, None, 64, 160, 256])])
def test_sqnorms_and_bucket_deterministic(name, widths):
    """Two runs, and runs under every forced tc_nt tile width (RD_TC_NT_BN, tests/test_tc_nt_tiling.py), give bitwise
    the same norms and bucket."""
    import os
    cfg, batch, _ = _setup(name, dropout=0.2)
    mode = EXACT if name == "p19_b37" else 1       # the widths listed are those of the mode
    runs = []
    for bn in widths:
        model = build_dropin(cfg, 21).train()
        plan = model._prepare(torch.device("cuda"))
        plan.obprop_mode = mode
        plan.rng_state.copy_(torch.tensor(RNG0, dtype=torch.int64))
        B = batch["src"].shape[1]
        s = _step(model, batch, B, max_grad_norm=0.1, noise_multiplier=0.5, expected_batch_size=B, noise_seed=3,
                  use_graph=False)
        try:
            if bn is not None:
                os.environ["RD_TC_NT_BN"] = str(bn)
            s.step()
            torch.cuda.synchronize()
        finally:
            os.environ.pop("RD_TC_NT_BN", None)
        runs.append((s.sqnorms.clone(), s.flat_g.clone()))
    for sq, g in runs[1:]:
        assert torch.equal(runs[0][0], sq) and torch.equal(runs[0][1].view(torch.int32), g.view(torch.int32))
