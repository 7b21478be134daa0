"""TracIn training-data influence (raindrop_b200.influence): per-sample gradient rows and their inner products."""
import json
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import GATE_SITES, build_dropin, gate_disagreements, normwise, read_gpu, to_dev
from raindrop_b200 import influence as IF
from raindrop_b200 import lib as L
from raindrop_b200 import privacy as PV
from raindrop_b200.synth import make_batch, model_config, used_param_keys

EXACT, FAST = 2, 1
HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "raindrop_b200.h")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "per_sample_grads.npz")
GRAD_TOL_EXACT = 2e-3          # as tests/test_gpu_parity.py: fp32 against the reference's own fp32 CPU backward
TOL_FAST = 2e-2                # as tests/test_input_grads.py: single-pass TF32 ob-prop layers against float64


# ---- host ------------------------------------------------------------------------------------------------------------------
def _cpu_model(name="TINY"):
    cfg = model_config(name, dropout=0.0)
    return cfg, build_dropin(cfg, 21, device="cpu")


@pytest.mark.parametrize("name", ["TINY", "TINY8", "P19", "PAM"])
def test_segment_planner_covers_exactly_the_selected_fields(name):
    _, m = _cpu_model(name)
    layout = IF.grad_layout(m)
    assert [k for k, _, _ in layout] == PV.sqnorm_fields(m)
    for (k, off, shape), p in zip(layout, m.used_parameters()):
        assert off % 4 == 0 and shape == tuple(p.shape)
    keys = [k for k, _, _ in layout]
    for fields in (None, keys[:1], keys[-2:], keys[::3]):
        off, ln = IF.plan_segments(layout, fields)
        assert off.dtype == np.int64 and ln.dtype == np.int64
        assert np.all(off % 4 == 0) and np.all(ln >= 1) and np.all(ln <= IF.SEGMENT)
        sel = set(keys if fields is None else fields)
        spans = {k: (o, o + math.prod(s)) for k, o, s in layout}
        for o, n in zip(off.tolist(), ln.tolist()):
            owner = [k for k, (a, b) in spans.items() if a <= o and o + n <= b]
            assert len(owner) == 1 and owner[0] in sel          # inside one selected field
        want = sum(math.prod(s) for k, _, s in layout if k in sel)
        assert int(ln.sum()) == want
        assert len(set(zip(off.tolist(), ln.tolist()))) == len(off)


def test_argument_errors_raise_on_the_host():
    cfg, m = _cpu_model()
    b = make_batch(cfg, 3, seed=1)
    q = dict(src=b["src"], static=b["static"], times=b["times"], lengths=b["lengths"], y=b["y"])
    m.eval()
    with pytest.raises(ValueError):
        IF.plan_segments(IF.grad_layout(m), ["no.such.field"])
    with pytest.raises(ValueError):
        IF.plan_segments(IF.grad_layout(m), [])
    with pytest.raises(ValueError):
        IF.tracin(m, q, q, internal_batch_size=0)
    with pytest.raises(ValueError):
        IF.tracin(m, q, dict(q, y=None))                      # train labels are required
    with pytest.raises(ValueError):
        IF.tracin(m, q, q, checkpoints=[({}, 1.0)])           # missing tensors
    with pytest.raises(ValueError):
        IF.tracin(m, q, q, checkpoints=[(m.state_dict(), float("nan"))])
    with pytest.raises(ValueError):
        IF.per_sample_grads(m, b["src"], b["static"], b["times"], b["lengths"], torch.tensor([0, 1, 2]))
    m.train()
    with pytest.raises(ValueError):
        IF.per_sample_grads(m, b["src"], b["static"], b["times"], b["lengths"], b["y"])
    with pytest.raises(ValueError):
        IF.tracin(m, q, q)


def test_entry_points_raise_without_cuda():
    if torch.cuda.is_available():
        pytest.skip("checks the CPU-only behaviour")
    cfg, m = _cpu_model()
    m.eval()
    b = make_batch(cfg, 3, seed=1)
    q = dict(src=b["src"], static=b["static"], times=b["times"], lengths=b["lengths"], y=b["y"])
    with pytest.raises(L.RaindropB200Error):
        IF.per_sample_grads(m, b["src"], b["static"], b["times"], b["lengths"], b["y"])
    with pytest.raises(L.RaindropB200Error):
        IF.tracin(m, q, q)
    with pytest.raises(L.RaindropB200Error):
        IF.self_influence(m, q)


def test_tracin_from_grads_weights_checkpoints():
    rng = np.random.default_rng(0)
    Gq, Gt, lrs = rng.normal(size=(3, 4, 50)), rng.normal(size=(3, 6, 50)), np.array([0.5, 1e-3, 2.0])
    got = IF.tracin_from_grads(Gq, Gt, lrs)
    ref = sum(lrs[c] * Gq[c] @ Gt[c].T for c in range(3))
    np.testing.assert_allclose(got, ref, rtol=1e-13, atol=0)
    np.testing.assert_allclose(IF.tracin_from_grads(Gq[1], Gt[1], 1e-3), 1e-3 * Gq[1] @ Gt[1].T, rtol=1e-13)
    with pytest.raises(ValueError):
        IF.tracin_from_grads(Gq, Gt[:2], lrs)


def _golden():
    z = np.load(GOLDEN)
    return z, json.loads(bytes(z["meta"]).decode())


def test_tracin_from_grads_reproduces_the_golden_matrix():
    z, meta = _golden()
    for name, cfg_name, B, seed in meta["cases"]:
        _, m = _cpu_model(cfg_name)
        layout = IF.grad_layout(m)
        assert sorted(k for k, _, _ in layout) == sorted(used_param_keys(model_config(cfg_name)))
        assert z[name + ".field_l2"].shape == (B, len(layout))
        if name in meta["full"]:
            G = z[name + ".G"]
            assert G.shape == (B, IF._bucket_length(layout))
            np.testing.assert_allclose(IF.tracin_from_grads(G, G, 1.0), z[name + ".tracin"], rtol=1e-12, atol=0)
            np.testing.assert_allclose(IF.tracin_from_grads([G, G], [G, G], [0.25, 0.5]), 0.75 * z[name + ".tracin"],
                                       rtol=1e-12, atol=0)
            l2 = np.array([[np.linalg.norm(G[b, o:o + math.prod(sh)]) for _, o, sh in layout] for b in range(B)])
            np.testing.assert_allclose(l2, z[name + ".field_l2"], rtol=1e-12)


def test_device_dataset_is_checked_against_the_model_on_the_host():
    from raindrop_b200.data import DeviceDataset
    cfg, m = _cpu_model()
    m.eval()
    b = make_batch(cfg, 4, seed=1)
    q = dict(src=b["src"], static=b["static"], times=b["times"], lengths=b["lengths"], y=b["y"])
    mk = lambda src, st, tm, y: DeviceDataset(src, st, tm, y, device="cpu")
    bad = [
        mk(b["src"][:-1], b["static"], b["times"][:-1], b["y"]),                 # shorter T
        mk(b["src"][:, :, :-2], b["static"], b["times"], b["y"]),                # narrower
        mk(b["src"], b["static"][:, :-1], b["times"], b["y"]),                   # static width
        mk(b["src"], b["static"], b["times"], torch.tensor([0, 1, 2, 1])),      # label out of range (2 classes)
        mk(b["src"], b["static"], b["times"], torch.tensor([0, -1, 0, 1])),
        mk(b["src"], b["static"], b["times"], None),                             # no labels
    ]
    for ds in bad:
        with pytest.raises(ValueError):
            IF.tracin(m, q, ds)
        with pytest.raises(ValueError):
            IF.self_influence(m, ds)
    ok = mk(b["src"], b["static"], b["times"], torch.tensor([0, 1, 5, 1]))
    for idx in ([0, 4], [-1], [0.5]):
        with pytest.raises(ValueError):
            IF.tracin(m, q, (ok, torch.tensor(idx)))
    with pytest.raises(ValueError):
        IF.tracin(m, q, (ok, torch.tensor([0, 2])))                              # the subset holds label 5
    with pytest.raises(ValueError):
        IF.tracin(m, q, dict(q, static=b["static"][:, :-1]))


def test_new_symbols_are_exported():
    header = open(HEADER).read()
    for name in ("rd_per_sample_grads_scratch_bytes", "rd_raindrop_v2_per_sample_grads",
                 "rd_per_sample_grad_dot_scratch_bytes", "rd_per_sample_grad_dot"):
        assert name in L.SIGNATURES and name + "(" in header
    assert "#define RD_GRAD_DOT_SEGMENT %d" % L.GRAD_DOT_SEGMENT in header
    assert L.GRAD_DOT_SEGMENT % 4 == 0 and L.ABI_VERSION == 2


# ---- GPU -------------------------------------------------------------------------------------------------------------------
CASES = {"tiny_b6": ("TINY", 6), "tiny8_b9": ("TINY8", 9), "p19_b37": ("P19", 37), "p12_b3": ("P12", 3),
         "pam_b2": ("PAM", 2)}


def _setup(name, B=None, seed=None):
    cfg_name, B0 = CASES[name]
    B = B0 if B is None else B
    cfg = model_config(cfg_name, dropout=0.2)
    batch = make_batch(cfg, B, seed=700 + B if seed is None else seed)
    model = build_dropin(cfg, 21)
    model._prepare(torch.device("cuda")).obprop_mode = EXACT
    model.eval()
    return cfg, to_dev(batch), model


def _args(d):
    return d["src"], d["static"], d["times"], d["lengths"], d["y"]


def _unflatten(model, row):
    return {k: row[o:o + math.prod(s)].view(s) for k, o, s in IF.grad_layout(model)}


def _module_grads(model, d, b):
    model.zero_grad(set_to_none=True)
    sl = slice(b, b + 1)
    st = None if d["static"] is None else d["static"][sl]
    logits, _, _ = model.forward(d["src"][:, sl], st, d["times"][:, sl], d["lengths"][sl])
    F.cross_entropy(logits, d["y"][sl]).backward()
    sd = dict(model.named_parameters())
    return {k: sd[k].grad.detach().clone() for k in PV.sqnorm_fields(model)}


def _eval_gates(model, cfg, d):
    """The ReLU decisions of the GPU's eval forward of this batch (helpers.read_gpu), for the oracle to replay: fp32 and
    float64 can land on different sides of a ReLU whose input is within rounding distance of zero."""
    plan = model._prepare(torch.device("cuda"))
    plan.debug_keep_workspace = True
    with torch.no_grad():
        model.forward(d["src"], d["static"], d["times"], d["lengths"])
    plan.debug_keep_workspace = False
    return read_gpu(cfg, plan.last_dims, plan.last_workspace)["gates"]


def _oracle_grads(cfg, d, keys, gates, tf32_model=False):
    """Per-sample gradients of the float64 oracle (weight seed 21) with the GPU's ReLU gates replayed; the replayed gates
    disagree with the oracle's own signs at no more than 1e-4 of each site's gates (test_train_parity.GATE_RATE).
    tf32_model: the oracle's TF32 rounding model of the single-pass ob-prop layers, whose signs the fast mode follows."""
    from oracle import dropout_masks as DM
    from oracle.raindrop_oracle import build_oracle_model
    from raindrop_b200.synth import synth_weights
    oracle = build_oracle_model(cfg).eval()
    synth_weights(oracle, cfg, seed=21)
    oracle.double().cuda()
    B = d["src"].shape[1]
    masks = DM.model_masks((0, 0), 0.0, cfg, B)         # p = 0: every mask keeps everything; the layers run written out
    st = None if d["static"] is None else d["static"].double()
    stages = {}
    logits, _, _ = oracle.forward_dense(d["src"].double(), st, d["times"].double(), d["lengths"], stages=stages,
                                        masks=masks, gates=gates, tf32_model=tf32_model)
    dis = gate_disagreements(cfg, gates, stages, masks, slice(0, B), B, {s_: [0, 0] for s_ in GATE_SITES})
    assert all(n <= max(1, 1e-4 * g) for n, g in dis.values()), dis
    params = dict(oracle.named_parameters())
    out = []
    for b in range(B):
        gs = torch.autograd.grad(F.cross_entropy(logits[b:b + 1], d["y"][b:b + 1]), [params[k] for k in keys],
                                 retain_graph=True)
        out.append(dict(zip(keys, gs)))
    return out


def _check_rows(model, cfg, d, tol, tf32_model=False):
    G = IF.per_sample_grads(model, *_args(d))
    B = d["src"].shape[1]
    assert G.shape == (B, IF._bucket_length(IF.grad_layout(model))) and G.dtype == torch.float32
    keys = PV.sqnorm_fields(model)
    refs = _oracle_grads(cfg, d, keys, _eval_gates(model, cfg, d), tf32_model)
    worst = 0.0
    for b in range(B):
        got = _unflatten(model, G[b])
        errs = {k: normwise(got[k], refs[b][k]) for k in keys}
        bad = {k: e for k, e in errs.items() if e > tol}
        assert not bad, (b, bad)
        worst = max(worst, max(errs.values()))
    return G, worst


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_rows_match_one_sample_backwards(name):
    cfg, d, model = _setup(name)
    if cfg["max_len"] * cfg["d_ob"] >= 1024:
        # PAM: the module's batched backward on one-sample batches (fp32, the same kernels' data-gradient chain)
        G = IF.per_sample_grads(model, *_args(d))
        keys = PV.sqnorm_fields(model)
        for b in range(d["src"].shape[1]):
            ref = _module_grads(model, d, b)
            got = _unflatten(model, G[b])
            bad = {k: normwise(got[k], ref[k]) for k in keys if normwise(got[k], ref[k]) > 1e-4}
            assert not bad, (b, bad)
    else:
        _check_rows(model, cfg, d, 1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny_b6", "p19_b37", "p12_b3"])
def test_rows_fast_mode_match_oracle(name):
    cfg, d, model = _setup(name)
    model._plan.obprop_mode = FAST
    _check_rows(model, cfg, d, TOL_FAST, tf32_model=True)


# test_hparams.py envelope points: d_ob 16 / nhead 4, nhead 1 / 4 layers, and 8 layers without statics (a full group of
# 32 weight-gradient items in one tile launch)
HPARAM_POINTS = {
    "d_ob16_nhead4": (dict(d_inp=40, d_ob=16, nhead=4, nhid=100, nlayers=1, max_len=20, d_static=3, n_classes=2), 4),
    "nhead1_4layers": (dict(d_inp=20, d_ob=4, nhead=1, nhid=200, nlayers=4, max_len=64, d_static=5, n_classes=5), 5),
    "8layers_nostatic": (dict(d_inp=7, d_ob=4, nhead=4, nhid=40, nlayers=8, max_len=24, d_static=0, n_classes=3), 3),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(HPARAM_POINTS))
def test_rows_across_hparams(name):
    from oracle.make_golden import hparam_config
    hp, B = HPARAM_POINTS[name]
    cfg = hparam_config(name, hp)
    d = to_dev(make_batch(cfg, B, seed=81))
    model = build_dropin(cfg, 21)
    model._prepare(torch.device("cuda")).obprop_mode = EXACT
    model.eval()
    G, _ = _check_rows(model, cfg, d, 1e-4)
    sq = PV.per_sample_grad_sqnorms(model, *_args(d))
    for f, (k, o, s_) in enumerate(IF.grad_layout(model)):
        got = G[:, o:o + math.prod(s_)].double().pow(2).sum(1)
        assert (((got - sq[:, f]).abs() / sq[:, f].abs().clamp(min=1e-30)) < 1e-5).all(), k


@pytest.mark.gpu
def test_rows_match_the_reference_golden():
    z, meta = _golden()
    for name, cfg_name, B, seed in meta["cases"]:
        cfg = model_config(cfg_name, dropout=0.2)
        model = build_dropin(cfg, meta["weight_seed"])
        model._prepare(torch.device("cuda")).obprop_mode = EXACT
        model.eval()
        d = to_dev(make_batch(cfg, B, seed=seed))
        G = IF.per_sample_grads(model, *_args(d)).double().cpu().numpy()
        layout = IF.grad_layout(model)
        l2 = np.array([[np.linalg.norm(G[b, o:o + math.prod(sh)]) for _, o, sh in layout] for b in range(B)])
        ref_l2 = z[name + ".field_l2"]
        assert (np.abs(l2 - ref_l2) <= GRAD_TOL_EXACT * ref_l2.max(axis=0)).all(), name
        if name in meta["full"]:
            Gr = z[name + ".G"]
            for b in range(B):
                for k, o, sh in layout:
                    n = math.prod(sh)
                    assert normwise(G[b, o:o + n], Gr[b, o:o + n]) < GRAD_TOL_EXACT, (name, b, k)
        ref_t = z[name + ".tracin"]
        assert np.abs(G @ G.T - ref_t).max() <= GRAD_TOL_EXACT * np.abs(ref_t).max(), name


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny_b6", "p19_b37", "p12_b3", "pam_b2"])
def test_row_mean_is_the_batch_gradient_and_padding_is_zero(name):
    cfg, d, model = _setup(name)
    G = IF.per_sample_grads(model, *_args(d))
    model.zero_grad(set_to_none=True)
    logits, _, _ = model.forward(d["src"], d["static"], d["times"], d["lengths"])
    F.cross_entropy(logits, d["y"]).backward()
    sd = dict(model.named_parameters())
    mean = G.double().mean(0)
    used = torch.zeros(G.shape[1], dtype=torch.bool, device=G.device)
    for k, o, s in IF.grad_layout(model):
        n = math.prod(s)
        used[o:o + n] = True
        err = normwise(mean[o:o + n], sd[k].grad.reshape(-1))
        # fp32 sums of up to 7,680 rows on either side (measured 3.5e-6 at P19, 8.6e-6 at PAM on an H100)
        assert err < 2e-5, (k, err)
    assert torch.count_nonzero(G[:, ~used]) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_row_norms_match_sqnorm_pass(name):
    cfg, d, model = _setup(name)
    G = IF.per_sample_grads(model, *_args(d)).double()
    sq = PV.per_sample_grad_sqnorms(model, *_args(d))
    for f, (k, o, s) in enumerate(IF.grad_layout(model)):
        got = G[:, o:o + math.prod(s)].pow(2).sum(1)
        rel = ((got - sq[:, f]).abs() / sq[:, f].abs().clamp(min=1e-30)).max().item()
        assert rel < 1e-5, (k, rel)


def _qt(d, y=True):
    return dict(src=d["src"], static=d["static"], times=d["times"], lengths=d["lengths"], y=d["y"] if y else None)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny_b6", "p19_b37", "p12_b3"])
def test_tracin_matches_float64_product_and_restores_the_model(name):
    cfg, d, model = _setup(name)
    _, dq, _ = _setup(name, B=5, seed=11)
    params0 = [p.detach().clone() for p in model.used_parameters()]
    rng0 = model._plan.rng_state.clone()
    keys = PV.sqnorm_fields(model)
    sd0 = model.state_dict()
    torch.manual_seed(9)
    ck = [({k: sd0[k] + 0.01 * torch.randn_like(sd0[k]) for k in keys}, 0.3), ({k: sd0[k].clone() for k in keys}, 1.7)]
    S = IF.tracin(model, _qt(dq, y=False), _qt(d), checkpoints=ck)
    assert S.dtype == torch.float64 and S.shape == (5, d["src"].shape[1])
    assert all(torch.equal(p, q) for p, q in zip(model.used_parameters(), params0))
    assert torch.equal(model._plan.rng_state, rng0) and not model.training
    # float64 product of the GPU's own rows, per checkpoint
    ref = torch.zeros_like(S)
    with IF._Weights(model) as w:
        for sd, lr in ck:
            w.load(sd)
            with torch.no_grad():
                logits, _, _ = model.forward(dq["src"], dq["static"], dq["times"], dq["lengths"])
            Gq = IF.per_sample_grads(model, *_args(dict(dq, y=logits.argmax(1)))).double()
            Gt = IF.per_sample_grads(model, *_args(d)).double()
            ref += lr * Gq @ Gt.T
            bound = 1e-5 * Gq.norm(dim=1)[:, None] * Gt.norm(dim=1)[None, :]
            one = IF.tracin(model, _qt(dq, y=False), _qt(d), checkpoints=[(sd, lr)])
            err = ((one - lr * Gq @ Gt.T).abs() / (abs(lr) * bound / 1e-5)).max().item()
            assert err <= 1e-5, err
    assert ((S - ref).abs() <= 1e-5 * ref.abs().max()).all()
    # several checkpoints = the lr-weighted single-checkpoint calls
    single = sum(IF.tracin(model, _qt(dq, y=False), _qt(d), checkpoints=[c]) for c in ck)
    assert ((S - single).abs() <= 1e-12 * S.abs().max()).all()
    # a fields subset = the sum of its single-field calls
    sub = [keys[0], keys[3], keys[-1], keys[-4]]
    whole = IF.tracin(model, _qt(dq, y=False), _qt(d), fields=sub)
    parts = sum(IF.tracin(model, _qt(dq, y=False), _qt(d), fields=[k]) for k in sub)
    assert ((whole - parts).abs() <= 1e-12 * whole.abs().max()).all()


@pytest.mark.gpu
def test_tracin_bitwise_across_chunking_sources_and_runs():
    from raindrop_b200.data import DeviceDataset
    cfg, d, model = _setup("p19_b37", B=300, seed=5)
    _, dq, _ = _setup("p19_b37", B=150, seed=6)
    ref = IF.tracin(model, _qt(dq), _qt(d))
    diff = lambda s: (s - ref).abs().max().item()
    again = IF.tracin(model, _qt(dq), _qt(d))
    assert torch.equal(ref, again), diff(again)
    for ibs in (1, 129, 300):          # row batch 128 at P19: blocks of 128, 256 and 384 rows
        got = IF.tracin(model, _qt(dq), _qt(d), internal_batch_size=ibs)
        assert torch.equal(ref, got), (ibs, diff(got))
    ds = DeviceDataset(d["src"], d["static"], d["times"], d["y"])
    got = IF.tracin(model, _qt(dq), ds, internal_batch_size=100)
    assert torch.equal(ref, got), diff(got)
    idx = torch.tensor([5, 0, 299, 17])          # a subset runs its rows in other batches: equal to fp32 level
    got = IF.tracin(model, _qt(dq), (ds, idx))
    assert ((got - ref[:, idx]).abs() <= 1e-5 * ref.abs().max()).all()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny_b6", "p19_b37", "pam_b2"])
def test_tracin_diagonal_is_self_influence(name):
    cfg, d, model = _setup(name)
    keys = PV.sqnorm_fields(model)
    for fields in (None, keys[2:5]):
        S = IF.tracin(model, _qt(d), _qt(d), fields=fields)
        si = IF.self_influence(model, _qt(d), fields=fields)
        rel = ((S.diagonal() - si).abs() / si.abs()).max().item()
        assert rel < 1e-5, (fields, rel)


@pytest.mark.gpu
def test_full_size_p19_against_float64_product():
    cfg = model_config("P19", dropout=0.2)
    model = build_dropin(cfg, 21)
    model.eval()
    dq = to_dev(make_batch(cfg, 128, seed=41))
    dt = to_dev(make_batch(cfg, 4096, seed=42))
    S = IF.tracin(model, _qt(dq, y=False), _qt(dt))
    assert torch.isfinite(S).all()
    g = torch.Generator().manual_seed(3)
    qi, ti = torch.randint(0, 128, (64,), generator=g), torch.randint(0, 4096, (64,), generator=g)
    with torch.no_grad():
        logits, _, _ = model.forward(dq["src"], dq["static"], dq["times"], dq["lengths"])
    pred = logits.argmax(1)
    sub = lambda dd, i: {k: (None if v is None else (v[:, i] if k in ("src", "times") else v[i])) for k, v in dd.items()}
    Gq = IF.per_sample_grads(model, *_args(dict(sub(dq, qi.cuda()), y=pred[qi.cuda()]))).double()
    Gt = IF.per_sample_grads(model, *_args(sub(dt, ti.cuda()))).double()
    ref = (Gq * Gt).sum(1)
    got = S[qi.cuda(), ti.cuda()]
    err = ((got - ref).abs() / (Gq.norm(dim=1) * Gt.norm(dim=1))).max().item()
    assert err <= 1e-5, err


@pytest.mark.gpu
@pytest.mark.parametrize("name,nq,nt", [("PAM", 16, 64), ("LARGE", 8, 32)])
def test_large_shapes_complete_within_the_scratch_plan(name, nq, nt):
    cfg = model_config(name, dropout=0.2)
    model = build_dropin(cfg, 21)
    model.eval()
    dq = to_dev(make_batch(cfg, nq, seed=51))
    dt = to_dev(make_batch(cfg, nt, seed=52))
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    S = IF.tracin(model, _qt(dq, y=False), _qt(dt))
    assert S.shape == (nq, nt) and torch.isfinite(S).all()
    assert torch.cuda.max_memory_allocated() - base < 4 * (1 << 30)
