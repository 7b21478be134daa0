"""TRAK training-data attribution (raindrop_b200.influence.trak*): host checks and the float64 restatement, and on the GPU
the margin seed, the margin rows, the fp64 Gram and rotation kernels and the scores."""
import json
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import GATE_SITES, build_dropin, gate_disagreements, normwise, to_dev
from raindrop_b200 import influence as IF
from raindrop_b200 import lib as L
from raindrop_b200 import privacy as PV
from raindrop_b200.synth import make_batch, model_config

HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "raindrop_b200.h")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "trak_margin_grads.npz")
GRAD_TOL_EXACT = 2e-3          # as tests/test_influence.py: fp32 rows against the reference's own fp32 CPU backward
ROW_TOL = 1e-4                 # as tests/test_influence.py: rows against the float64 oracle with the ReLU gates replayed
EXACT = 2
NEW_SYMBOLS = ("rd_trak_margin_seed", "rd_trak_gram", "rd_trak_rotate")


def _cpu_model(name="TINY"):
    cfg = model_config(name, dropout=0.0)
    m = build_dropin(cfg, 21, device="cpu")
    m.eval()
    return cfg, m


def _q(b, y=True):
    return dict(src=b["src"], static=b["static"], times=b["times"], lengths=b["lengths"], y=b["y"] if y else None)


def _features(model, M=1, n=5, dim=128, **kw):
    layout = tuple((k, tuple(s)) for k, _, s in IF.grad_layout(model))
    fp = IF._fingerprint(model.used_parameters())
    base = dict(features=torch.zeros(M, n, dim), eigenvalues=torch.ones(M, dim, dtype=torch.float64),
                eigenvectors=torch.eye(dim, dtype=torch.float64).repeat(M, 1, 1), Q=torch.ones(M, n, dtype=torch.float64),
                dim=dim, seed=3, fields=None, layout=layout, fingerprints=(fp,) * M)
    base.update(kw)
    return IF.TRAKFeatures(**base)


# ---- host ------------------------------------------------------------------------------------------------------------------
def test_new_symbols_are_declared_and_exported():
    header = open(HEADER).read()
    for name in NEW_SYMBOLS:
        assert name in L.SIGNATURES and name + "(" in header
    assert "#define RD_TRAK_DIM_MAX %d" % L.TRAK_DIM_MAX in header
    lib = L.load()
    for name in NEW_SYMBOLS:
        assert hasattr(lib, name)
    assert L.ABI_VERSION == 2 and lib.rd_abi_version() == 2
    for name in ("per_sample_margin_grads", "trak_features", "trak", "trak_self_influence", "trak_from_features",
                 "trak_weights", "TRAKFeatures"):
        assert hasattr(IF, name)


def test_kernels_refuse_bad_sizes_before_any_launch():
    lib = L.load()
    for dim in (0, 64, 100, 8192 + 128):
        assert lib.rd_trak_gram(16, 3, dim, 16, None) == -2
        assert lib.rd_trak_rotate(16, 3, dim, 16, 16, None) == -2
    assert lib.rd_trak_gram(16, -1, 128, 16, None) == -2
    assert lib.rd_trak_gram(4, 3, 128, 16, None) == -2                       # misaligned Phi
    assert lib.rd_trak_rotate(16, 65535 * 64 + 1, 128, 16, 16, None) == -2
    assert lib.rd_trak_margin_seed(16, 3, 1, 16, 16, 16, None) == -2          # one class has no margin
    assert b"rd_trak_margin_seed" in lib.rd_last_error_string()
    assert lib.rd_trak_gram(16, 0, 128, 16, None) == 0 and lib.rd_trak_margin_seed(16, 0, 2, 16, 16, 16, None) == 0


def test_argument_errors_raise_on_the_host():
    cfg, m = _cpu_model()
    b = make_batch(cfg, 3, seed=1)
    q = _q(b)
    for dim in (0, 64, 100, 8192 + 128, 2.5, True):
        with pytest.raises(ValueError):
            IF.trak_features(m, q, dim=dim)
    for seed in (-1, 2 ** 64):
        with pytest.raises(ValueError):
            IF.trak_features(m, q, seed=seed)
    with pytest.raises(ValueError):
        IF.trak_features(m, dict(q, y=None))                         # training labels are required
    with pytest.raises(ValueError):
        IF.trak_features(m, dict(q, y=torch.tensor([0, 2, 1])))      # label out of range (2 classes)
    with pytest.raises(ValueError):
        IF.per_sample_margin_grads(m, b["src"], b["static"], b["times"], b["lengths"], torch.tensor([0, -1, 1]))
    with pytest.raises(ValueError):
        IF.trak_features(m, q, internal_batch_size=0)
    with pytest.raises(ValueError):
        IF.trak_features(m, q, checkpoints=[(m.state_dict(), 1.0)])  # state dicts, not TracIn's (sd, lr) pairs
    with pytest.raises(ValueError):
        IF.trak_features(m, q, fields=["no.such.field"])
    f = _features(m)
    for bad in (-1.0, float("inf"), float("nan"), "1", True, None):
        with pytest.raises(ValueError):
            IF.trak(m, q, f, damping=bad)
        with pytest.raises(ValueError):
            IF.trak_self_influence(f, damping=bad)
        with pytest.raises(ValueError):
            IF.trak_weights(torch.ones(1, 128), damping=bad)
    for bad in (-1e-3, float("nan"), "x"):
        with pytest.raises(ValueError):
            IF.trak(m, q, f, rcond=bad)
    with pytest.raises(TypeError):
        IF.trak(m, q, "features")
    m.train()
    for call in (lambda: IF.trak_features(m, q), lambda: IF.trak(m, q, f),
                 lambda: IF.per_sample_margin_grads(m, b["src"], b["static"], b["times"], b["lengths"])):
        with pytest.raises(ValueError):
            call()


def test_features_that_do_not_match_are_refused():
    cfg, m = _cpu_model()
    q = _q(make_batch(cfg, 3, seed=1))
    keys = PV.sqnorm_fields(m)
    refused = [
        _features(m, fingerprints=("0" * 64,)),                                     # other weights
        _features(m, M=2),                                                          # two models, one given
        _features(m, dim=100, features=torch.zeros(1, 5, 100)),                     # dim not a multiple of 128
        _features(m, dim=256, features=torch.zeros(1, 5, 128)),                     # dim against the features' 128
        _features(m, seed=-1),                                                      # no valid projection seed
        _features(m, fields=("no.such.field",)),
        _features(m, layout=_features(m).layout[:-1]),
        _features(m, Q=torch.ones(1, 4, dtype=torch.float64)),
    ]
    for f in refused:
        with pytest.raises(ValueError):
            IF.trak(m, q, f)
    _, m8 = _cpu_model("TINY8")
    q8 = _q(make_batch(model_config("TINY8", dropout=0.0), 2, seed=1))
    with pytest.raises(ValueError, match="layout"):
        IF.trak(m8, q8, _features(m))
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    with pytest.raises(ValueError, match="other weights"):
        IF.trak(m, q, _features(m), checkpoints=[{k: v + (1.0 if k == keys[0] else 0.0) for k, v in sd.items()}])
    with pytest.raises(ValueError, match="models"):
        IF.trak(m, q, _features(m), checkpoints=[sd, sd])


def test_entry_points_raise_without_cuda():
    if torch.cuda.is_available():
        pytest.skip("checks the CPU-only behaviour")
    cfg, m = _cpu_model()
    b = make_batch(cfg, 3, seed=1)
    q = _q(b)
    with pytest.raises(L.RaindropB200Error):
        IF.per_sample_margin_grads(m, b["src"], b["static"], b["times"], b["lengths"], b["y"])
    with pytest.raises(L.RaindropB200Error):
        IF.trak_features(m, q, dim=128)
    with pytest.raises(L.RaindropB200Error):
        IF.trak(m, q, _features(m))
    with pytest.raises(L.RaindropB200Error):
        IF.trak_self_influence(_features(m))


def test_features_save_load_round_trip(tmp_path):
    _, m = _cpu_model()
    g = torch.Generator().manual_seed(0)
    f = _features(m, M=2, n=4, features=torch.randn(2, 4, 128, generator=g),
                  eigenvalues=torch.rand(2, 128, generator=g, dtype=torch.float64),
                  eigenvectors=torch.randn(2, 128, 128, generator=g, dtype=torch.float64),
                  Q=torch.rand(2, 4, generator=g, dtype=torch.float64), seed=2 ** 63 + 5, fields=tuple(PV.sqnorm_fields(m)[:2]))
    p = str(tmp_path / "f.pt")
    f.save(p)
    r = IF.TRAKFeatures.load(p)
    for name in ("features", "eigenvalues", "eigenvectors", "Q"):
        a, b = getattr(r, name), getattr(f, name)
        assert torch.equal(a, b) and a.dtype == b.dtype, name
    for name in ("dim", "seed", "fields", "layout", "fingerprints"):
        assert getattr(r, name) == getattr(f, name), name
    f.fields = None
    f.save(p)
    assert IF.TRAKFeatures.load(p, map_location="cpu").fields is None


def test_weights_follow_the_pseudo_inverse_rule():
    lam = np.array([[-1e-20, 1e-15, 1e-3, 1.0, 4.0]])
    w = IF.trak_weights(lam)
    np.testing.assert_array_equal(w, [[0.0, 0.0, 1e3, 1.0, 0.25]])           # rcond = 5 * 2^-52 of the largest
    np.testing.assert_allclose(IF.trak_weights(lam, damping=1.0), [[0, 0, 1 / 1.001, 0.5, 0.2]], rtol=1e-15)
    np.testing.assert_array_equal(IF.trak_weights(lam, rcond=0.01)[0, :3], 0.0)
    assert not IF.trak_weights(np.zeros((2, 8))).any()                          # an all-zero sketch keeps nothing


@pytest.mark.parametrize("n,dim", [(7, 24), (60, 16)])
def test_unweighted_train_scores_are_a_hat_matrix(n, dim):
    rng = np.random.default_rng(n)
    Phi = rng.normal(size=(n, dim)) * np.exp(rng.uniform(-3, 3, size=dim))
    if n > dim:
        Phi[:, -3:] = Phi[:, :3] @ rng.normal(size=(3, 3))                  # rank dim - 3
    H = IF.trak_from_features(Phi, Phi, np.ones(n))
    rank = np.linalg.matrix_rank(Phi)
    assert rank == min(n, dim) - (3 if n > dim else 0)
    np.testing.assert_allclose(H, H.T, atol=1e-10)
    np.testing.assert_allclose(H @ H, H, atol=1e-9)
    assert abs(np.trace(H) - rank) < 1e-9
    # Q scales the training columns
    Q = rng.uniform(0.1, 0.9, size=n)
    np.testing.assert_allclose(IF.trak_from_features(Phi, Phi, Q), H * Q[None, :], rtol=1e-12, atol=1e-14)


def test_large_damping_tends_to_the_weighted_inner_products():
    rng = np.random.default_rng(3)
    Fq, Ft, Q = rng.normal(size=(4, 32)), rng.normal(size=(50, 32)), rng.uniform(0, 1, size=50)
    for d in (1e6, 1e9):
        got = d * IF.trak_from_features(Fq, Ft, Q, damping=d)
        ref = (Fq @ Ft.T) * Q[None, :]
        err = np.abs(got - ref).max() / np.abs(ref).max()
        assert err < 1e3 / d, (d, err)        # relative error ~ max(lambda) / damping


def test_models_combine_as_defined():
    rng = np.random.default_rng(4)
    M, nq, nt, dim = 3, 4, 20, 12
    Fq, Ft = rng.normal(size=(M, nq, dim)), rng.normal(size=(M, nt, dim))
    Q = rng.uniform(0.05, 0.95, size=(M, nt))
    per = [IF.trak_from_features(Fq[k], Ft[k], np.ones(nt), damping=0.5) for k in range(M)]
    want = sum(per) / M * Q.mean(axis=0)[None, :]
    np.testing.assert_allclose(IF.trak_from_features(Fq, Ft, Q, damping=0.5), want, rtol=1e-12, atol=1e-14)
    mean_of_scores = sum(p * Q[k][None, :] for k, p in enumerate(per)) / M
    assert np.abs(want - mean_of_scores).max() > 1e-3 * np.abs(want).max()
    with pytest.raises(ValueError):
        IF.trak_from_features(Fq, Ft[:2], Q)


def _golden():
    z = np.load(GOLDEN)
    return z, json.loads(bytes(z["meta"]).decode())


def test_golden_margin_rows_satisfy_the_loss_identity():
    """The reference's margin rows of the fixture: Q = sigmoid(-m) in (0, 1), rows in the gradient-row layout."""
    z, meta = _golden()
    for name, cfg_name, B, _ in meta["cases"]:
        _, m = _cpu_model(cfg_name)
        assert z[name + ".G"].shape == (B, IF._bucket_length(IF.grad_layout(m)))
        assert ((z[name + ".Q"] > 0) & (z[name + ".Q"] < 1)).all()


# ---- GPU -------------------------------------------------------------------------------------------------------------------
def _seed(logits, y):
    B, C = logits.shape
    d = torch.empty(B, C, dtype=torch.float32, device="cuda")
    Q = torch.empty(B, dtype=torch.float64, device="cuda")
    L.check(L.load().rd_trak_margin_seed(logits.data_ptr(), B, C, y.data_ptr(), d.data_ptr(), Q.data_ptr(),
                                         L.stream_ptr()), "rd_trak_margin_seed")
    return d, Q


def _margin64(z, y):
    z = z.double()
    rest = z.clone()
    rest[torch.arange(len(y)), y] = float("-inf")
    return z.gather(1, y[:, None])[:, 0] - torch.logsumexp(rest, dim=1)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [2, 8])
def test_margin_seed_against_float64(C):
    g = torch.Generator().manual_seed(C)
    B = 300
    z = torch.randn(B, C, generator=g) * 4
    y = torch.randint(0, C, (B,), generator=g)
    z[:20] *= 1e3                                          # saturated: p_y -> 1 or 0
    z[20:30] = 0.0                                         # ties
    z[30:40, :] = -80.0
    z[30:40].scatter_(1, y[30:40, None], 80.0)             # p_y = 1 - 1e-70
    d, Q = _seed(z.cuda(), y.cuda())
    d, Q = d.cpu().double(), Q.cpu()
    assert torch.isfinite(d).all() and torch.isfinite(Q).all() and (Q >= 0).all() and (Q <= 1).all()
    zr = z.double().requires_grad_(True)
    m = _margin64(zr, y)
    (grad,) = torch.autograd.grad(m.sum(), zr)
    ref = grad / B
    assert ((d - ref).abs() <= 2 ** -24 * ref.abs() + 2.0 ** -149).all()      # one fp32 rounding (subnormals absolute)
    mref = _margin64(z, y)
    Qref = torch.sigmoid(-mref)
    assert ((Q - Qref).abs() <= 1e-12 * Qref + 1e-300).all()
    assert (Q[30:40] > 0).all() and (Q[30:40] < 1e-60).all()
    big = ref.abs() > 1e-30
    assert torch.equal(torch.sign(d[big]), torch.sign(ref[big]))
    # d CE / d logits = -Q d m / d logits
    ce = (torch.softmax(z.double(), 1) - F.one_hot(y, C).double()) / B
    assert ((ce - (-Q[:, None] * ref)).abs() <= 1e-12 / B).all()


def _oracle_margin_grads(cfg, d, keys, gates):
    """Per-sample margin gradients of the float64 oracle (weight seed 21) with the GPU's ReLU gates replayed."""
    from oracle import dropout_masks as DM
    from oracle.raindrop_oracle import build_oracle_model
    from raindrop_b200.synth import synth_weights
    oracle = build_oracle_model(cfg).eval()
    synth_weights(oracle, cfg, seed=21)
    oracle.double().cuda()
    B = d["src"].shape[1]
    masks = DM.model_masks((0, 0), 0.0, cfg, B)
    st = None if d["static"] is None else d["static"].double()
    stages = {}
    logits, _, _ = oracle.forward_dense(d["src"].double(), st, d["times"].double(), d["lengths"], stages=stages,
                                        masks=masks, gates=gates)
    dis = gate_disagreements(cfg, gates, stages, masks, slice(0, B), B, {s_: [0, 0] for s_ in GATE_SITES})
    assert all(n <= max(1, 1e-4 * g) for n, g in dis.values()), dis
    params = dict(oracle.named_parameters())
    m = _margin64(logits, d["y"])
    out = []
    for b in range(B):
        out.append(dict(zip(keys, torch.autograd.grad(m[b], [params[k] for k in keys], retain_graph=True))))
    return out, torch.sigmoid(-m.detach())


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


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny_b6", "tiny8_b9", "p19_b37", "p12_b3"])
def test_margin_rows_against_the_float64_oracle(name):
    from test_influence import _eval_gates, _unflatten
    cfg, d, model = _setup(name)
    G, Q = IF.per_sample_margin_grads(model, *_args(d))
    assert G.dtype == torch.float32 and Q.dtype == torch.float64
    keys = PV.sqnorm_fields(model)
    refs, Qref = _oracle_margin_grads(cfg, d, keys, _eval_gates(model, cfg, d))
    assert ((Q - Qref).abs() <= 1e-5 * Qref.clamp_min(1e-3)).all(), (Q, Qref)
    for b in range(d["src"].shape[1]):
        got = _unflatten(model, G[b])
        bad = {k: normwise(got[k], refs[b][k]) for k in keys if normwise(got[k], refs[b][k]) > ROW_TOL}
        assert not bad, (b, bad)


@pytest.mark.gpu
def test_margin_rows_match_the_reference_golden():
    z, meta = _golden()
    for name, cfg_name, B, seed in meta["cases"]:
        cfg = model_config(cfg_name, dropout=0.2)
        model = build_dropin(cfg, meta["weight_seed"])
        model._prepare(torch.device("cuda")).obprop_mode = EXACT
        model.eval()
        d = to_dev(make_batch(cfg, B, seed=seed))
        G, Q = IF.per_sample_margin_grads(model, *_args(d))
        G = G.double().cpu().numpy()
        np.testing.assert_allclose(Q.cpu().numpy(), z[name + ".Q"], rtol=GRAD_TOL_EXACT)
        Gr = z[name + ".G"]
        for b in range(B):
            for k, o, sh in IF.grad_layout(model):
                n = math.prod(sh)
                assert normwise(G[b, o:o + n], Gr[b, o:o + n]) < GRAD_TOL_EXACT, (name, b, k)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_loss_rows_are_minus_q_times_margin_rows(name):
    cfg, d, model = _setup(name)
    Gm, Q = IF.per_sample_margin_grads(model, *_args(d))
    Gl = IF.per_sample_grads(model, *_args(d))
    ok = (Q > 0.02) & (Q < 0.98)
    assert ok.any()
    for b in torch.nonzero(ok)[:, 0].tolist():
        err = normwise(Gl[b].double(), -Q[b] * Gm[b].double())
        assert err < ROW_TOL, (b, err)
    # y None: the predicted class; with 2 classes its margin is >= 0, so Q <= 1/2
    _, Qp = IF.per_sample_margin_grads(model, *_args(dict(d, y=None)))
    assert torch.isfinite(Qp).all() and (cfg["n_classes"] > 2 or (Qp <= 0.5).all())


def _gram(Phi, K=None):
    n, dim = Phi.shape
    K = torch.zeros(dim, dim, dtype=torch.float64, device="cuda") if K is None else K
    L.check(L.load().rd_trak_gram(Phi.data_ptr(), n, dim, K.data_ptr(), L.stream_ptr()), "rd_trak_gram")
    return K


def _rotate(Phi, V):
    out = torch.full(Phi.shape, float("nan"), dtype=torch.float32, device="cuda")
    L.check(L.load().rd_trak_rotate(Phi.data_ptr(), Phi.shape[0], Phi.shape[1], V.data_ptr(), out.data_ptr(),
                                    L.stream_ptr()), "rd_trak_rotate")
    return out


def _operand(n, dim, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, dim, generator=g) * torch.exp2(torch.randint(-8, 9, (n, dim), generator=g).float())


@pytest.mark.gpu
@pytest.mark.parametrize("n,dim", [(1, 128), (37, 256), (1001, 384), (4100, 128)])
def test_gram_against_float64_symmetric_and_reproducible(n, dim):
    Phi = _operand(n, dim, n)
    K = _gram(Phi.cuda())
    ref = Phi.double().T @ Phi.double()
    err = ((K.cpu() - ref).norm() / ref.norm()).item()
    assert err <= 1e-12, err
    assert torch.equal(K, K.T)
    assert torch.equal(_gram(Phi.cuda()), K)
    # another allocation, and K += on a symmetric start
    buf = torch.empty(n * dim + 64, dtype=torch.float32, device="cuda")
    buf[16:16 + n * dim] = Phi.reshape(-1).cuda()
    assert torch.equal(_gram(buf[16:16 + n * dim].view(n, dim)), K)
    S = torch.randn(dim, dim, dtype=torch.float64, device="cuda")
    S = S + S.T
    K2 = _gram(Phi.cuda(), S.clone())
    assert torch.equal(K2, K2.T) and torch.equal(K2, S + K)
    # rows past n contribute nothing: one zero row appended leaves K bitwise unchanged
    assert torch.equal(_gram(torch.cat([Phi, torch.zeros(1, dim)]).cuda()), K)


@pytest.mark.gpu
def test_gram_completes_from_128_to_8192():
    for dim in (128, 1024, 4096, 8192):
        Phi = _operand(300, dim, dim).cuda()
        K = _gram(Phi)
        d = Phi.double().pow(2).sum(0)
        assert torch.isfinite(K).all() and torch.equal(K, K.T)
        assert ((K.diagonal() - d).abs() <= 1e-12 * d).all(), dim


@pytest.mark.gpu
@pytest.mark.parametrize("n,dim", [(1, 128), (70, 256), (300, 512)])
def test_rotation_rounds_once_and_is_bitwise_per_row(n, dim):
    Phi = _operand(n, dim, 7 * n).cuda()
    V = torch.linalg.qr(torch.randn(dim, dim, dtype=torch.float64, generator=torch.Generator().manual_seed(n)))[0]
    V = V.contiguous().cuda()                              # row-major, as the kernel reads it
    got = _rotate(Phi, V)
    ref = Phi.double() @ V
    bound = 2 ** -24 * ref.abs() + 1e-13 * (Phi.double().abs() @ V.abs())
    assert ((got.double() - ref).abs() <= bound).all()
    for rows in ([0], [n - 1], list(range(0, n, 3))):
        idx = torch.tensor(rows, device="cuda")
        assert torch.equal(_rotate(Phi[idx].contiguous(), V), got[idx])
    if n > 1:
        perm = torch.randperm(n, generator=torch.Generator().manual_seed(1)).cuda()
        assert torch.equal(_rotate(Phi[perm].contiguous(), V), got[perm])


@pytest.mark.gpu
def test_rotated_training_features_have_a_diagonal_gram():
    Phi = _operand(500, 256, 3).cuda()
    lam, V = IF._trak_eigh(IF._trak_gram(Phi))
    Pr = IF._trak_rotate(Phi, V)
    G = Pr.double().T @ Pr.double()
    err = ((G - torch.diag(lam)).abs().max() / lam.max()).item()
    assert err < 1e-6, err
    assert torch.equal(lam, torch.sort(lam).values)


def _device_sketch(model, d, dim, seed, fields, y=True):
    """Projected margin rows and Q of a batch at the current weights, on trak_features' own path (_trak_sketch: the
    same row batches, so bitwise the rows the features and the query blocks of trak are made of)."""
    layout = IF.grad_layout(model)
    ldg = IF._bucket_length(layout)
    R = IF._row_batch(L.load(), model._plan, ldg)
    n, fetch = IF._source(_args_dict(d, y), "data")
    seg = IF._segments(*IF.plan_segments(layout, fields))
    return IF._trak_sketch(model, fetch, n, dim, seed, seg, R * -(-n // R), R, ldg)


def _bound(Fq, Ft, Q, damping=0.0):
    """sum_j w_j |phi~_q j| |phi~_t j| times Q (one model, float64): the scale of each score's rounding."""
    lam, V = np.linalg.eigh(Ft.T @ Ft)
    w = IF.trak_weights(lam[None], damping)[0]
    return (np.abs(Fq @ V) * w) @ np.abs(Ft @ V).T * Q[None, :]


TRAK_CASES = {"tiny_b6": ("tiny_b6", 40, 256), "p19_b37": ("p19_b37", 300, 128), "p12_b3": ("p12_b3", 24, 512),
              "pam_b2": ("pam_b2", 12, 256)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(TRAK_CASES))
def test_trak_against_the_restatement_on_the_devices_features(name):
    case, nt, dim = TRAK_CASES[name]
    cfg, dt, model = _setup(case, B=nt, seed=5)
    _, dq, _ = _setup(case, B=7, seed=6)
    keys = PV.sqnorm_fields(model)
    params0 = [p.detach().clone() for p in model.used_parameters()]
    rng0 = model._plan.rng_state.clone()
    for p in model.used_parameters():
        p.grad = None
    for fields in (None, [keys[0], keys[3], keys[-1]]):
        feats = IF.trak_features(model, _args_dict(dt), dim=dim, seed=11, fields=fields)
        assert feats.features.shape == (1, nt, dim) and feats.Q.shape == (1, nt)
        S = IF.trak(model, _args_dict(dq, y=False), feats)
        assert S.dtype == torch.float64 and S.shape == (7, nt)
        Ft, Qt = _device_sketch(model, dt, dim, 11, fields)
        Fq, _ = _device_sketch(model, dq, dim, 11, fields, y=False)
        assert torch.equal(Qt, feats.Q[0])
        Ftn, Fqn, Qn = Ft.double().cpu().numpy(), Fq.double().cpu().numpy(), Qt.cpu().numpy()
        ref = IF.trak_from_features(Fqn, Ftn, Qn)
        bound = _bound(Fqn, Ftn, Qn)
        err = (np.abs(S.cpu().numpy() - ref) / bound.clip(min=1e-300)).max()
        assert err <= 1e-4, (fields, err)
    assert all(torch.equal(p, q) for p, q in zip(model.used_parameters(), params0))
    assert all(p.grad is None for p in model.used_parameters())
    assert torch.equal(model._plan.rng_state, rng0) and not model.training


def _args_dict(d, y=True):
    return dict(src=d["src"], static=d["static"], times=d["times"], lengths=d["lengths"], y=d["y"] if y else None)


@pytest.mark.gpu
def test_trak_with_damping_against_float64_rows_and_host_signs():
    from oracle.projection_signs import project_rows
    cfg, dt, model = _setup("p19_b37", B=60, seed=5)
    _, dq, _ = _setup("p19_b37", B=5, seed=6)
    dim, seed = 256, 2 ** 33 + 1
    feats = IF.trak_features(model, _args_dict(dt), dim=dim, seed=seed)
    damping = 0.1 * feats.eigenvalues.max().item()
    S = IF.trak(model, _args_dict(dq, y=False), feats, damping=damping).cpu().numpy()
    Gt, Qt = IF.per_sample_margin_grads(model, *_args(dt))
    Gq, _ = IF.per_sample_margin_grads(model, *_args(dict(dq, y=None)))
    off, ln = IF.plan_segments(IF.grad_layout(model))
    Ft = project_rows(Gt.double().cpu().numpy(), dim, seed, off, ln)
    Fq = project_rows(Gq.double().cpu().numpy(), dim, seed, off, ln)
    ref = IF.trak_from_features(Fq, Ft, Qt.cpu().numpy(), damping=damping)
    err = np.abs(S - ref).max() / np.abs(ref).max()
    assert err <= 1e-4, err


@pytest.mark.gpu
def test_trak_bitwise_across_chunking_sources_and_runs():
    from raindrop_b200.data import DeviceDataset
    cfg, dt, model = _setup("p19_b37", B=300, seed=5)
    _, dq, _ = _setup("p19_b37", B=150, seed=6)
    keys = PV.sqnorm_fields(model)
    sd0 = model.state_dict()
    torch.manual_seed(9)
    ck = [{k: (sd0[k] + 0.01 * torch.randn_like(sd0[k]) if k in keys else sd0[k].clone()) for k in sd0},
          {k: v.clone() for k, v in sd0.items()}]         # state_dict() aliases the parameters the calls load into
    ref_f = IF.trak_features(model, _args_dict(dt), checkpoints=ck, dim=512, seed=3)
    assert len(set(ref_f.fingerprints)) == 2
    ref = IF.trak(model, _args_dict(dq), ref_f, damping=1e-3, checkpoints=ck)
    ds = DeviceDataset(dt["src"], dt["static"], dt["times"], dt["y"])
    for kw, train in ((dict(), _args_dict(dt)), (dict(internal_batch_size=1), _args_dict(dt)),
                      (dict(internal_batch_size=129), ds), (dict(), (ds, torch.arange(300)))):
        f = IF.trak_features(model, train, checkpoints=ck, dim=512, seed=3, **kw)
        for name in ("features", "eigenvalues", "eigenvectors", "Q"):
            assert torch.equal(getattr(f, name), getattr(ref_f, name)), (kw, name)
    for ibs in (1, 129, 300):
        assert torch.equal(IF.trak(model, _args_dict(dq), ref_f, damping=1e-3, checkpoints=ck, internal_batch_size=ibs),
                           ref), ibs
    # two models combine as defined: the Q-free per-model scores averaged, times the mean Q
    one = [IF.trak(model, _args_dict(dq), _single(ref_f, k), damping=1e-3, checkpoints=[ck[k]]) for k in range(2)]
    qk = [ref_f.Q[k][None, :] for k in range(2)]
    want = (one[0] / qk[0] + one[1] / qk[1]) / 2 * ref_f.Q.mean(0)[None, :]
    assert ((ref - want).abs() <= 1e-12 * ref.abs().max()).all()


def _single(f, k):
    return IF.TRAKFeatures(features=f.features[k:k + 1], eigenvalues=f.eigenvalues[k:k + 1],
                           eigenvectors=f.eigenvectors[k:k + 1], Q=f.Q[k:k + 1], dim=f.dim, seed=f.seed, fields=f.fields,
                           layout=f.layout, fingerprints=f.fingerprints[k:k + 1])


@pytest.mark.gpu
@pytest.mark.parametrize("nt,dim", [(40, 256), (300, 128)])
def test_hat_matrix_identity_and_self_influence(nt, dim):
    cfg, dt, model = _setup("p19_b37", B=nt, seed=5)
    feats = IF.trak_features(model, _args_dict(dt), dim=dim, seed=1)
    S = IF.trak(model, _args_dict(dt), feats)
    Qbar = feats.Q[0]
    si = IF.trak_self_influence(feats)
    rel = ((S.diagonal() - si).abs() / si.abs().clamp_min(1e-300)).max().item()
    # the scores' dot runs 3xTF32 products (about 2^-21 relative each; measured 1.04e-6 at n 300, dim 128 on an H100)
    assert rel < 2e-6, rel
    lev = si / Qbar
    rank = int((IF.trak_weights(feats.eigenvalues) > 0).sum())
    assert rank == min(nt, dim)
    assert (lev >= -1e-6).all() and (lev <= 1 + 1e-6).all()
    assert abs(lev.sum().item() - rank) < 1e-4 * rank
    # (scores / Q-bar) Phi~ = each query's rotated feature on the kept directions
    Pr = feats.features[0].double()
    keep = torch.from_numpy(IF.trak_weights(feats.eigenvalues)[0] > 0).cuda()
    back = (S / Qbar[None, :]) @ Pr
    err = ((back - Pr)[:, keep].norm(dim=1) / Pr[:, keep].norm(dim=1)).max().item()
    assert err < 1e-4, err


@pytest.mark.gpu
@pytest.mark.parametrize("name,n", [("PAM", 24), ("LARGE", 24)])
def test_large_shapes_complete_within_the_scratch_plan(name, n):
    cfg = model_config(name, dropout=0.2)
    model = build_dropin(cfg, 21)
    model.eval()
    d = to_dev(make_batch(cfg, n, seed=52))
    dq = to_dev(make_batch(cfg, 8, seed=53))
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    f = IF.trak_features(model, _args_dict(d), dim=4096, seed=1)
    S = IF.trak(model, _args_dict(dq, y=False), f)
    assert S.shape == (8, n) and torch.isfinite(S).all() and S.abs().amax().item() > 0
    assert torch.isfinite(IF.trak_self_influence(f)).all()
    assert torch.cuda.max_memory_allocated() - base < 4 * (1 << 30)
