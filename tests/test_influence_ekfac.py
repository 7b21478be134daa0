"""EK-FAC influence functions of Raindrop_v2 (raindrop_b200.influence.ekfac_*): host checks, the numpy restatements, and
on the GPU the factors against the float64 oracle's layer operands, the rotated rows, Lambda and the scores."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch.overrides import TorchFunctionMode

from helpers import build_dropin, to_dev
from oracle.fisher_labels import fisher_labels, fisher_uniforms
from raindrop_b200 import influence as IF
from raindrop_b200 import lib as L
from raindrop_b200.synth import make_batch, model_config

HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "raindrop_b200.h")


def _cpu_model(name="TINY"):
    cfg = model_config(name, dropout=0.0)
    m = build_dropin(cfg, 21, device="cpu")
    m.eval()
    return cfg, m


def _q(b, y=True):
    return dict(src=b["src"], static=b["static"], times=b["times"], lengths=b["lengths"], y=b["y"] if y else None)


def _identity_factors(model, fields=None, lam=None):
    blocks = IF.kfac_blocks(model)
    layout = tuple((k, tuple(s)) for k, _, s in IF.grad_layout(model))
    ldg = IF._bucket_length(IF.grad_layout(model))
    bases = tuple((np.eye(kin + 1), np.eye(nout)) for _, _, nout, kin in blocks)
    return IF.EKFACFactors(bases=bases, bases_flat=IF._flat_bases(blocks, bases),
                           eigenvalues=torch.zeros(ldg, dtype=torch.float64) if lam is None else lam, n=1,
                           fisher="empirical", seed=0, fields=fields, layout=layout,
                           fingerprint=IF._fingerprint(model.used_parameters()))


# ---- host ------------------------------------------------------------------------------------------------------------------
def test_argument_checks_raise_on_the_host():
    cfg, m = _cpu_model()
    q = _q(make_batch(cfg, 3, seed=1))
    w, b, _, _ = IF.kfac_blocks(m)[1]
    with pytest.raises(ValueError):
        IF.ekfac_factors(m, q, fields=[w])                      # weight without its bias
    with pytest.raises(ValueError):
        IF.ekfac_factors(m, q, fields=[b])
    with pytest.raises(ValueError):
        IF.ekfac_factors(m, q, fisher="model")
    with pytest.raises(ValueError):
        IF.ekfac_factors(m, q, seed=-1)
    with pytest.raises(ValueError):
        IF.ekfac_factors(m, q, internal_batch_size=0)
    f = _identity_factors(m)
    for bad in (0.0, -1.0, float("inf"), float("nan"), "1", True):
        with pytest.raises(ValueError):
            IF.ekfac_influence(m, q, q, f, damping=bad)
    with pytest.raises(ValueError):
        IF.ekfac_influence(m, q, dict(q, y=None), f)             # train labels are required
    with pytest.raises(TypeError):
        IF.ekfac_influence(m, q, q, "factors")
    # factors of other weights, another layout or unsplittable fields are refused
    with torch.no_grad():
        m.used_parameters()[0].add_(1.0)
    with pytest.raises(ValueError, match="other weights"):
        IF.ekfac_influence(m, q, q, f)
    with pytest.raises(ValueError, match="other weights"):
        IF.ekfac_self_influence(m, q, f)
    with torch.no_grad():
        m.used_parameters()[0].sub_(1.0)
    _, m8 = _cpu_model("TINY8")
    with pytest.raises(ValueError, match="layout"):
        q8 = _q(make_batch(model_config("TINY8", dropout=0.0), 2, seed=1))
        IF.ekfac_influence(m8, q8, q8, f)
    g = _identity_factors(m, fields=(w,))
    with pytest.raises(ValueError):
        IF.ekfac_influence(m, q, q, g)
    m.train()
    with pytest.raises(ValueError):
        IF.ekfac_factors(m, q)


def test_entry_points_raise_without_cuda():
    if torch.cuda.is_available():
        pytest.skip("checks the CPU-only behaviour")
    cfg, m = _cpu_model()
    q = _q(make_batch(cfg, 3, seed=1))
    f = _identity_factors(m)
    with pytest.raises(L.RaindropB200Error):
        IF.ekfac_factors(m, q)
    with pytest.raises(L.RaindropB200Error):
        IF.kfac_covariances(m, q, fisher="empirical")
    with pytest.raises(L.RaindropB200Error):
        IF.ekfac_influence(m, q, q, f)
    with pytest.raises(L.RaindropB200Error):
        IF.ekfac_self_influence(m, q, f)


def test_new_symbols_are_exported():
    header = open(HEADER).read()
    for name in ("rd_kfac_factors_doubles", "rd_ekfac_bases_floats", "rd_kfac_factors_scratch_bytes",
                 "rd_raindrop_v2_kfac_factors", "rd_ekfac_rows_scratch_bytes", "rd_raindrop_v2_ekfac_rows",
                 "rd_ekfac_accumulate_sq", "rd_ekfac_scale_rows", "rd_fisher_labels", "rd_debug_fisher_uniforms"):
        assert name in L.SIGNATURES and name + "(" in header
    for name in ("ekfac_factors", "ekfac_influence", "ekfac_self_influence", "ekfac_from_grads", "EKFACFactors",
                 "kfac_covariances", "kfac_blocks"):
        assert hasattr(IF, name)
    assert L.ABI_VERSION == 2


def test_blocks_and_flat_bases_follow_the_header_layout():
    for name in ("TINY", "PAM"):
        _, m = _cpu_model(name)
        blocks = IF.kfac_blocks(m)
        assert len(blocks) == 4 * 2 + 2
        rng = np.random.default_rng(0)
        bases = tuple((rng.normal(size=(kin + 1, kin + 1)), rng.normal(size=(nout, nout))) for _, _, nout, kin in blocks[:2])
        flat = IF._flat_bases(blocks[:2], bases).double().numpy()
        off = 0
        for (_, _, nout, kin), (QA, QS) in zip(blocks[:2], bases):
            npad = (kin + 4) // 4 * 4
            np.testing.assert_allclose(flat[off:off + nout * nout].reshape(nout, nout), QS.T, rtol=1e-6)
            off += (nout * nout + 3) // 4 * 4
            qa = flat[off:off + npad * kin].reshape(npad, kin)
            np.testing.assert_allclose(qa[:kin + 1], QA[:kin].T, rtol=1e-6)
            assert not qa[kin + 1:].any()
            off += npad * kin
            np.testing.assert_allclose(flat[off:off + kin + 1], QA[kin], rtol=1e-6)
            off += npad


def test_save_load_round_trips(tmp_path):
    _, m = _cpu_model()
    ldg = IF._bucket_length(IF.grad_layout(m))
    f = _identity_factors(m, lam=torch.arange(ldg, dtype=torch.float64))
    f.fields = tuple(IF.kfac_blocks(m)[0][:2])
    p = str(tmp_path / "f.pt")
    f.save(p)
    g = IF.EKFACFactors.load(p)
    assert (g.n, g.fisher, g.seed, g.fields, g.layout, g.fingerprint) == (f.n, f.fisher, f.seed, f.fields, f.layout,
                                                                          f.fingerprint)
    assert torch.equal(g.eigenvalues, f.eigenvalues) and torch.equal(g.bases_flat, f.bases_flat)
    assert all(np.array_equal(a, c) and np.array_equal(b, d) for (a, b), (c, d) in zip(g.bases, f.bases))


def test_label_sampler_restatement_is_pinned():
    u = fisher_uniforms(4, 0)
    assert [x.hex() for x in u.tolist()] == ['0x1.f02628d357f04p-3', '0x1.278fc503c5484p-1', '0x1.c76e403be2d90p-3',
                                             '0x1.f3521aa03b256p-2']
    assert fisher_uniforms(2, 12345, index0=1 << 33).tolist() == [0.26126238914564837, 0.7654636184820666]
    assert fisher_uniforms(3, 7, index0=5)[1] == fisher_uniforms(1, 7, index0=6)[0]        # a draw depends on its index
    # u = 0.242, 0.577, 0.222, 0.488: equal logits split at 1/2; p = (0.953, 0.047) takes class 0 below 0.953;
    # a 50-logit margin takes class 1
    lg = np.array([[0., 0.], [0., 0.], [2., -1.], [0., 50.]], np.float32)
    assert fisher_labels(lg, 0).tolist() == [0, 1, 0, 1]
    assert fisher_labels(np.array([[0., 0., 0.]] * 4, np.float32), 0).tolist() == [0, 1, 0, 1]


def test_from_grads_with_identity_bases_and_large_damping_is_tracin():
    _, m = _cpu_model()
    ldg = IF._bucket_length(IF.grad_layout(m))
    rng = np.random.default_rng(1)
    Gq, Gt = rng.normal(size=(3, ldg)), rng.normal(size=(5, ldg))
    pad = np.ones(ldg, bool)
    for _, off, s in IF.grad_layout(m):
        pad[off:off + math.prod(s)] = False
    Gq[:, pad] = 0
    Gt[:, pad] = 0
    lam = torch.from_numpy(rng.uniform(0, 1, size=ldg))
    f = _identity_factors(m, lam=lam)
    big = 1e12
    got = big * IF.ekfac_from_grads(Gq, Gt, f, damping=big)
    np.testing.assert_allclose(got, IF.tracin_from_grads(Gq, Gt, 1.0), rtol=1e-9, atol=1e-9 * np.abs(got).max())
    # finite damping: the diagonal preconditioner 1 / (lam + 0.1 mean(lam) per group), exactly
    w = IF.ekfac_weights(f)
    np.testing.assert_allclose(IF.ekfac_from_grads(Gq, Gt, f), (Gq * w) @ Gt.T, rtol=1e-12)
    # rotation by random orthogonal bases keeps the plain inner product (the bases' columns are orthonormal)
    blocks = IF.kfac_blocks(m)
    bases = tuple((np.linalg.qr(rng.normal(size=(kin + 1, kin + 1)))[0], np.linalg.qr(rng.normal(size=(nout, nout)))[0])
                  for _, _, nout, kin in blocks)
    f.bases = bases
    np.testing.assert_allclose(big * IF.ekfac_from_grads(Gq, Gt, f, damping=big), Gq @ Gt.T, rtol=1e-8,
                               atol=1e-8 * np.abs(Gq @ Gt.T).max())


# ---- GPU -------------------------------------------------------------------------------------------------------------------
EXACT = 2
# the fp32 forward / backward's layer operands differ from float64 by up to ~2e-5 normwise at P19 / P12 (the rows they
# make are held to 1e-4 in test_influence.py); the factor sums add no error of that size
FACTOR_TOL = 5e-5
CASES = {"tiny_b6": ("TINY", 6), "p19_b37": ("P19", 37), "p12_b3": ("P12", 3), "pam_b2": ("PAM", 2)}


def _setup(name, B=None, seed=None):
    cfg_name, B0 = CASES[name]
    B = B0 if B is None else B
    cfg = model_config(cfg_name, dropout=0.2)
    batch = make_batch(cfg, B, seed=700 + B if seed is None else seed)
    model = build_dropin(cfg, 21)
    model._prepare(torch.device("cuda")).obprop_mode = EXACT
    model.eval()
    return cfg, to_dev(batch), model


def _rel(a, b):
    return float((a - b).norm() / b.norm())


@pytest.mark.gpu
def test_device_labels_equal_the_restatement():
    lib = L.load()
    st = L.stream_ptr()
    out = torch.empty(1000, dtype=torch.float64, device="cuda")
    for seed, i0 in ((0, 0), (2 ** 64 - 1, 2 ** 40 + 3)):
        L.check(lib.rd_debug_fisher_uniforms(seed, i0, 1000, out.data_ptr(), st), "rd_debug_fisher_uniforms")
        assert np.array_equal(out.cpu().numpy(), fisher_uniforms(1000, seed, i0))
    g = torch.Generator().manual_seed(0)
    for ncls in (2, 8):
        logits = (3 * torch.randn(777, ncls, generator=g)).float().cuda()
        y = torch.empty(777, dtype=torch.int64, device="cuda")
        L.check(lib.rd_fisher_labels(logits.data_ptr(), 777, ncls, 42, 1000, y.data_ptr(), st), "rd_fisher_labels")
        assert np.array_equal(y.cpu().numpy(), fisher_labels(logits.cpu().numpy(), 42, 1000))


class _Operands(TorchFunctionMode):
    """Records the input and output of every product with one of `weights` (the encoder's x @ W.T and the ob-prop
    layers' F.linear), so the backward's output gradients can be read from the outputs."""

    def __init__(self, weights):
        super().__init__()
        self.w = {id(p): k for k, p in weights.items()}
        self.x, self.y = {}, {}

    def __torch_function__(self, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        out = func(*args, **kwargs)
        key = None
        if func is F.linear:
            key = self.w.get(id(args[1] if len(args) > 1 else kwargs["weight"]))
        elif getattr(func, "__name__", "") in ("matmul", "__matmul__") and len(args) == 2 and \
                isinstance(args[1], torch.Tensor):
            base = args[1]._base
            if base is not None and id(base) in self.w and args[1].shape == base.T.shape:
                key = self.w[id(base)]
        if key is not None:
            assert key not in self.x, key
            self.x[key] = args[0]
            out.retain_grad()
            self.y[key] = out
        return out


def _oracle_factors(cfg, d, y, model):
    """float64 A, S per block from the oracle's layer operands, with the GPU's ReLU gates replayed."""
    from oracle import dropout_masks as DM
    from oracle.raindrop_oracle import build_oracle_model
    from raindrop_b200.synth import synth_weights
    from test_influence import _eval_gates
    gates = _eval_gates(model, cfg, d)
    oracle = build_oracle_model(cfg).eval()
    synth_weights(oracle, cfg, seed=21)
    oracle.double().cuda()
    B = d["src"].shape[1]
    masks = DM.model_masks((0, 0), 0.0, cfg, B)
    st = None if d["static"] is None else d["static"].double()
    params = dict(oracle.named_parameters())
    blocks = IF.kfac_blocks(model)
    grab = _Operands({w: params[w] for w, _, _, _ in blocks})
    with grab:
        logits, _, _ = oracle.forward_dense(d["src"].double(), st, d["times"].double(), d["lengths"], masks=masks,
                                            gates=gates)
    F.cross_entropy(logits, y, reduction="sum").backward()
    out = []
    for w, _, nout, kin in blocks:
        x = grab.x[w].detach().reshape(-1, kin)
        xt = torch.cat([x, torch.ones_like(x[:, :1])], 1)
        dy = grab.y[w].grad.reshape(-1, nout)
        out.append((xt.T @ xt / B, dy.T @ dy / B))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny_b6", "p19_b37", "p12_b3"])
@pytest.mark.parametrize("fisher", ["true", "empirical"])
def test_factors_match_the_float64_oracle(name, fisher):
    cfg, d, model = _setup(name)
    cov = IF.kfac_covariances(model, _q(d), fisher=fisher, seed=3)
    if fisher == "true":
        with torch.no_grad():
            logits, _, _ = model.forward(d["src"], d["static"], d["times"], d["lengths"])
        y = torch.from_numpy(fisher_labels(logits.cpu().numpy(), 3)).cuda()
    else:
        y = d["y"]
    ref = _oracle_factors(cfg, d, y, model)
    errs = [(_rel(A, Ar), _rel(S, Sr)) for (A, S), (Ar, Sr) in zip(cov, ref)]
    assert max(max(e) for e in errs) <= FACTOR_TOL, (name, errs)
    again = IF.kfac_covariances(model, _q(d), fisher=fisher, seed=3)
    assert all(torch.equal(a, b) and torch.equal(s, t) for (a, s), (b, t) in zip(cov, again))


def _rows(model, d, factors):
    ldg = IF._bucket_length(IF.grad_layout(model))
    bases = factors.bases_flat.cuda()
    with torch.no_grad():
        return IF._backward(model, *[d[k] for k in ("src", "static", "times", "lengths", "y")], "rows", ldg=ldg, bases=bases)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny_b6", "p19_b37", "p12_b3", "pam_b2"])
def test_rotated_rows_rotate_back_to_the_gradients(name):
    cfg, d, model = _setup(name)
    f = IF.ekfac_factors(model, _q(d), fisher="empirical")
    G = IF.per_sample_grads(model, *[d[k] for k in ("src", "static", "times", "lengths", "y")]).double().cpu().numpy()
    Gr = _rows(model, d, f).double().cpu().numpy()
    # back-rotation Q_S G~ Q_A^T is the rotation by the transposed bases
    back = IF.EKFACFactors(**{**f.__dict__, "bases": tuple((QA.T, QS.T) for QA, QS in f.bases)})
    Gb = IF.ekfac_rotate(Gr, back)
    err = (np.linalg.norm(Gb - G, axis=1) / np.linalg.norm(G, axis=1)).max()
    assert err <= 1e-5, err
    # identity bases give the plain rows
    Gi = _rows(model, d, _identity_factors(model)).double().cpu().numpy()
    err = (np.linalg.norm(Gi - G, axis=1) / np.linalg.norm(G, axis=1)).max()
    assert err <= 1e-6, err


@pytest.mark.gpu
@pytest.mark.parametrize("fisher", ["empirical", "true"])
def test_eigenvalues_are_the_mean_squared_rotated_rows(fisher):
    cfg, d, model = _setup("p19_b37", B=200, seed=8)
    keys = [k for k, _, _ in IF.grad_layout(model)]
    blocks = IF.kfac_blocks(model)
    for fields in (None, [blocks[1][0], blocks[1][1], keys[0]]):
        f = IF.ekfac_factors(model, _q(d), fisher=fisher, seed=5, fields=fields)
        ldg = IF._bucket_length(IF.grad_layout(model))
        R = IF._row_batch(L.load(), model._plan, ldg)
        _, fetch = IF._source(_q(d), "d")
        G = IF._ekfac_rows_aligned(model, fetch, 0, 200, R, ldg, f.bases_flat.cuda(),
                                   5 if fisher == "true" else None).double()
        ref = (G * G).mean(0)
        off, ln = IF.plan_segments(IF.grad_layout(model), fields)
        cols = torch.from_numpy(np.concatenate([np.arange(o, o + n) for o, n in zip(off, ln)])).cuda()
        lam = f.eigenvalues
        assert ((lam[cols] - ref[cols]).abs() <= 1e-6 * ref[cols].abs() + 1e-300).all()
        mask = torch.ones(ldg, dtype=torch.bool, device="cuda")
        mask[cols] = False
        assert not lam[mask].any()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny_b6", "p19_b37"])
def test_scores_match_the_float64_restatement(name):
    cfg, d, model = _setup(name, B=40, seed=9)
    _, dq, _ = _setup(name, B=7, seed=10)
    params0 = [p.detach().clone() for p in model.used_parameters()]
    rng0 = model._plan.rng_state.clone()
    f = IF.ekfac_factors(model, _q(d), fisher="true", seed=1)
    S = IF.ekfac_influence(model, _q(dq, y=False), _q(d), f)
    assert S.dtype == torch.float64 and S.shape == (7, 40)
    assert all(torch.equal(p, q) for p, q in zip(model.used_parameters(), params0))
    assert torch.equal(model._plan.rng_state, rng0) and not model.training
    with torch.no_grad():
        logits, _, _ = model.forward(dq["src"], dq["static"], dq["times"], dq["lengths"])
    args = lambda dd, y: (dd["src"], dd["static"], dd["times"], dd["lengths"], y)
    Gq = IF.per_sample_grads(model, *args(dq, logits.argmax(1))).double().cpu().numpy()
    Gt = IF.per_sample_grads(model, *args(d, d["y"])).double().cpu().numpy()
    ref = IF.ekfac_from_grads(Gq, Gt, f)
    assert _rel(S.cpu(), torch.from_numpy(ref)) <= 1e-5
    # lambda -> infinity: lambda * score -> tracin
    lam = 1e6 * f.eigenvalues.max().item()
    tr = IF.tracin(model, _q(dq, y=False), _q(d))
    got = lam * IF.ekfac_influence(model, _q(dq, y=False), _q(d), f, damping=lam)
    assert _rel(got, tr) <= 1e-3, _rel(got, tr)
    # self-influence is the diagonal of influence(q, q), bitwise
    Sd = IF.ekfac_influence(model, _q(d), _q(d), f)
    assert torch.equal(Sd.diagonal(), IF.ekfac_self_influence(model, _q(d), f))


@pytest.mark.gpu
def test_scores_match_the_dense_preconditioner_on_one_block():
    cfg, d, model = _setup("tiny_b6", B=30, seed=12)
    _, dq, _ = _setup("tiny_b6", B=4, seed=13)
    w, b, nout, kin = IF.kfac_blocks(model)[1]
    f = IF.ekfac_factors(model, _q(d), fisher="empirical", fields=[w, b])
    S = IF.ekfac_influence(model, _q(dq), _q(d), f).cpu().numpy()
    QA, QS = f.bases[1]
    off = {k: o for k, o, _ in IF.grad_layout(model)}
    lay = {k: o for k, o, _ in IF.grad_layout(model)}
    args = lambda dd: (dd["src"], dd["static"], dd["times"], dd["lengths"], dd["y"])
    lamv = f.eigenvalues.cpu().numpy()
    wts = IF.ekfac_weights(f)

    def block(G):          # [n, Nout, Kin + 1] = [W | b] flattened row-major
        G = G.double().cpu().numpy()
        M = np.concatenate([G[:, off[w]:off[w] + nout * kin].reshape(-1, nout, kin), G[:, off[b]:off[b] + nout, None]], 2)
        return M.reshape(len(G), -1)

    def diag(v):           # the block's weights in the same [Nout, Kin + 1] order
        return np.concatenate([v[lay[w]:lay[w] + nout * kin].reshape(nout, kin), v[lay[b]:lay[b] + nout, None]], 1).ravel()
    Q = np.kron(QS, QA)                                  # vec(Q_S^T M Q_A) = (Q_S (x) Q_A)^T vec(M), row-major
    P = Q @ np.diag(diag(wts)) @ Q.T
    gq, gt = block(IF.per_sample_grads(model, *args(dq))), block(IF.per_sample_grads(model, *args(d)))
    ref = gq @ P @ gt.T
    assert np.abs(S - ref).max() <= 1e-5 * np.abs(ref).max()
    assert (diag(lamv) >= 0).all()


@pytest.mark.gpu
def test_bitwise_across_chunking_sources_and_runs():
    from raindrop_b200.data import DeviceDataset
    cfg, d, model = _setup("p19_b37", B=300, seed=5)
    _, dq, _ = _setup("p19_b37", B=150, seed=6)
    f = IF.ekfac_factors(model, _q(d), seed=2)
    ds = DeviceDataset(d["src"], d["static"], d["times"], d["y"])
    g = IF.ekfac_factors(model, ds, seed=2, internal_batch_size=1)
    assert torch.equal(f.eigenvalues, g.eigenvalues) and torch.equal(f.bases_flat, g.bases_flat)
    ref = IF.ekfac_influence(model, _q(dq), _q(d), f)
    assert torch.equal(ref, IF.ekfac_influence(model, _q(dq), _q(d), f))
    for ibs in (1, 129, 300):
        assert torch.equal(ref, IF.ekfac_influence(model, _q(dq), _q(d), f, internal_batch_size=ibs)), ibs
    assert torch.equal(ref, IF.ekfac_influence(model, _q(dq), ds, f, internal_batch_size=100))
    si = IF.ekfac_self_influence(model, _q(d), f)
    assert torch.equal(si, IF.ekfac_self_influence(model, ds, f, internal_batch_size=7))


@pytest.mark.gpu
def test_full_size_p19_completes():
    cfg = model_config("P19", dropout=0.2)
    model = build_dropin(cfg, 21)
    model.eval()
    dq = to_dev(make_batch(cfg, 512, seed=41))
    dt = to_dev(make_batch(cfg, 4096, seed=42))
    f = IF.ekfac_factors(model, _q(dt))
    S = IF.ekfac_influence(model, _q(dq, y=False), _q(dt), f)
    assert S.shape == (512, 4096) and torch.isfinite(S).all()
    si = IF.ekfac_self_influence(model, _q(dt), f)
    assert (si > 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("name,nq,nt", [("PAM", 8, 32), ("LARGE", 4, 16)])
def test_large_shapes_complete_within_the_scratch_plan(name, nq, nt):
    cfg = model_config(name, dropout=0.2)
    model = build_dropin(cfg, 21)
    model.eval()
    dq = to_dev(make_batch(cfg, nq, seed=51))
    dt = to_dev(make_batch(cfg, nt, seed=52))
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    f = IF.ekfac_factors(model, _q(dt))
    S = IF.ekfac_influence(model, _q(dq, y=False), _q(dt), f)
    assert S.shape == (nq, nt) and torch.isfinite(S).all()
    assert torch.cuda.max_memory_allocated() - base <= 3 * IF.DEFAULT_SCRATCH_BYTES
