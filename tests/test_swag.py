"""SWA / SWAG / MultiSWAG (raindrop_b200.swag).  On the host: the float64 restatements against the direct definitions,
pinned site-102 normals, the covariance of restated samples, the scratch query, argument checks and save / load.  On the
GPU: collection bitwise against swag_from_snapshots over real training trajectories (TrainStep eager and replayed,
FlatAdam, a plain module), the sampler against swag_sample_from_state, the predictive against module forwards on the
exported weights, chunking, the key algebra, CUDA-graph replay, MultiSWAG and the deep ensemble, and side effects.

Every GPU test pins plan.obprop_mode, so the forward's arithmetic does not follow the chunk's row count."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from helpers import build_dropin, to_dev
from raindrop_b200 import lib as L
from raindrop_b200 import swag as SW
from raindrop_b200.influence import _bucket_length, grad_layout
from raindrop_b200.synth import make_batch, model_config
from raindrop_b200.uncertainty import mc_dropout_from_logits

EXACT, FAST = 2, 1
FIELDS = ("mean_probs", "variance", "predictive_entropy", "expected_entropy", "mutual_information", "samples")
# the first eight site-102 normals at seed 1, step 2 (elements 0 .. 7), as float32 hex
KAT_NORMALS = ["-0x1.fdc6500000000p-1", "-0x1.1316800000000p-5", "0x1.9426f00000000p+0", "0x1.6196380000000p+0",
               "0x1.0913480000000p+0", "0x1.73eedc0000000p-4", "0x1.3f87e60000000p+0", "0x1.b5294c0000000p-3"]
# rd_swag_predictive_scratch_bytes(dims(B, eval), rows_per_chunk)
SCRATCH = {('TINY', 5, 1): 294912, ('TINY', 5, 7): 514560, ('TINY', 5, 64): 2585088, ('TINY', 128, 1): 300544,
           ('TINY', 128, 7): 520192, ('TINY', 128, 64): 2590720, ('P19', 5, 1): 6427136, ('P19', 5, 7): 11444224,
           ('P19', 5, 64): 59092736, ('P19', 128, 1): 6432768, ('P19', 128, 7): 11449856, ('P19', 128, 64): 59098368,
           ('PAM', 5, 1): 149745920, ('PAM', 5, 7): 211368192, ('PAM', 5, 64): 727653120, ('PAM', 128, 1): 149766400,
           ('PAM', 128, 7): 211388672, ('PAM', 128, 64): 727673600}


# ---- host -------------------------------------------------------------------------------------------------------------
def _direct_moments(th, rank):
    """The moments straight from their definitions: arithmetic means over all snapshots, deviations of the last
    min(c, rank) snapshots from the running mean at their time."""
    th = np.asarray(th, dtype=np.float64)
    c, n = th.shape
    dev = np.zeros((rank, n))
    for i in range(c):
        if rank:
            dev[i % rank] = th[i] - th[:i + 1].mean(axis=0)
    return th.mean(axis=0), (th ** 2).mean(axis=0), dev


@pytest.mark.parametrize("c,rank", [(1, 4), (3, 4), (9, 4), (6, 0), (5, 1)])
def test_moments_against_direct_definitions(c, rank):
    rng = np.random.default_rng(c * 10 + rank)
    base = rng.normal(scale=0.3, size=64).astype(np.float32)
    th = (base + np.cumsum(rng.normal(scale=1e-3, size=(c, 64)), axis=0)).astype(np.float32)
    mean, sq, dev, k = SW.swag_from_snapshots(th, rank)
    dm, ds, dd = _direct_moments(th, rank)
    assert k == min(c, rank) and dev.dtype == np.float32 and dev.shape == (rank, 64)
    np.testing.assert_allclose(mean, dm, rtol=1e-14, atol=1e-16)
    np.testing.assert_allclose(sq, ds, rtol=1e-14, atol=1e-16)
    np.testing.assert_allclose(dev, dd, rtol=1e-6, atol=1e-12)
    if c == 1:         # one snapshot: the mean is the snapshot, its deviation 0, the low-rank term off (k < 2)
        assert np.array_equal(mean, th[0].astype(np.float64)) and np.all(dev == 0) and k <= 1


def test_sample_formula_against_direct_evaluation():
    rng = np.random.default_rng(5)
    n, rank = 40, 6
    th = (rng.normal(size=n) + rng.normal(scale=1e-2, size=(9, n))).astype(np.float32)
    mean, sq, dev, k = SW.swag_from_snapshots(th, rank)
    for scale, kk in ((0.5, k), (1.0, k), (0.0, k), (0.5, 1), (0.5, 0)):
        got = SW.swag_sample_from_state(mean, sq, dev, kk, scale, seed=3, step=7, replicate=2)
        z = SW.swag_normals(3, 9, np.arange(n + kk)).astype(np.float64)
        want = mean + math.sqrt(scale) * np.sqrt(np.maximum(sq - mean ** 2, 0)) * z[:n]
        if kk >= 2:
            want = want + math.sqrt(scale) * (dev[:kk].astype(np.float64).T @ z[n:]) / math.sqrt(kk - 1)
        np.testing.assert_allclose(got, want.astype(np.float32), rtol=2e-7, atol=1e-9)
    assert np.array_equal(SW.swag_sample_from_state(mean, sq, dev, k, 0.0, 1, 2), mean.astype(np.float32))


def test_pinned_site_102_normals():
    z = SW.swag_normals(1, 2, np.arange(8))
    assert [float(v).hex() for v in z] == [float.fromhex(h).hex() for h in KAT_NORMALS]
    # the key algebra: (seed, step) at replicate r is (seed, step + r) at replicate 0; far indices are drawn directly
    assert np.array_equal(SW.swag_normals(1, 2, [10 ** 9 + 3]), SW.swag_normals(1, 2, np.arange(10 ** 9, 10 ** 9 + 4))[3:])
    assert not np.array_equal(SW.swag_normals(1, 3, np.arange(8)), z)


def test_restated_sample_covariance():
    """20,000 restated draws on a 12-element bucket against scale (diag var + D D^T / (k - 1)), within 6 sigma of the
    sampling error of each moment."""
    rng = np.random.default_rng(2)
    n, rank, S, scale = 12, 4, 20000, 0.5
    th = (rng.normal(size=n) + rng.normal(scale=0.1, size=(7, n))).astype(np.float32)
    mean, sq, dev, k = SW.swag_from_snapshots(th, rank)
    X = np.stack([SW.swag_sample_from_state(mean, sq, dev, k, scale, seed=0, step=s) for s in range(S)]).astype(np.float64)
    D = dev[:k].astype(np.float64).T
    cov = scale * (np.diag(np.maximum(sq - mean ** 2, 0)) + D @ D.T / (k - 1))
    sd = np.sqrt(np.diag(cov))
    assert np.all(np.abs(X.mean(axis=0) - mean) <= 6 * sd / math.sqrt(S))
    emp = np.cov(X, rowvar=False)
    # var of the sample covariance of a Gaussian: (cov_ij^2 + cov_ii cov_jj) / S
    tol = 6 * np.sqrt((cov ** 2 + np.outer(np.diag(cov), np.diag(cov))) / S)
    assert np.all(np.abs(emp - cov) <= tol)


def test_scratch_query_pinned():
    lib = L.load()
    for (name, B, rpc), want in SCRATCH.items():
        model = build_dropin(model_config(name, dropout=0.2), 3, device="cpu")
        d = model._plan.dims(B, False)
        assert lib.rd_swag_predictive_scratch_bytes(C.byref(d), rpc) == want, (name, B, rpc)
        assert lib.rd_swag_predictive_scratch_bytes(C.byref(d), 0) == 0


def _cpu_model(name="TINY", wseed=3):
    cfg = model_config(name, dropout=0.2)
    return build_dropin(cfg, wseed, device="cpu").eval(), make_batch(cfg, 3, seed=1)


def _fake_posterior(model, rank=3, c=4, seed=0):
    p = SW.SWAG(model, rank=rank)
    rng = np.random.default_rng(seed)
    th = rng.normal(size=(c, p.n)).astype(np.float32)
    mean, sq, dev, _ = SW.swag_from_snapshots(th, rank)
    p.mean.copy_(torch.from_numpy(mean))
    p.sq_mean.copy_(torch.from_numpy(sq))
    p.dev.copy_(torch.from_numpy(dev))
    p.n_collected = c
    return p


def test_argument_validation():
    model, b = _cpu_model()
    args = (b["src"], b["static"], b["times"], b["lengths"])
    for r in (-1, 1.5, L.SWAG_MAX_RANK + 1, True):
        with pytest.raises(ValueError):
            SW.SWAG(model, rank=r)
    post = SW.SWAG(model, rank=2)
    assert post.n == _bucket_length(grad_layout(model)) and post.k == 0 and post.dev.shape == (2, post.n)
    with pytest.raises(ValueError, match="empty"):
        SW.swag_predictive(model, post, *args)
    with pytest.raises(ValueError, match="empty"):
        post.load_mean(model)
    with pytest.raises(ValueError, match="empty"):
        post.sample_weights()
    full = _fake_posterior(model)
    for kw in (dict(n_samples=0), dict(n_samples=2.5), dict(scale=-0.1), dict(scale=float("inf")), dict(seed=-1),
               dict(seed=1 << 64), dict(step=-1), dict(step=(1 << 64) - 2, n_samples=3), dict(internal_batch_size=0)):
        with pytest.raises(ValueError):
            SW.swag_predictive(model, full, *args, **kw)
    with pytest.raises(ValueError):
        SW.swag_predictive(model, [], *args)
    with pytest.raises(TypeError):
        SW.swag_predictive(model, [full, "x"], *args)
    other, _ = _cpu_model("TINY8")
    with pytest.raises(ValueError):
        SW.swag_predictive(other, full, *args)
    with pytest.raises(ValueError, match="layout"):
        SW.swag_predictive(model, [full, _fake_posterior(other)], *args)
    with pytest.raises(ValueError, match="layout"):
        full.load_mean(other)
    with pytest.raises(TypeError):
        full.collect(torch.zeros(full.n))
    with pytest.raises(TypeError):
        SW.swag_predictive(torch.nn.Linear(2, 2), full, *args)
    for bad in (dict(scale=-1.0), dict(seed=-1), dict(step=-1)):
        with pytest.raises(ValueError):
            full.sample_weights(**bad)
    with pytest.raises(ValueError):
        SW.swag_sample_from_state(full.mean, full.sq_mean, full.dev, 2, -0.5, 0, 0)


def test_no_cuda_raises(monkeypatch):
    model, b = _cpu_model()
    post = _fake_posterior(model)
    with pytest.raises(L.RaindropB200Error):
        post.collect(model)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(L.RaindropB200Error):
        SW.swag_predictive(model, post, b["src"], b["static"], b["times"], b["lengths"], n_samples=2)


def test_save_load_round_trip_and_refusal(tmp_path):
    model, _ = _cpu_model()
    post = _fake_posterior(model, rank=3, c=5)
    path = str(tmp_path / "swag.pt")
    post.save(path)
    got = SW.SWAG.load(path, model)
    assert got.rank == 3 and got.n_collected == 5 and got.k == 3
    for f in ("mean", "sq_mean", "dev"):
        assert torch.equal(getattr(got, f), getattr(post, f)), f
    other, _ = _cpu_model("TINY8")
    with pytest.raises(ValueError, match="layout"):
        SW.SWAG.load(path, other)
    # load_mean writes fp32(mean) into the trained tensors
    got.load_mean(model)
    for (_, off, shape), p in zip(got.layout, model.used_parameters()):
        assert torch.equal(p.detach(), got.mean[off:off + math.prod(shape)].view(shape).float())


# ---- GPU --------------------------------------------------------------------------------------------------------------
# name -> (config, B)
CASES = {"tiny": ("TINY", 6), "tiny8": ("TINY8", 9), "p19": ("P19", 13), "p12": ("P12", 3), "pam": ("PAM", 2)}


def _setup(name, wseed=21, mode=EXACT, B=None):
    cfg_name, B0 = CASES[name]
    cfg = model_config(cfg_name, dropout=0.2)
    batch = to_dev(make_batch(cfg, B or B0, seed=200 + (B or B0)))
    model = build_dropin(cfg, wseed)
    model._plan.obprop_mode = mode
    return cfg, batch, model


def _args(d):
    return d["src"], d["static"], d["times"], d["lengths"]


def _trajectory(model, d, steps, rank, collect_every=1, use_graph=False, lr=1e-3):
    """A TrainStep run collecting every `collect_every` steps: (posterior, snapshots [c, n] of flat_p, TrainStep)."""
    from raindrop_b200.train import TrainStep
    ts = TrainStep(model, d["src"].shape[1], lr=lr, use_graph=use_graph)
    ts.load_batch(d)
    post = SW.SWAG(model, rank=rank)
    snaps = []
    for i in range(steps):
        ts.step()
        if (i + 1) % collect_every == 0:
            post.collect(ts)
            snaps.append(ts.flat_p.detach().cpu().numpy().copy())
    torch.cuda.synchronize()
    return post, np.stack(snaps), ts


def _check_against_snapshots(post, snaps):
    mean, sq, dev, k = SW.swag_from_snapshots(snaps, post.rank)
    assert post.n_collected == len(snaps) and post.k == k
    assert np.array_equal(post.mean.cpu().numpy(), mean)
    assert np.array_equal(post.sq_mean.cpu().numpy(), sq)
    assert np.array_equal(post.dev.cpu().numpy(), dev)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_collect_from_train_step_bitwise(name):
    """Six collects into rank 4 (a wrap past the ring) over an eager TrainStep run; the trajectory is bitwise the one
    of the same run without collects."""
    cfg, d, model = _setup(name)
    post, snaps, ts = _trajectory(model, d, 6, rank=4)
    _check_against_snapshots(post, snaps)
    assert not np.array_equal(snaps[0], snaps[-1])
    _, _, plain = _setup(name)
    from raindrop_b200.train import TrainStep
    ts2 = TrainStep(plain, d["src"].shape[1], lr=1e-3, use_graph=False)
    ts2.load_batch(d)
    for _ in range(6):
        ts2.step()
    assert torch.equal(ts2.flat_p, ts.flat_p)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny8", "p19"])
def test_collect_from_graph_replay_and_diagonal(name):
    cfg, d, model = _setup(name)
    post, snaps, ts = _trajectory(model, d, 7, rank=3, collect_every=2, use_graph=True)
    assert ts.graph is not None
    _check_against_snapshots(post, snaps)
    # rank 0: the moments alone
    _, _, m0 = _setup(name)
    diag, snaps0, _ = _trajectory(m0, d, 3, rank=0, use_graph=True)
    _check_against_snapshots(diag, snaps0)
    assert diag.dev.numel() == 0


def _bucket_of(model, layout):
    out = torch.zeros(_bucket_length(layout), dtype=torch.float32)
    for (_, off, shape), p in zip(layout, model.used_parameters()):
        out[off:off + math.prod(shape)] = p.detach().reshape(-1).cpu()
    return out.numpy()


@pytest.mark.gpu
def test_collect_from_flat_adam_and_module():
    import torch.nn.functional as F
    from raindrop_b200.optim import FlatAdam
    cfg, d, model = _setup("tiny")
    model.train()
    opt = FlatAdam(model, lr=1e-3)
    post = SW.SWAG(model, rank=2)
    via_model = SW.SWAG(model, rank=2)
    snaps = []
    for _ in range(3):
        logits, _, _ = model(*_args(d))
        F.cross_entropy(logits, d["y"]).backward()
        opt.step()
        post.collect(opt)
        via_model.collect(model)
        snaps.append(opt.flat_p.detach().cpu().numpy().copy())
    torch.cuda.synchronize()
    _check_against_snapshots(post, np.stack(snaps))
    _check_against_snapshots(via_model, np.stack(snaps))
    # a plain module (no bucket): its parameters packed into the layout
    _, _, plain = _setup("p19")
    p2 = SW.SWAG(plain, rank=2)
    p2.collect(plain)
    with torch.no_grad():
        for p in plain.used_parameters():
            p.mul_(0.5)
    p2.collect(plain)
    _check_against_snapshots(p2, np.stack([_bucket_of(plain, p2.layout) * 2, _bucket_of(plain, p2.layout)]))


def _ulp_close(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ulp = np.maximum(np.spacing(np.abs(a)), np.spacing(np.abs(b)))
    return np.abs(a.astype(np.float64) - b.astype(np.float64)) <= ulp


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_sample_weights_against_restatement(name):
    cfg, d, model = _setup(name)
    post, snaps, _ = _trajectory(model, d, 5, rank=3)
    mean, sq, dev, k = post.mean.cpu().numpy(), post.sq_mean.cpu().numpy(), post.dev.cpu().numpy(), post.k
    for seed, step, scale in ((0, 0, 0.5), (0x2B7E151628AED2A6, (1 << 32) - 1, 2.0)):
        got = post.sample_weights(seed=seed, step=step, scale=scale).cpu().numpy()
        want = SW.swag_sample_from_state(mean, sq, dev, k, scale, seed, step)
        close = _ulp_close(got, want)
        assert close.all(), (name, int((~close).sum()))
        assert not np.array_equal(got, mean.astype(np.float32))
    # padding lanes stay 0, and scale 0 is fp32(mean)
    pad = np.ones(post.n, dtype=bool)
    for _, off, shape in post.layout:
        pad[off:off + math.prod(shape)] = False
    assert np.all(got[pad] == 0)
    assert np.array_equal(post.sample_weights(scale=0.0).cpu().numpy(), mean.astype(np.float32))


def _forward_with(model, theta, d, layout):
    """The module's eval forward with the bucket theta loaded into the trained tensors (restored afterwards)."""
    params = model.used_parameters()
    saved = [p.detach().clone() for p in params]
    was = model.training
    model.eval()
    with torch.no_grad():
        for (_, off, shape), p in zip(layout, params):
            p.copy_(theta[off:off + math.prod(shape)].view(shape))
        out = model(*_args(d))[0].clone()
        for p, s in zip(params, saved):
            p.copy_(s)
    model.train(was)
    return out


def _check_stats(res, logits):
    """The device statistics against mc_dropout_from_logits of the same logits: the same fp64 arithmetic rounded to fp32
    at the end, so within 1e-10 plus the fp32 rounding of each output."""
    ref = mc_dropout_from_logits(logits)
    for f in FIELDS[:5]:
        got, want = getattr(res, f).double().cpu().numpy(), getattr(ref, f)
        assert np.all(np.abs(got - want) <= 1e-10 + 2.0 ** -24 * np.abs(want) + 1e-12), f


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_predictive_equals_module_forwards(name):
    cfg, d, model = _setup(name)
    post, _, _ = _trajectory(model, d, 4, rank=3, lr=3e-3)
    model.eval()
    S, seed, step = 3, 7, 11
    res = SW.swag_predictive(model, post, *_args(d), n_samples=S, seed=seed, step=step, return_samples=True)
    for r in range(S):
        theta = post.sample_weights(seed=seed, step=step + r)
        assert torch.equal(res.samples[r], _forward_with(model, theta, d, post.layout)), (name, r)
    assert not torch.equal(res.samples[0], res.samples[1])
    _check_stats(res, res.samples)
    # scale 0: every replicate is the SWA model
    zero = SW.swag_predictive(model, post, *_args(d), n_samples=2, scale=0.0, return_samples=True)
    swa = build_dropin(cfg, 21)
    swa._plan.obprop_mode = EXACT
    post.load_mean(swa)
    with torch.no_grad():
        want = swa.eval()(*_args(d))[0]
    assert torch.equal(zero.samples[0], want) and torch.equal(zero.samples[1], want)
    # identical replicates: the reduction's variance and MI are 0 up to its fp64 rounding (as mc_dropout at p = 0)
    assert zero.variance.abs().max().item() <= 1e-14 and zero.mutual_information.abs().max().item() <= 1e-12


@pytest.mark.gpu
def test_multiswag_and_deep_ensemble():
    cfg, d, m_a = _setup("p19", wseed=21)
    _, _, m_b = _setup("p19", wseed=22)
    a, _, _ = _trajectory(m_a, d, 4, rank=3, lr=3e-3)
    b, _, _ = _trajectory(m_b, d, 3, rank=3, lr=3e-3)
    model = m_a.eval()
    S = 3
    multi = SW.swag_predictive(model, [a, b], *_args(d), n_samples=S, seed=5, step=9, return_samples=True)
    ra = SW.swag_predictive(model, a, *_args(d), n_samples=S, seed=5, step=9, return_samples=True)
    rb = SW.swag_predictive(model, b, *_args(d), n_samples=S, seed=5, step=9 + S, return_samples=True)
    assert torch.equal(multi.samples, torch.cat([ra.samples, rb.samples]))
    _check_stats(multi, multi.samples)
    # the deep ensemble: scale 0, one sample per member = the average of the SWA models' softmax
    ens = SW.swag_predictive(model, [a, b], *_args(d), n_samples=1, scale=0.0, return_samples=True)
    probs = []
    for p in (a, b):
        swa = build_dropin(cfg, 21)
        swa._plan.obprop_mode = EXACT
        p.load_mean(swa)
        with torch.no_grad():
            lg = swa.eval()(*_args(d))[0]
        probs.append(torch.softmax(lg.double(), dim=1))
        assert torch.equal(ens.samples[len(probs) - 1], lg)
    want = (probs[0] + probs[1]) / 2
    assert (ens.mean_probs.double() - want).abs().max().item() <= 1e-7


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [EXACT, FAST])
def test_chunking_key_algebra_and_graph(mode):
    cfg, d, model = _setup("tiny8", mode=mode)
    post, _, _ = _trajectory(model, d, 4, rank=3, lr=3e-3)
    model.eval()
    B = d["src"].shape[1]
    kw = dict(n_samples=5, seed=3, step=(1 << 32) - 2, return_samples=True)
    outs = [SW.swag_predictive(model, post, *_args(d), internal_batch_size=ibs, **kw) for ibs in (None, 1, 4, B)]
    for o in outs[1:]:
        for f in FIELDS:
            assert torch.equal(getattr(o, f), getattr(outs[0], f)), (mode, f)
    head = SW.swag_predictive(model, post, *_args(d), n_samples=2, seed=3, step=(1 << 32) - 2, return_samples=True)
    tail = SW.swag_predictive(model, post, *_args(d), n_samples=3, seed=3, step=(1 << 32), return_samples=True)
    assert torch.equal(torch.cat([head.samples, tail.samples]), outs[0].samples)
    # CUDA-graph replay equals the eager call; a later eager call with another key does not disturb the graph
    gkw = dict(kw, internal_batch_size=4)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eager = SW.swag_predictive(model, post, *_args(d), **gkw)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = SW.swag_predictive(model, post, *_args(d), **gkw)
    SW.swag_predictive(model, post, *_args(d), n_samples=2, step=5, internal_batch_size=B)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        for f in FIELDS:
            assert torch.equal(getattr(out, f), getattr(eager, f)), f


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["train_step", "flat_adam"])
def test_no_side_effects(kind):
    import torch.nn.functional as F
    cfg, d, model = _setup("p19")
    post = SW.SWAG(model, rank=3)
    if kind == "train_step":
        from raindrop_b200.train import TrainStep
        bound = TrainStep(model, d["src"].shape[1], lr=1e-3, use_graph=False)
        bound.load_batch(d)
        for _ in range(3):
            bound.step()
            post.collect(bound)
        snap = {"flat_p": bound.flat_p, "flat_g": bound.flat_g, "exp_avg": bound.exp_avg, "exp_avg_sq": bound.exp_avg_sq,
                "step": bound.step_count}
    else:
        from raindrop_b200.optim import FlatAdam
        model.train()
        bound = FlatAdam(model, lr=1e-3)
        for _ in range(3):
            logits, _, _ = model(*_args(d))
            F.cross_entropy(logits, d["y"]).backward()
            bound.step()
            post.collect(bound)
        snap = {"flat_p": bound.flat_p.detach(), "flat_g": bound.flat_g, "exp_avg": bound.exp_avg,
                "exp_avg_sq": bound.exp_avg_sq, "step": bound.step_count}
    model.train()
    snap["rng"] = model._plan.rng_state
    snap.update({"param." + k: p.detach() for k, p in model.named_parameters()})
    grads = {k: (None if p.grad is None else p.grad.clone()) for k, p in model.named_parameters()}
    inputs = {k: v.clone() for k, v in d.items() if v is not None}
    before = {k: v.clone() for k, v in snap.items()}
    res = SW.swag_predictive(model, post, *_args(d), n_samples=3, return_samples=True)
    post.sample_weights(seed=1)
    torch.cuda.synchronize()
    assert model.training
    for k, v in snap.items():
        assert torch.equal(v, before[k]), k
    for k, p in model.named_parameters():
        assert (p.grad is None) == (grads[k] is None) and (p.grad is None or torch.equal(p.grad, grads[k])), k
    assert all(torch.equal(d[k], v) for k, v in inputs.items())
    # train() mode still runs eval arithmetic: equal to the call on the model in eval()
    again = SW.swag_predictive(model.eval(), post, *_args(d), n_samples=3, return_samples=True)
    assert torch.equal(res.samples, again.samples)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name,B,ibs", [("P19", 3880, None), ("LARGE", 64, 16)])
def test_full_size(cfg_name, B, ibs):
    cfg = model_config(cfg_name, dropout=0.2)
    model = build_dropin(cfg, 21).eval()
    model._plan.obprop_mode = EXACT
    d = to_dev(make_batch(cfg, B, seed=3))
    post = SW.SWAG(model, rank=4)
    post.collect(model)
    with torch.no_grad():
        for p in model.used_parameters():
            p.mul_(1.01)
    post.collect(model)
    res = SW.swag_predictive(model, post, *_args(d), n_samples=2, internal_batch_size=ibs, return_samples=True)
    torch.cuda.synchronize()
    assert torch.isfinite(res.samples).all() and torch.isfinite(res.mean_probs).all()
    _check_stats(res, res.samples)
