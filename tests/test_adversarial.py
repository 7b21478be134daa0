"""PGD adversarial examples and adversarial training of Raindrop_v2 (raindrop_b200.adversarial, rd_raindrop_v2_pgd).

CPU: the exported symbols, the host argument checks and a numpy restatement of the random-start stream.  GPU: the
threat model's invariants, bitwise identities (eps = 0, chunking, repeat calls, the module forward on the returned
input), the random start against the restatement, L2 PGD and FGSM against the float64 oracle, and AdversarialTrainStep
against TrainStep.  Every GPU test pins plan.obprop_mode: the auto mode picks the ob-prop arithmetic from the row count."""
import os
import subprocess

import numpy as np
import pytest
import torch

from helpers import build_dropin, to_dev
from raindrop_b200 import adversarial as ADV
from raindrop_b200.synth import make_batch, model_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXACT, FAST = 2, 1
SITE_PGD_START = 98
SEED = 0x2B7E151628AED2A6
# name -> (config, B, make_batch options)
CASES = {
    "tiny_b6": ("TINY", 6, {}),
    "tiny8_b5": ("TINY8", 5, {}),                       # no statics
    "p19_b9": ("P19", 9, {"first_time_zero": True}),    # padded rows
    "p12_b3": ("P12", 3, {}),                           # T = 215
    "pam_b2": ("PAM", 2, {}),                           # T = 600, C = 2400
}


# ---- numpy restatement of the random start ---------------------------------------------------------------------------
def _words(seed, step, idx):
    from oracle.dropout_masks import dropout_words_at
    return dropout_words_at(seed, step, SITE_PGD_START, idx)


def _normals(seed, step, idx):
    """Box-Muller on the Philox block's word pairs, as rd_dp_add_noise: element i takes (x, y) for i & 3 in {0, 1},
    (z, w) for {2, 3}, and the cos branch for even i."""
    from oracle.dropout_masks import philox4x32_10
    seed, step = int(seed), int(step)
    idx = np.asarray(idx, dtype=np.uint64)
    blk = idx >> np.uint64(2)
    ctr = np.stack([blk & np.uint64(0xFFFFFFFF), blk >> np.uint64(32), np.full_like(blk, SITE_PGD_START),
                    np.full_like(blk, step & 0xFFFFFFFF)], -1)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) ^ (step >> 32)], dtype=np.uint64)
    w = philox4x32_10(ctr, key).astype(np.uint64)
    hi = (idx & np.uint64(2)) != 0
    a = np.where(hi, w[..., 2], w[..., 0])
    b = np.where(hi, w[..., 3], w[..., 1])
    u1 = ((a >> np.uint64(8)).astype(np.float64) + 1.0) / 16777216.0
    u2 = (b >> np.uint64(8)).astype(np.float64) / 16777216.0
    r, t = np.sqrt(-2.0 * np.log(u1)), 2.0 * np.pi * u2
    return np.where((idx & np.uint64(1)) != 0, r * np.sin(t), r * np.cos(t)).astype(np.float32)


def random_start(src, static, norm, eps, seed, step, sensors=None, perturb_static=False):
    """delta_0 of every sample: (delta_src [T, B, N] fp32, delta_static [B, ds] fp32 or None), drawn where the kernels
    draw it (element e of sample b at index b*(T*N + ds + 1) + e, the l2 radius at b*(T*N + ds + 1) + T*N + ds)."""
    src = np.asarray(src, dtype=np.float32)
    T, B, N2 = src.shape
    N = N2 // 2
    ds = 0 if static is None else np.asarray(static).shape[1]
    E = T * N + ds
    pert = src[:, :, N:] > 0
    if sensors is not None:
        pert &= np.asarray(sensors, dtype=bool)[None, None, :]
    d_src = np.zeros((T, B, N), np.float32)
    d_st = None if static is None else np.zeros((B, ds), np.float32)
    e_cells = (np.arange(T)[:, None] * N + np.arange(N)[None, :]).astype(np.uint64)
    for b in range(B):
        base = np.uint64(b * (E + 1))
        p = pert[:, b, :]
        ps = np.full(ds, bool(perturb_static))
        if norm == "linf":
            u = (_words(seed, step, base + e_cells) >> np.uint32(8)).astype(np.float32) / np.float32(16777216.0)
            d_src[:, b, :] = np.where(p, np.float32(eps) * (np.float32(2.0) * u - np.float32(1.0)), 0).astype(np.float32)
            if ds and perturb_static:
                us = (_words(seed, step, base + np.uint64(T * N) + np.arange(ds, dtype=np.uint64)) >> np.uint32(8))
                us = us.astype(np.float32) / np.float32(16777216.0)
                d_st[b] = np.float32(eps) * (np.float32(2.0) * us - np.float32(1.0))
            continue
        z = np.where(p, _normals(seed, step, base + e_cells), 0).astype(np.float32)
        zs = _normals(seed, step, base + np.uint64(T * N) + np.arange(ds, dtype=np.uint64)) if ds else np.zeros(0, np.float32)
        zs = np.where(ps, zs, 0).astype(np.float32)
        d = int(p.sum() + ps.sum())
        zz = float((z.astype(np.float64) ** 2).sum() + (zs.astype(np.float64) ** 2).sum())
        if d == 0 or zz == 0:
            continue
        r = float(_words(seed, step, np.array([base + np.uint64(E)]))[0] >> np.uint32(8)) / 16777216.0
        s = float(np.float32(eps)) * r ** (1.0 / d) / np.sqrt(zz)
        d_src[:, b, :] = (z.astype(np.float64) * s).astype(np.float32)
        if ds:
            d_st[b] = (zs.astype(np.float64) * s).astype(np.float32)
    return d_src, d_st


# ---- CPU --------------------------------------------------------------------------------------------------------------
def test_symbols_exported():
    lib_path = os.path.join(ROOT, "raindrop_b200", "csrc", "librd_b200.so")
    out = subprocess.run(["nm", "-D", "--defined-only", lib_path], capture_output=True, text=True, check=True).stdout
    names = {line.split()[-1] for line in out.splitlines() if line.strip()}
    assert {"rd_pgd_scratch_bytes", "rd_raindrop_v2_pgd"} <= names


def test_scratch_query():
    import ctypes as C
    from raindrop_b200 import lib as L
    cfg = model_config("P19", dropout=0.2)
    model = build_dropin(cfg, 1, device="cpu")
    lib = L.load()
    dims = model._plan.dims(128, False)
    n1, n8 = lib.rd_pgd_scratch_bytes(C.byref(dims), 1), lib.rd_pgd_scratch_bytes(C.byref(dims), 8)
    assert 0 < n1 < n8
    assert lib.rd_pgd_scratch_bytes(C.byref(dims), 0) == 0


def _cpu_model():
    cfg = model_config("TINY", dropout=0.2)
    return build_dropin(cfg, 3, device="cpu").eval(), make_batch(cfg, 3, seed=1), cfg


def test_argument_validation():
    model, b, cfg = _cpu_model()
    args = (b["src"], b["static"], b["times"], b["lengths"])
    with pytest.raises(ValueError, match="eval"):
        ADV.pgd(model.train(), *args, eps=0.1)
    model.eval()
    bad = [dict(eps=-0.1), dict(eps=float("nan")), dict(eps=float("inf")), dict(eps=0.1, n_steps=-1),
           dict(eps=0.1, norm="l1"), dict(eps=0.1, step_size=-1.0), dict(eps=0.1, sensors=np.ones(cfg["d_inp"] + 1, bool)),
           dict(eps=0.1, sensors=np.ones(cfg["d_inp"], np.int64)), dict(eps=0.1, internal_batch_size=0),
           dict(eps=0.1, seed=-1), dict(eps=0.1, step=1 << 64)]
    for kw in bad:
        with pytest.raises(ValueError):
            ADV.pgd(model, *args, **kw)
    with pytest.raises(ValueError):
        ADV.pgd(model, *args, y=torch.tensor([0, 1, 99]), eps=0.1)
    with pytest.raises(ValueError):
        ADV.pgd(model, b["src"][:, :, :3], b["static"], b["times"], b["lengths"], eps=0.1)
    cfg8 = model_config("TINY8", dropout=0.2)
    m8, b8 = build_dropin(cfg8, 3, device="cpu").eval(), make_batch(cfg8, 2, seed=1)
    with pytest.raises(ValueError, match="static"):
        ADV.pgd(m8, b8["src"], None, b8["times"], b8["lengths"], eps=0.1, perturb_static=True)
    assert ADV._check_attack(0.2, "linf", 10, None)[3] == pytest.approx(0.05)
    assert ADV._check_attack(0.2, "l2", 0, None)[1:] == (1, 0, 0.0)


def test_no_cuda_raises(monkeypatch):
    from raindrop_b200.lib import RaindropB200Error
    model, b, _ = _cpu_model()
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RaindropB200Error):
        ADV.pgd(model, b["src"], b["static"], b["times"], b["lengths"], eps=0.1)


@pytest.mark.parametrize("norm", ["linf", "l2"])
@pytest.mark.parametrize("perturb_static", [False, True])
def test_random_start_restatement(norm, perturb_static):
    """The restated stream: linf draws fill [-eps, eps) and look uniform; l2 starts lie in the ball, with radii spread
    as r^(1/d); only perturbable cells move; the (seed, step) key changes the draw."""
    cfg = model_config("P19", dropout=0.2)
    b = make_batch(cfg, 64, seed=4)
    N, eps = cfg["d_inp"], 0.25
    sensors = np.arange(N) % 3 != 0
    d, ds = random_start(b["src"].numpy(), b["static"].numpy(), norm, eps, SEED, 5, sensors, perturb_static)
    pert = (b["src"].numpy()[:, :, N:] > 0) & sensors
    assert np.all(d[~pert] == 0) and pert.sum() > 100
    if not perturb_static:
        assert np.all(ds == 0)
    if norm == "linf":
        v = d[pert]
        assert np.all(np.abs(v) <= np.float32(eps)) and v.min() < -0.9 * eps and v.max() > 0.9 * eps
        assert abs(float(v.mean())) < 0.05 * eps and abs(float((v / eps).var()) - 1.0 / 3.0) < 0.05
    else:
        n = np.sqrt((d.astype(np.float64) ** 2).sum(axis=(0, 2)) + (ds.astype(np.float64) ** 2).sum(axis=1))
        n = n[pert.any(axis=(0, 2)) | perturb_static]
        assert np.all(n <= eps * (1 + 1e-6)) and n.max() > 0.9 * eps and n.min() > 0.5 * eps
    d2, _ = random_start(b["src"].numpy(), b["static"].numpy(), norm, eps, SEED, 6, sensors, perturb_static)
    assert not np.array_equal(d, d2)


# ---- GPU --------------------------------------------------------------------------------------------------------------
def _setup(name, mode=EXACT, wseed=9, dseed=3):
    cfg_name, B, opts = CASES[name]
    cfg = model_config(cfg_name, dropout=0.2)
    d = to_dev(make_batch(cfg, B, seed=dseed, **opts))
    model = build_dropin(cfg, wseed).eval()
    model._plan.obprop_mode = mode
    return cfg, d, model


def _args(d):
    return d["src"], d["static"], d["times"], d["lengths"]


def _ce(logits, y):
    return torch.nn.functional.cross_entropy(logits.double(), y, reduction="none")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_identity_without_budget(name):
    cfg, d, model = _setup(name)
    for kw in (dict(eps=0.0, n_steps=5), dict(eps=0.3, n_steps=0)):
        r = ADV.pgd(model, *_args(d), d["y"], random_start=False, **kw)
        assert torch.equal(r.src.view(torch.int32), d["src"].view(torch.int32))
        if d["static"] is not None:
            assert torch.equal(r.static, d["static"])
        assert torch.equal(r.logits, r.clean_logits)
        assert torch.allclose(r.loss.double(), _ce(r.clean_logits, d["y"]), rtol=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("norm", ["linf", "l2"])
@pytest.mark.parametrize("rs", [False, True], ids=["x0", "random"])
def test_invariants(name, norm, rs):
    cfg, d, model = _setup(name)
    N, eps = cfg["d_inp"], 0.3 if norm == "linf" else 1.5
    sensors = torch.arange(N) % 4 != 1
    ps = d["static"] is not None
    r = ADV.pgd(model, *_args(d), d["y"], eps=eps, norm=norm, n_steps=4, random_start=rs, seed=SEED, step=3,
                sensors=sensors, perturb_static=ps)
    src, x = r.src, d["src"]
    pert = (x[:, :, N:] > 0) & sensors.cuda()
    delta = (src[:, :, :N].double() - x[:, :, :N].double())
    bits, xbits = src.view(torch.int32), x.view(torch.int32)
    assert torch.equal(bits[:, :, N:], xbits[:, :, N:])
    assert torch.equal(bits[:, :, :N][~pert], xbits[:, :, :N][~pert])
    if norm == "linf":
        ulp = torch.finfo(torch.float32).eps * (x[:, :, :N].double().abs() + eps)
        assert torch.all(delta.abs() <= eps + ulp)
        if ps:
            assert torch.all((r.static.double() - d["static"].double()).abs() <= eps * (1 + 1e-6) + 1e-6)
    else:
        n2 = (delta ** 2).sum(dim=(0, 2))
        if ps:
            n2 = n2 + ((r.static.double() - d["static"].double()) ** 2).sum(1)
        # the delta read back through x + delta carries one fp32 rounding per cell
        slack = (torch.finfo(torch.float32).eps * (x[:, :, :N].double().abs() + delta.abs()) * pert).pow(2).sum(dim=(0, 2)).sqrt()
        assert torch.all(n2.sqrt() <= eps * (1 + 1e-6) + slack), (n2.sqrt(), slack)
    assert torch.allclose(r.loss.double(), _ce(r.logits, d["y"]), rtol=1e-5, atol=1e-6)
    if not rs:
        assert torch.all(r.loss.double() >= _ce(r.clean_logits, d["y"]).float().double() - 1e-6)
        assert float(r.loss.sum()) > float(_ce(r.clean_logits, d["y"]).sum())     # the attack does something
    assert torch.equal(r.success, r.logits.argmax(1) != d["y"])


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("mode", [EXACT, FAST], ids=["exact", "fast"])
def test_logits_are_module_forward(name, mode):
    """With one chunk of B rows, logits_adv is bitwise the module's eval forward on the returned input."""
    cfg, d, model = _setup(name, mode)
    B = d["src"].shape[1]
    r = ADV.pgd(model, *_args(d), d["y"], eps=0.2, n_steps=3, seed=1, perturb_static=d["static"] is not None,
                internal_batch_size=B)
    with torch.no_grad():
        f = model.forward(r.src, r.static if r.static is not None else d["static"], d["times"], d["lengths"])[0]
        c = model.forward(*_args(d))[0]
    assert torch.equal(r.logits, f)
    assert torch.equal(r.clean_logits, c)


def _oracle(cfg, wseed):
    from oracle.raindrop_oracle import build_oracle_model
    from raindrop_b200.synth import synth_weights
    o = build_oracle_model(cfg).eval()
    synth_weights(o, cfg, seed=wseed)
    return o.double()


def _oracle_grad(o, src, static, times, lengths, y):
    """Per-sample cross-entropies and their gradient w.r.t. the value half (and static) in float64."""
    s = src.clone().requires_grad_(True)
    st = static.clone().requires_grad_(True) if static is not None else None
    logits = o.forward_dense(s, st, times, lengths)[0]
    ce = torch.nn.functional.cross_entropy(logits, y, reduction="none")
    g = torch.autograd.grad(ce.sum(), [s] + ([st] if st is not None else []))
    return ce.detach(), g[0], (g[1] if st is not None else None)


def _oracle_pgd_l2(o, d, eps, alpha, K, ps):
    """L2 PGD without random start in float64, with the iterates' losses."""
    src, st = d["src"].cpu().double(), None if d["static"] is None else d["static"].cpu().double()
    times, lengths, y = d["times"].cpu().double(), d["lengths"].cpu(), d["y"].cpu()
    N = src.shape[2] // 2
    pert = (src[:, :, N:] > 0).double()
    dx = torch.zeros_like(src[:, :, :N])
    dst = torch.zeros_like(st) if (ps and st is not None) else None
    losses, deltas = [], []
    for k in range(K + 1):
        x = src.clone()
        x[:, :, :N] += dx
        sx = st + dst if dst is not None else st
        ce, g, gs = _oracle_grad(o, x, sx, times, lengths, y)
        losses.append(ce)
        deltas.append((dx.clone(), None if dst is None else dst.clone()))
        if k == K:
            break
        g = g[:, :, :N] * pert
        gn2 = (g ** 2).sum(dim=(0, 2))
        if dst is not None:
            gs = gs.clone()
            gn2 = gn2 + (gs ** 2).sum(1)
        gn = gn2.sqrt()
        step = torch.where(gn > 0, alpha / gn.clamp(min=1e-300), torch.zeros_like(gn))
        dx = dx + step[None, :, None] * g
        if dst is not None:
            dst = dst + step[:, None] * gs
        dn2 = (dx ** 2).sum(dim=(0, 2)) + ((dst ** 2).sum(1) if dst is not None else 0)
        sc = torch.clamp(eps / dn2.sqrt().clamp(min=1e-300), max=1.0)
        dx = dx * sc[None, :, None]
        if dst is not None:
            dst = dst * sc[:, None]
    return torch.stack(losses), deltas


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_l2_pgd_matches_oracle(name):
    cfg, d, model = _setup(name, EXACT)
    N, K = cfg["d_inp"], 3
    eps = 0.05 * float(np.sqrt(cfg["max_len"] * N))      # ~0.05 per cell, so the iterates' losses separate
    alpha = 0.5 * eps
    ps = d["static"] is not None
    r = ADV.pgd(model, *_args(d), d["y"], eps=eps, norm="l2", n_steps=K, step_size=alpha, random_start=False,
                perturb_static=ps)
    losses, deltas = _oracle_pgd_l2(_oracle(cfg, 9), d, eps, alpha, K, ps)
    got = (r.src[:, :, :N].double() - d["src"][:, :, :N].double()).cpu()
    tol = 1e-2 if cfg["max_len"] * cfg["d_ob"] >= 1024 else 2e-3
    checked = 0
    for b in range(got.shape[1]):
        lb = losses[:, b]
        srt = lb.sort(descending=True).values
        if srt[0] - srt[1] < 1e-4 * (1 + srt[0].abs()):       # near-tie in the best-iterate choice
            continue
        kb = int(lb.argmax())
        ref = deltas[kb][0][:, b]
        assert float((got[:, b] - ref).abs().max()) <= tol * max(float(ref.abs().max()), 1e-12), (b, kb)
        if ps:
            rs = deltas[kb][1][b]
            gs = (r.static[b].double() - d["static"][b].double()).cpu()
            assert float((gs - rs).abs().max()) <= tol * max(float(rs.abs().max()), 1e-12)
        assert abs(float(r.loss[b]) - float(lb[kb])) <= tol * (1 + abs(float(lb[kb])))
        checked += 1
    print(name, "samples checked against the oracle:", checked, "of", got.shape[1])
    assert checked >= 1


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_fgsm_signs_match_oracle(name):
    cfg, d, model = _setup(name, EXACT)
    N, eps = cfg["d_inp"], 0.05
    r = ADV.pgd(model, *_args(d), d["y"], eps=eps, n_steps=1, step_size=eps, random_start=False)
    o = _oracle(cfg, 9)
    src = d["src"].cpu().double()
    _, g, _ = _oracle_grad(o, src, None if d["static"] is None else d["static"].cpu().double(), d["times"].cpu().double(),
                           d["lengths"].cpu(), d["y"].cpu())
    g = g[:, :, :N] * (src[:, :, N:] > 0)
    ce0 = _ce(r.clean_logits, d["y"]).cpu()
    ce1 = _ce(r.logits, d["y"]).cpu()
    moved = (ce1 > ce0).cpu()                              # samples whose FGSM iterate was returned
    delta = (r.src[:, :, :N].double() - d["src"][:, :, :N].double()).cpu()
    big = g.abs() > 1e-3 * g.abs().amax(dim=(0, 2), keepdim=True)
    sel = big & moved[None, :, None]
    assert sel.any()
    assert torch.equal(torch.sign(delta[sel]), torch.sign(g[sel]))
    assert torch.all(delta[~moved[None, :, None].expand_as(delta)] == 0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny_b6", "tiny8_b5", "p12_b3"])
@pytest.mark.parametrize("norm", ["linf", "l2"])
def test_random_start_matches_restatement(name, norm):
    cfg, d, model = _setup(name)
    N, eps = cfg["d_inp"], 0.4
    ps = d["static"] is not None
    kw = dict(eps=eps, norm=norm, n_steps=0, random_start=True, seed=SEED, perturb_static=ps)
    r = ADV.pgd(model, *_args(d), d["y"], step=7, **kw)
    x = d["src"].cpu().numpy()
    dl, dls = random_start(x, None if d["static"] is None else d["static"].cpu().numpy(), norm, eps, SEED, 7, None, ps)
    want = np.where(dl == 0, x[:, :, :N], x[:, :, :N] + dl)
    got = r.src[:, :, :N].cpu().numpy()
    ulp = np.spacing(np.abs(want).astype(np.float32))
    assert np.all(np.abs(got - want) <= 2 * ulp)
    if ps:
        sw = d["static"].cpu().numpy() + dls
        assert np.all(np.abs(r.static.cpu().numpy() - sw) <= 2 * np.spacing(np.abs(sw).astype(np.float32)))
    r2 = ADV.pgd(model, *_args(d), d["y"], step=7, **kw)
    assert torch.equal(r.src, r2.src)
    r3 = ADV.pgd(model, *_args(d), d["y"], step=8, **kw)
    assert not torch.equal(r.src, r3.src)


@pytest.mark.gpu
@pytest.mark.parametrize("norm", ["linf", "l2"])
def test_chunking_and_repeat_bitwise_and_no_side_effects(norm):
    cfg, d, model = _setup("p19_b9", FAST)
    B = d["src"].shape[1]
    plan = model._prepare(torch.device("cuda"))
    snap = {"rng": plan.rng_state.clone()}
    snap.update({"param." + k: p.detach().clone() for k, p in model.named_parameters()})
    kw = dict(eps=0.3 if norm == "linf" else 2.0, norm=norm, n_steps=3, seed=5, step=2, perturb_static=True)
    res = [ADV.pgd(model, *_args(d), None, internal_batch_size=ib, **kw) for ib in (1, 7, B, B)]
    for r in res[1:]:
        for a, b in zip((r.src, r.static, r.logits, r.clean_logits, r.loss, r.success),
                        (res[0].src, res[0].static, res[0].logits, res[0].clean_logits, res[0].loss, res[0].success)):
            assert torch.equal(a, b)
    torch.cuda.synchronize()
    assert torch.equal(plan.rng_state, snap["rng"])
    for k, p in model.named_parameters():
        assert torch.equal(p.detach(), snap["param." + k]) and p.grad is None, k
    # y = None attacks the predicted class
    assert torch.equal(res[0].success, res[0].logits.argmax(1) != res[0].clean_logits.argmax(1))


# ---- adversarial training ---------------------------------------------------------------------------------------------
RNG0 = (0x1234ABCD5678, 11)


def _train_model(cfg, mode=EXACT):
    model = build_dropin(cfg, 21).train()
    plan = model._prepare(torch.device("cuda"))
    plan.obprop_mode = mode
    plan.rng_state.copy_(torch.tensor(RNG0, dtype=torch.int64))
    return model


def _run(step, n):
    losses = [step.step().clone() for _ in range(n)]
    torch.cuda.synchronize()
    return (step.flat_p.clone(), step.exp_avg.clone(), step.exp_avg_sq.clone(), torch.cat(losses),
            step.plan.rng_state.clone())


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
def test_adv_step_with_zero_budget_is_train_step(use_graph):
    from raindrop_b200.train import TrainStep
    cfg = model_config("P19", dropout=0.2)
    B = 37
    batch = to_dev(make_batch(cfg, B, seed=5))
    out = []
    for adv in (False, True):
        model = _train_model(cfg)
        s = ADV.AdversarialTrainStep(model, B, eps=0.0, n_steps=2, attack_seed=3, use_graph=use_graph) if adv \
            else TrainStep(model, B, use_graph=use_graph)
        s.load_batch(batch)
        out.append(_run(s, 3))
    for a, b in zip(*out):
        assert torch.equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("norm", ["linf", "l2"])
def test_adv_step_is_train_step_on_pgd_batch(use_graph, norm):
    """One step from a given state equals TrainStep on the batch pgd returns from that state; the attack key advances
    by one per step; unattacked slots train on their clean input."""
    from raindrop_b200.train import TrainStep
    cfg = model_config("TINY", dropout=0.2)
    B = 6
    batch = to_dev(make_batch(cfg, B, seed=7))
    attack = torch.tensor([True, False, True, True, False, True], device="cuda")
    eps, K = (0.3, 3) if norm == "linf" else (1.5, 3)
    model = _train_model(cfg)
    s = ADV.AdversarialTrainStep(model, B, eps=eps, norm=norm, n_steps=K, attack_seed=SEED, use_graph=use_graph, lr=1e-3)
    s.set_attack_key(SEED, 4)
    s.load_batch(dict(batch, attack=attack))
    s.step()                                        # moves the parameters: the second step attacks a trained model
    torch.cuda.synchronize()
    assert s.attack_key_state() == (SEED, 5)
    state = [t.clone() for t in s._state()]
    ref_model = _train_model(cfg)
    ref = TrainStep(ref_model, B, use_graph=False, lr=1e-3)
    ref.flat_p.copy_(s.flat_p); ref.exp_avg.copy_(s.exp_avg); ref.exp_avg_sq.copy_(s.exp_avg_sq)
    ref.step_count.copy_(s.step_count); ref.plan.rng_state.copy_(s.plan.rng_state)
    ref_model.eval()
    a = ADV.pgd(ref_model, *_args(batch), batch["y"], eps=eps, norm=norm, n_steps=K, seed=SEED, step=5,
                internal_batch_size=B)
    unatt = ~attack
    src = torch.where(attack[None, :, None], a.src, batch["src"])
    ref_model.train()
    ref.load_batch(dict(batch, src=src))
    got = _run(s, 1)
    want = _run(ref, 1)
    for x, y in zip(got, want):
        assert torch.equal(x, y)
    assert torch.equal(s.adv_src[:, unatt], batch["src"][:, unatt])
    assert torch.equal(s.adv_src[:, attack], a.src[:, attack])
    assert s.attack_key_state() == (SEED, 6)
    # resume: restoring the state and the key reproduces the step
    for t, v in zip(s._state(), state):
        t.copy_(v)
    s.set_attack_key(SEED, 5)
    again = _run(s, 1)
    for x, y in zip(got, again):
        assert torch.equal(x, y)


@pytest.mark.gpu
def test_adv_step_p19_graph_equals_eager():
    cfg = model_config("P19", dropout=0.2)
    B = 128
    batch = to_dev(make_batch(cfg, B, seed=12))
    out = []
    for use_graph in (False, True):
        s = ADV.AdversarialTrainStep(_train_model(cfg, FAST), B, eps=0.1, n_steps=3, attack_seed=1, use_graph=use_graph)
        s.load_batch(batch)
        out.append(_run(s, 2) + (s.adv_src.clone(), s.adv_loss.clone()))
    for a, b in zip(*out):
        assert torch.equal(a, b)
    assert torch.isfinite(out[0][3]).all()


def test_world_refused(monkeypatch):
    import torch.distributed as dist
    from raindrop_b200.lib import RaindropB200Error
    cfg = model_config("TINY", dropout=0.2)
    model = build_dropin(cfg, 3, device="cpu")
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    with pytest.raises(RaindropB200Error, match="one GPU"):
        ADV.AdversarialTrainStep(model, 4, eps=0.1)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 1)
    with pytest.raises(ValueError):
        ADV.AdversarialTrainStep(model, 4, eps=-1.0)
