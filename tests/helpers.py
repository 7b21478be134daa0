"""Shared test helpers (tests may import oracle/; the product never does)."""
import json
import os

import numpy as np
import torch

from raindrop_b200.synth import make_batch, model_config, synth_weights

N_SAMPLE = 509


def fingerprint(t):
    """Same summary as oracle/make_golden.py stores for tensors too large to commit."""
    f = t.detach().double().flatten().cpu()
    step = max(1, f.numel() // N_SAMPLE)
    return dict(stats=np.array([float(f.sum()), float(f.abs().sum()), float((f * f).sum().sqrt())]),
                sample=f[::step][:N_SAMPLE].float().numpy())


def sparse_structure(n, seed):
    g = torch.Generator().manual_seed(seed)
    a = (torch.rand(n, n, generator=g) < 0.35).float() * torch.rand(n, n, generator=g)
    a[n - 1, :] = 0
    a[:, 1] = 0
    return a


def load_golden(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name + ".npz"))
    meta = json.loads(bytes(z["meta"]).decode())
    return z, meta


def case_setup(meta):
    """cfg + batch of a golden case, regenerated from its seeds."""
    cfg = model_config(meta["config"], dropout=0.2)
    opt = meta["options"]
    if "sparse" in opt:
        cfg["global_structure"] = sparse_structure(cfg["d_inp"], opt["sparse"])
    batch = make_batch(cfg, meta["batch"], seed=meta["data_seed"], first_time_zero=opt.get("first_time_zero", False),
                       zero_sensors=opt.get("zero_sensors", 0))
    return cfg, batch


def normwise(a, b):
    a = torch.as_tensor(a).double().cpu()
    b = torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def rel_l2(a, b):
    a = torch.as_tensor(a).double().cpu()
    b = torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def check_against_golden(z, full, name, tensor, tol, errs, metric=normwise):
    """Compares `tensor` with the golden entry `name` (full tensor or fingerprint)."""
    if full:
        e = metric(tensor, z[name])
    else:
        fp = fingerprint(tensor)
        e = metric(fp["sample"], z[name + "#sample"])
        ref_stats = z[name + "#stats"]
        # l2 norm must agree too (catches errors outside the strided sample)
        e = max(e, abs(fp["stats"][2] - ref_stats[2]) / (ref_stats[2] + 1e-30))
    errs[name] = e
    assert e < tol, "%s: %s error %.3e >= %.1e" % (name, metric.__name__, e, tol)


def random_shape_case(seed):
    """(cfg, batch, weight_seed) of a seeded model shape the BASELINE configs do not hit: odd sensor counts (head dim
    not a multiple of 4), tiny and ragged T, 1..8 classes, with / without statics, random sparse weighted graphs,
    batch sizes around the 128-row tile edges."""
    g = torch.Generator().manual_seed(1000 + seed)
    ri = lambda lo, hi: int(torch.randint(lo, hi + 1, (1,), generator=g))
    N, T, B = ri(1, 13), ri(2, 70), [1, 2, 3, 5, 9, 17, 33, 64, 130][ri(0, 8)]
    static = bool(ri(0, 1))
    cfg = dict(name="RND", d_inp=N, max_len=T, d_static=ri(1, 7) if static else 0, n_classes=ri(2, 8), static=static,
               batch=B, p_obs=0.5, d_ob=4, d_model=4 * N, nhid=8 * N, nlayers=ri(1, 3), nhead=2, dropout=0.2, MAX=100)
    if ri(0, 1):
        a = (torch.rand(N, N, generator=g) < 0.4).float() * torch.rand(N, N, generator=g)
        cfg["global_structure"] = a
    batch = make_batch(cfg, B, seed=seed, first_time_zero=bool(ri(0, 1)))
    return cfg, batch, 40 + seed


def build_dropin(cfg, weight_seed, device="cuda"):
    from raindrop_b200.models_rd import Raindrop_v2
    torch.manual_seed(1)
    gs = cfg.get("global_structure")
    gs = torch.ones(cfg["d_inp"], cfg["d_inp"]) if gs is None else gs.clone()
    kw = {} if cfg["static"] else {"static": False}
    m = Raindrop_v2(cfg["d_inp"], cfg["d_model"], cfg["nhead"], cfg["nhid"], cfg["nlayers"], cfg["dropout"],
                    cfg["max_len"], cfg["d_static"], cfg["MAX"], 0.5, "mean", cfg["n_classes"], gs, **kw)
    synth_weights(m, cfg, seed=weight_seed)
    return m.to(device) if device != "cpu" else m


def to_dev(batch, device="cuda"):
    return {k: (v.to(device) if v is not None else None) for k, v in batch.items()}
