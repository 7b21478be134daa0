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


# ---- the GPU's ReLU decisions, for the gate-replaying oracle (RaindropV2Oracle.forward_dense(gates=...)) -------------
GATE_SITES = ("h1", "obs", "ffn", "head")


def ws_view(dims, ws, which):
    """Named buffer `which` (rd_ws_buffer) of a forward's workspace."""
    import ctypes as C
    from raindrop_b200 import lib as L
    n = C.c_int64(0)
    off = L.load().rd_workspace_offset(C.byref(dims), which, C.byref(n))
    assert off >= 0, which
    return ws[off // 4: off // 4 + n.value]


def read_gpu(cfg, dims, ws):
    """What a forward left in its workspace: the gates of the four ReLU sites in forward_dense's layout (H1 > 0; the obs
    columns of the encoder input > 0; each layer's FFN activation > 0, whatever its gate where the mask dropped; the
    head's hidden activation > 0), the (rounded) layer-1 output and the encoder input and output."""
    from raindrop_b200 import lib as L
    T, B, N, d_ob = dims.T, dims.B, cfg["d_inp"], cfg["d_ob"]
    D = N * d_ob + 16
    h1 = ws_view(dims, ws, L.WS_H1).view(B, N, -1)
    enc_in = ws_view(dims, ws, L.WS_ENC_IN).view(T, B, D)
    ffn = [ws_view(dims, ws, L.WS_FFN + l).view(T * B, -1) for l in range(cfg["nlayers"])]
    gates = dict(h1=h1 > 0, obs=enc_in[:, :, :N * d_ob] > 0, ffn=[f > 0 for f in ffn],
                 head=ws_view(dims, ws, L.WS_HEAD_HIDDEN).view(B, -1) > 0)
    return dict(gates=gates, h1=h1.clone(), enc_in=enc_in.clone(),
                enc_out=ws_view(dims, ws, L.WS_ENC_OUT).view(T, B, D).clone())


def gate_disagreements(cfg, gates, stages, masks, sl, B, counts):
    """Adds to counts[site] = [disagreeing, gates] the gates of samples `sl` (a slice of a batch of B) where the GPU's
    decision differs from the sign of the oracle's own ReLU input (`stages` of forward_dense on those samples).  FFN
    gates count only where the mask kept the element (all of them without an FFN mask: eval)."""
    T, N, d_ob = cfg["max_len"], cfg["d_inp"], cfg["d_ob"]
    Bc = sl.stop - sl.start
    dev = stages["obs"].device
    pre2 = stages["obprop_pre"][1].reshape(Bc, N, T, d_ob).permute(2, 0, 1, 3).reshape(T, Bc, N * d_ob)
    for site, mine, own in (("h1", gates["h1"][sl], stages["obprop_pre"][0] > 0), ("obs", gates["obs"][:, sl], pre2 > 0),
                            ("head", gates["head"][sl], stages["head_pre"] > 0)):
        counts[site][0] += int((mine.to(dev) != own).sum())
        counts[site][1] += mine.numel()
    for l, f in enumerate(stages.get("ffn_pre", [])):
        mk = None if masks is None else masks["layers"][l].get("ffn")
        kept = torch.ones_like(f, dtype=torch.bool) if mk is None else \
            torch.as_tensor(mk, device=dev).reshape(T, B, -1)[:, sl] > 0
        mine = gates["ffn"][l].reshape(T, B, -1)[:, sl].to(dev)
        counts["ffn"][0] += int(((mine != (f > 0)) & kept).sum())
        counts["ffn"][1] += int(kept.sum())
    return counts


def tf32_ulp_distance(gpu_h1, own_h1, counts):
    """Adds to counts = [elements, 1 TF32 ulp apart, more than 1 ulp apart, GPU values not TF32-representable] the
    comparison of the GPU's TF32-rounded layer-1 output with the rounding model's own (stages["h1_own"]), over the
    elements where both are positive (where one is not, the gate disagreement counts see it).  Both should hold TF32
    values, so their fp32 bit patterns differ by a multiple of 2^13 and, for positive values, the pattern difference
    >> 13 is their distance in TF32 ulps."""
    a, b = gpu_h1.float(), own_h1.to(gpu_h1.device).float()
    ia = a.view(torch.int32)
    both = (a > 0) & (b > 0)
    d = ((ia - b.view(torch.int32)).abs() >> 13)[both]
    counts[0] += int(both.sum())
    counts[1] += int((d == 1).sum())
    counts[2] += int((d > 1).sum())
    counts[3] += int(((ia & 0x1FFF) != 0).sum())
    return counts


def h1_ulp_ok(counts, rates):
    """counts of tf32_ulp_distance within rates = (1-ulp rate, more-than-1-ulp rate); every GPU value TF32."""
    n, one, more, unrounded = counts
    return n > 0 and unrounded == 0 and one <= rates[0] * n and more <= rates[1] * n
