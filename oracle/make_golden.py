"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/*.npz by running the reference's own,
unmodified files (oracle/ref_harness.py) on CPU in the build container:

    RAINDROP_REFERENCE=<checkout of mims-harvard/Raindrop> python -m oracle.make_golden      # from the repo root

A fixture stores seeds + the reference's outputs; inputs and weights are regenerated from the
seeds by raindrop_b200.synth (make_batch / synth_weights), so the files stay small.  Stored per
case: logits, distance, the observation-propagation output `obs` [T,B,4N] (input of the temporal
attention, code/models_rd.py:341), the encoder output `enc` [T,B,D] (code/models_rd.py:358), the
cross-entropy loss and the gradient of every parameter that receives one -- in full for tiny
shapes, as fingerprints (sum / abs-sum / l2 / strided sample) for the BASELINE shapes.
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_harness  # noqa: E402
from raindrop_b200.synth import make_batch, model_config, synth_weights, used_param_keys  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
N_SAMPLE = 509


def fingerprint(t):
    """Order-sensitive summary used when the full tensor is too big to commit."""
    f = t.detach().double().flatten()
    step = max(1, f.numel() // N_SAMPLE)
    return dict(sum=float(f.sum()), asum=float(f.abs().sum()), l2=float((f * f).sum().sqrt()),
                sample=f[::step][:N_SAMPLE].float().numpy())


def sparse_structure(n, seed):
    g = torch.Generator().manual_seed(seed)
    a = (torch.rand(n, n, generator=g) < 0.35).float() * torch.rand(n, n, generator=g)
    a[n - 1, :] = 0   # a node with no outgoing edges ...
    a[:, 1] = 0       # ... and one whose only incoming edge is the forced self loop
    return a


CASES = [
    # name, config, batch, data seed, weight seed, options
    ("tiny_dense", "TINY", 3, 11, 7, {}),
    ("tiny_t0", "TINY", 3, 12, 8, {"first_time_zero": True}),
    ("tiny_sparse", "TINY", 4, 13, 9, {"sparse": 5}),
    ("tiny8_nostatic", "TINY8", 4, 14, 10, {}),
    ("p19_b4", "P19", 4, 15, 11, {}),
    ("p19_b5_leave10", "P19", 5, 16, 12, {"zero_sensors": 10}),
    ("p12_b2", "P12", 2, 17, 13, {"first_time_zero": True}),
    ("pam_b2", "PAM", 2, 18, 14, {"first_time_zero": True}),
]


def run_case(name, cfg_name, B, dseed, wseed, opt):
    cfg = model_config(cfg_name, dropout=0.2)
    if "sparse" in opt:
        cfg["global_structure"] = sparse_structure(cfg["d_inp"], opt["sparse"])
    model = ref_harness.build_reference_model(cfg).eval()   # eval: dropout off, parity is exact
    synth_weights(model, cfg, seed=wseed)
    batch = make_batch(cfg, B, seed=dseed, first_time_zero=opt.get("first_time_zero", False),
                       zero_sensors=opt.get("zero_sensors", 0))
    grabbed = {}
    h1 = model.transformer_encoder.register_forward_hook(lambda m, i, o: grabbed.update(enc=o, obs=i[0]))
    logits, distance, _ = model.forward(batch["src"], batch["static"], batch["times"], batch["lengths"])
    h1.remove()
    loss = F.cross_entropy(logits, batch["y"])
    model.zero_grad()
    loss.backward()
    tiny = cfg_name.startswith("TINY")
    out = dict(logits=logits.detach().numpy(), distance=np.float32(distance.item()),
               loss=np.float32(loss.item()))
    D4 = cfg["d_inp"] * cfg["d_ob"]
    tensors = dict(obs=grabbed["obs"][:, :, :D4], pe=grabbed["obs"][:, :, D4:], enc=grabbed["enc"])
    grads = {}
    params = dict(model.named_parameters())
    with_grad = sorted(k for k, p in params.items() if p.grad is not None)
    assert with_grad == sorted(used_param_keys(cfg)), set(with_grad) ^ set(used_param_keys(cfg))
    for k in with_grad:
        grads["grad." + k] = params[k].grad
    tensors.update(grads)
    for k, t in tensors.items():
        if tiny:
            out[k] = t.detach().numpy()
        else:
            fp = fingerprint(t)
            out[k + "#sample"] = fp["sample"]
            out[k + "#stats"] = np.array([fp["sum"], fp["asum"], fp["l2"]], dtype=np.float64)
    meta = dict(case=name, config=cfg_name, batch=B, data_seed=dseed, weight_seed=wseed, options=opt,
                torch=torch.__version__, reference_commit="892eb57",
                generator="oracle/make_golden.py", full_tensors=tiny)
    out["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(GOLDEN, name + ".npz"), **out)
    print("%-18s logits[0]=%s loss=%.6f  %d arrays" % (name, logits[0].tolist(), loss.item(), len(out)))


# Raindrop_v2 away from the defaults of synth.model_config (d_ob = 4, nhead = 2, nhid = 2 d_model, 2 layers): name ->
# (hyper-parameters, batch, data seed, weight seed).  D = N d_ob + 16; tests/test_hparams.py builds the same models.
HPARAM_CASES = {
    # D = 52, hd = 13, nhid % 4 != 0, d_ob = 3, five layers
    "A": (dict(d_inp=12, d_ob=3, nhead=4, nhid=50, nlayers=5, max_len=40, d_static=4, n_classes=3), 9, 411, 41),
    # D = 32, hd = 4, eight layers, no statics
    "B": (dict(d_inp=8, d_ob=2, nhead=8, nhid=64, nlayers=8, max_len=48, d_static=0, n_classes=2), 6, 252, 42),
    # D = 26 (D % 4 != 0), d_ob = 1, C = T = 130
    "C": (dict(d_inp=10, d_ob=1, nhead=2, nhid=37, nlayers=3, max_len=130, d_static=2, n_classes=4), 3, 53, 43),
}
HPARAM_FULL_MAX = 4096      # tensors up to this many elements are stored in full, larger ones as fingerprints


def hparam_config(name, hp):
    """synth-style cfg of a HPARAM_CASES entry (dropout 0.2 as everywhere; fixtures are taken in eval mode)."""
    cfg = dict(hp, name="HP_" + name, static=hp["d_static"] > 0, p_obs=0.5, dropout=0.2, MAX=100)
    cfg["d_model"] = cfg["d_inp"] * cfg["d_ob"]
    return cfg


def hparam_cases():
    """The reference's own Raindrop_v2 (eval mode) at HPARAM_CASES -> hparams_<case>.npz: logits, loss, the obs / pe /
    enc stages and the gradient of every parameter that gets one.  `meta` carries the full cfg."""
    for name, (hp, B, dseed, wseed) in HPARAM_CASES.items():
        cfg = hparam_config(name, hp)
        model = ref_harness.build_reference_model(cfg).eval()
        synth_weights(model, cfg, seed=wseed)
        batch = make_batch(cfg, B, seed=dseed)
        grabbed = {}
        h = model.transformer_encoder.register_forward_hook(lambda m, i, o: grabbed.update(enc=o, obs=i[0]))
        logits, distance, _ = model.forward(batch["src"], batch["static"], batch["times"], batch["lengths"])
        h.remove()
        loss = F.cross_entropy(logits, batch["y"])
        model.zero_grad()
        loss.backward()
        D4 = cfg["d_inp"] * cfg["d_ob"]
        tensors = dict(obs=grabbed["obs"][:, :, :D4], pe=grabbed["obs"][:, :, D4:], enc=grabbed["enc"])
        params = dict(model.named_parameters())
        with_grad = sorted(k for k, p in params.items() if p.grad is not None)
        assert with_grad == sorted(used_param_keys(cfg)), set(with_grad) ^ set(used_param_keys(cfg))
        tensors.update({"grad." + k: params[k].grad for k in with_grad})
        out = dict(logits=logits.detach().numpy(), distance=np.float32(distance.item()), loss=np.float32(loss.item()))
        for k, t in tensors.items():
            if t.numel() <= HPARAM_FULL_MAX:
                out[k] = t.detach().numpy()
            else:
                fp = fingerprint(t)
                out[k + "#sample"] = fp["sample"]
                out[k + "#stats"] = np.array([fp["sum"], fp["asum"], fp["l2"]], dtype=np.float64)
        meta = dict(case="hparams_" + name, cfg=cfg, batch=B, data_seed=dseed, weight_seed=wseed, torch=torch.__version__,
                    reference_commit="892eb57", generator="oracle/make_golden.py hparams")
        out["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
        np.savez_compressed(os.path.join(GOLDEN, "hparams_%s.npz" % name), **out)
        print("hparams_%s  logits[0]=%s loss=%.6f  %d arrays" % (name, logits[0].tolist(), loss.item(), len(out)))


def operator_cases():
    """Operator-level fixtures: `Observation_progation` with use_beta both ways on a sparse
    weighted graph, and `TransformerConv` with and without supplied edge weights."""
    ref = ref_harness.load_reference()
    from raindrop_b200.synth import _stream
    out = {}
    N, T, d_ob = 6, 5, 4
    C = T * d_ob
    torch.manual_seed(3)
    layer = ref.Observation_progation(in_channels=C, out_channels=C, heads=1, n_nodes=N, ob_dim=d_ob)
    adj = sparse_structure(N, 21)
    adj[torch.arange(N), torch.arange(N)] = 1
    ei = torch.nonzero(adj).T.contiguous()
    ew = adj[ei[0], ei[1]]
    x = torch.from_numpy(_stream(5, "op.x", N * C)).float().view(N, C) - 0.3
    p_t = torch.from_numpy(_stream(5, "op.pt", T * 16)).float().view(T, 16)
    for k, v in layer.state_dict().items():
        out["obprop.sd." + k] = v.numpy()
    for ub in (False, True):
        o, (ei2, al) = layer(x, p_t=p_t, edge_index=ei, edge_weights=ew, use_beta=ub, edge_attr=None,
                             return_attention_weights=True)
        tag = "obprop.beta%d." % int(ub)
        out[tag + "out"] = o.detach().numpy()
        out[tag + "edge_index"] = ei2.numpy()
        out[tag + "alpha"] = al.detach().numpy()
    out["obprop.x"], out["obprop.p_t"] = x.numpy(), p_t.numpy()
    out["obprop.edge_index"], out["obprop.edge_w"] = ei.numpy(), ew.numpy()

    # with supplied edge weights the reference only works for heads == 1 (alpha is [E,1] and is
    # viewed as [-1, heads, 1], code/transformer_conv.py:199-206); the QK path takes any heads.
    xn = torch.from_numpy(_stream(6, "tc.x", N * 7)).float().view(N, 7) - 0.5
    out["tconv.x"] = xn.numpy()
    for tag, heads, w, seed in (("tconv.w.", 1, ew, 4), ("tconv.qk.", 2, None, 5)):
        torch.manual_seed(seed)
        conv = ref.TransformerConv(in_channels=7, out_channels=5, heads=heads)
        for k, v in conv.state_dict().items():
            out[tag + "sd." + k] = v.numpy()
        o, (_, al) = conv(xn, edge_index=ei, edge_weights=w, edge_attr=None, return_attention_weights=True)
        out[tag + "out"] = o.detach().numpy()
        out[tag + "alpha"] = al.detach().numpy()
    np.savez_compressed(os.path.join(GOLDEN, "operators.npz"), **out)
    print("operators          %d arrays" % len(out))


def operator_grad_cases():
    """Gradient fixtures of the two graph operators (reference autograd through code/Ob_propagation.py and
    code/transformer_conv.py under the PyG shim): loss = sum(out * G) [+ sum(alpha * g) for use_beta=True, whose
    returned alpha is differentiable and feeds layer 2 in code/models_rd.py:332-336].  Inputs / weights are the ones
    of operators.npz; written to operators_grad.npz."""
    ref = ref_harness.load_reference()
    from raindrop_b200.synth import _stream
    z = np.load(os.path.join(GOLDEN, "operators.npz"))
    out = {}
    ei = torch.from_numpy(z["obprop.edge_index"])
    N, C = z["obprop.x"].shape
    T, d_ob = z["obprop.p_t"].shape[0], 4
    layer = ref.Observation_progation(in_channels=C, out_channels=C, heads=1, n_nodes=N, ob_dim=d_ob)
    layer.load_state_dict({k[len("obprop.sd."):]: torch.from_numpy(z[k]) for k in z.files if k.startswith("obprop.sd.")})
    G = torch.from_numpy(_stream(9, "opg.G", N * C)).float().view(N, C) - 0.5
    out["obprop.G"] = G.numpy()
    for ub in (False, True):
        layer.zero_grad()
        x = torch.from_numpy(z["obprop.x"]).clone().requires_grad_(True)
        p_t = torch.from_numpy(z["obprop.p_t"]).clone().requires_grad_(True)
        ew = torch.from_numpy(z["obprop.edge_w"]).clone().requires_grad_(True)
        o, (ei2, al) = layer(x, p_t=p_t, edge_index=ei, edge_weights=ew, use_beta=ub, edge_attr=None, return_attention_weights=True)
        loss = (o * G).sum()
        tag = "obprop.beta%d." % int(ub)
        if ub:
            g = torch.from_numpy(_stream(9, "opg.g", al.numel())).float() - 0.5
            out[tag + "g_alpha"] = g.numpy()
            loss = loss + (al * g).sum()
        loss.backward()
        out[tag + "d_x"] = x.grad.numpy()
        out[tag + "d_edge_w"] = (ew.grad if ew.grad is not None else torch.zeros_like(ew)).numpy()
        if ub:
            out[tag + "d_p_t"] = p_t.grad.numpy()
        for k, prm in layer.named_parameters():
            if prm.grad is not None:
                out[tag + "grad." + k] = prm.grad.numpy()
    xn0 = torch.from_numpy(z["tconv.x"])
    for tag, heads, use_w in (("tconv.w.", 1, True), ("tconv.qk.", 2, False)):
        conv = ref.TransformerConv(in_channels=7, out_channels=5, heads=heads)
        conv.load_state_dict({k[len(tag + "sd."):]: torch.from_numpy(z[k]) for k in z.files if k.startswith(tag + "sd.")})
        xn = xn0.clone().requires_grad_(True)
        ew = torch.from_numpy(z["obprop.edge_w"]).clone().requires_grad_(True)
        G2 = torch.from_numpy(_stream(9, tag + "G", N * 5 * heads)).float().view(N, 5 * heads) - 0.5
        o, _ = conv(xn, edge_index=ei, edge_weights=ew if use_w else None, edge_attr=None, return_attention_weights=True)
        (o * G2).sum().backward()
        out[tag + "G"] = G2.numpy()
        out[tag + "d_x"] = xn.grad.numpy()
        if use_w:
            out[tag + "d_edge_w"] = ew.grad.numpy()
        for k, prm in conv.named_parameters():
            out[tag + "grad." + k] = (prm.grad if prm.grad is not None else torch.zeros_like(prm)).numpy()
    np.savez_compressed(os.path.join(GOLDEN, "operators_grad.npz"), **out)
    print("operators_grad     %d arrays: %s" % (len(out), sorted(out)[:60]))


# name, batch, data seed, model seed, (d_model, nhead, nhid, nlayers), graph density, isolated sensor (or None)
V1_CASES = [
    ("v1_p12_b3", 3, 77, 5, (72, 2, 144, 2), 0.5, None),
    ("v1_sparse_b5", 5, 78, 6, (36, 2, 64, 1), 0.15, 7),      # 1075 rows; sensor 7 keeps only its forced self loop
    ("v1_b1", 1, 79, 7, (72, 4, 36, 1), 0.5, None),           # one graph: the batched operator with n_graphs = 1
]


def v1_case(name, B, data_seed, model_seed, shape, density, isolated):
    """Legacy `Raindrop` v1 (code/models_rd.py:46-191; hard-coded to 36 sensors / 215 steps, so a case can vary the
    batch, the encoder's shape and the sensor graph but not d_inp or T): logits, loss and the gradient of every
    parameter that gets one, eval mode.  Weights: seeded default init, but `encoder` / `emb` re-drawn at a useful scale
    (the reference initialises them to +-1e-10, which would hide the graph layer)."""
    ref = ref_harness.load_reference()
    from raindrop_b200.synth import CONFIGS
    cfg = dict(CONFIGS["P12"]); cfg["name"] = "P12"
    batch = make_batch(dict(cfg, d_ob=2), B, seed=data_seed)
    torch.manual_seed(model_seed)
    gs = (torch.rand(36, 36) < density).float() * torch.rand(36, 36)
    if isolated is not None:
        gs[isolated, :] = 0
        gs[:, isolated] = 0
    d_model, nhead, nhid, nlayers = shape
    ctor = [36, d_model, nhead, nhid, nlayers, 0.2, 215, 9, 100, 0.5, "mean", 2]
    model = ref.Raindrop(*ctor, gs.clone()).eval()
    with torch.no_grad():
        model.encoder.weight.uniform_(-0.3, 0.3)
        model.emb.weight.uniform_(-0.3, 0.3)
    logits, distance, _ = model.forward(batch["src"], batch["static"], batch["times"], batch["lengths"])
    loss = F.cross_entropy(logits, batch["y"])
    model.zero_grad()
    loss.backward()
    out = dict(logits=logits.detach().numpy(), loss=np.float32(loss.item()), distance=np.float32(float(distance)),
               global_structure=gs.numpy())
    for k, v in model.state_dict().items():
        out["sd." + k] = v.numpy()
    for k, prm in model.named_parameters():
        if prm.grad is not None:
            out["grad." + k] = prm.grad.numpy()
    meta = dict(case=name, batch=B, data_seed=data_seed, ctor=ctor, torch=torch.__version__, reference_commit="892eb57",
                generator="oracle/make_golden.py v1")
    out["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(GOLDEN, name + ".npz"), **out)
    print("%s  logits[0]=%s loss=%.6f distance=%g grads for %d tensors" %
          (name, logits[0].tolist(), loss.item(), float(distance), sum(1 for k in out if k.startswith("grad."))))


def data_utils_case():
    """The reference's own host-side data functions (code/utils_rd.py) on oracle.data_oracle.synthetic_raw(seed=4)
    -> data_utils.npz (pins oracle/data_oracle.py)."""
    ref_harness.load_reference()                       # puts the reference's code/ on sys.path
    import utils_rd as U
    from oracle import data_oracle as DO
    P, minutes, static, y = DO.synthetic_raw(seed=4)
    out = {}
    try:
        mf, stdf = U.getStats(P)
        out["getStats.mf"], out["getStats.stdf"] = mf, stdf
    except ValueError:
        # numpy >= 1.24 rejects `np.max([stdf[f], eps])` (code/utils_rd.py:160); the rest runs on the restatement's stats
        mf, stdf = DO.get_stats(P)
    out["mask_normalize"] = U.mask_normalize(P.copy(), mf, stdf)
    ms, ss = U.getStats_static(static, dataset="P12")
    out["getStats_static.ms"], out["getStats_static.ss"] = np.asarray(ms), np.asarray(ss)
    out["mask_normalize_static"] = U.mask_normalize_static(static.copy(), ms, ss)
    Plist = [{"arr": P[i], "time": minutes[i][:, None], "extended_static": static[i]} for i in range(len(P))]
    for i, t in enumerate(U.tensorize_normalize(Plist, y, mf, stdf, ms, ss)):
        out["tensorize_normalize.%d" % i] = t.numpy()
    np.savez_compressed(os.path.join(GOLDEN, "data_utils.npz"), **out)
    print("data_utils  %d arrays" % len(out))


def live_tiny_case():
    """Raindrop_v2 of the reference built and run on the TINY configuration -> live_tiny.npz: digests of its initial state
    dict (in module order) and eval-mode logits on make_batch(cfg, 3, seed=1)."""
    cfg = model_config("TINY", dropout=0.2)
    ref = ref_harness.build_reference_model(cfg).eval()
    batch = make_batch(cfg, 3, seed=1)
    with torch.no_grad():
        logits = ref.forward(batch["src"], batch["static"], batch["times"], batch["lengths"])[0]
    # the state dict is pinned bit for bit through SHA-256 digests of its float32 bytes (the tensors themselves are 300 KB)
    digests = [hashlib.sha256(v.contiguous().numpy().tobytes()).hexdigest() for v in ref.state_dict().values()]
    out = {"state_sha256": np.array(digests), "logits": logits.numpy()}
    np.savez_compressed(os.path.join(GOLDEN, "live_tiny.npz"), **out)
    print("live_tiny  logits[0]=%s, %d state tensors" % (logits[0].tolist(), len(digests)))


if __name__ == "__main__":
    os.makedirs(GOLDEN, exist_ok=True)
    torch.set_num_threads(8)
    if len(sys.argv) > 1 and sys.argv[1] == "operators_grad":      # add-on fixtures: leaves the existing files untouched
        operator_grad_cases()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "v1":          # optionally followed by the case names to (re)generate
        for case in V1_CASES:
            if len(sys.argv) == 2 or case[0] in sys.argv[2:]:
                v1_case(*case)
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "hparams":
        hparam_cases()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "live":
        data_utils_case()
        live_tiny_case()
        sys.exit(0)
    for case in CASES:
        run_case(*case)
    operator_cases()
    operator_grad_cases()
    for case in V1_CASES:
        v1_case(*case)
    data_utils_case()
    live_tiny_case()
    hparam_cases()
