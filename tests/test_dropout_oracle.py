"""CPU: the numpy restatement of the kernels' dropout stream (oracle/dropout_masks.py) and the mask-replaying
train-mode oracle (encoder_layer_explicit / RaindropV2Oracle.forward_dense with `masks=`) that the train-mode GPU
parity tests (test_train_parity.py) compare against."""
import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from helpers import normwise
from oracle import dropout_masks as DM
from oracle.raindrop_oracle import build_oracle_model, encoder_layer_explicit
from raindrop_b200.synth import make_batch, model_config, synth_weights, used_param_keys


# Random123 known-answer vectors for philox4x32_10 (kat_vectors): counter, key -> output
@pytest.mark.parametrize("ctr,key,out", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(ctr, key, out):
    assert DM.philox4x32_10(np.array(ctr), np.array(key)).tolist() == list(out)


def test_dropout_stream_layout():
    """Element idx takes word idx & 3 of the block with counter (idx >> 2, site, step lo) under key (seed lo,
    seed hi ^ step hi); the vectorised stream agrees with single-block calls, the decision with the 24-bit test."""
    seed, step, site = 0x0123456789ABCDEF, (5 << 32) | 17, 48 + 1
    n = 4 * 1000 + 3
    words = DM.dropout_words(seed, step, site, n)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) ^ (step >> 32)])
    for idx in (0, 1, 2, 3, 4, 2001, 4001, n - 1):
        blk = DM.philox4x32_10(np.array([idx >> 2, 0, site, step & 0xFFFFFFFF]), key)
        assert words[idx] == blk[idx & 3], idx
    for p in (0.1, 0.2, 0.5):
        m = DM.dropout_mask(seed, step, site, n, p)
        inv_keep = np.float32(1) / (np.float32(1) - np.float32(p))       # fp32 arithmetic, as in the kernels
        assert m.dtype == np.float32 and set(np.unique(m).tolist()) == {0.0, float(inv_keep)}
        assert np.array_equal(m > 0, (words >> 8) >= int(np.ceil(np.float32(p) * 2.0 ** 24)))
        assert abs((m > 0).mean() - (1 - p)) < 6 * np.sqrt(p * (1 - p) / n)
    # every input of the key/counter matters: seed hi, step hi, step lo, site
    for other in ((seed ^ (1 << 40), step, site), (seed, step ^ (1 << 33), site), (seed, step + 1, site),
                  (seed, step, site + 1)):
        assert not np.array_equal(DM.dropout_words(*other, n), words), other
    # the step's high word enters through the key only: flipping the same bit of seed hi and step hi cancels out
    assert np.array_equal(DM.dropout_words(seed ^ (1 << 40), step ^ (1 << 40), site, n), words)


def test_model_masks_layout():
    cfg = model_config("TINY", dropout=0.2)
    B, rng = 3, (7, 9)
    m = DM.model_masks(rng, 0.2, cfg, B)
    T, N, D = cfg["max_len"], cfg["d_inp"], cfg["d_inp"] * 4 + 16
    assert m["lift"].shape == (T, B, 4 * N) and len(m["layers"]) == cfg["nlayers"]
    L1 = m["layers"][1]
    assert L1["attn"].shape == (B, 2, T, T) and L1["resid1"].shape == (T * B, D)
    assert L1["ffn"].shape == (T * B, cfg["nhid"]) and L1["resid2"].shape == (T * B, D)
    # [b, h, query, key] is the row-major order of the index space [B, H, T, T] of site 16 + layer
    assert np.array_equal(L1["attn"].reshape(-1), DM.dropout_mask(7, 9, DM.SITE_ATTN + 1, B * 2 * T * T, 0.2))
    assert np.array_equal(m["lift"].reshape(-1), DM.dropout_mask(7, 9, DM.SITE_LIFT, T * B * 4 * N, 0.2))
    assert not np.array_equal(m["layers"][0]["resid1"], L1["resid1"])         # layers draw from their own sites
    assert not np.array_equal(L1["resid1"], L1["resid2"])


class _MaskMul(nn.Module):
    def __init__(self, mask):
        super().__init__()
        self.mask = mask

    def forward(self, x):
        return x * self.mask.reshape(x.shape)


def _torch_layer(D, H, nhid, p, seed):
    torch.manual_seed(seed)
    layer = nn.TransformerEncoderLayer(D, H, nhid, p).double()
    with torch.no_grad():
        for prm in layer.parameters():          # default LayerNorm affine is (1, 0): perturb so every term counts
            prm.add_(0.1 * torch.randn_like(prm))
    return layer


def _layer_case(seed):
    T, B, D, H, nhid = 9, 4, 24, 2, 40
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, B, D, generator=g, dtype=torch.float64)
    lengths = torch.tensor([9, 3, 1, 6])
    pad = torch.arange(T)[None, :] >= lengths[:, None]
    return T, B, D, H, nhid, x, pad


def test_masked_explicit_layer_with_unit_masks_matches_torch_eval():
    T, B, D, H, nhid, x, pad = _layer_case(0)
    layer = _torch_layer(D, H, nhid, 0.2, 0).eval()
    with torch.no_grad():
        ref = layer(x, src_key_padding_mask=pad)
    ones = dict(attn=np.ones((B, H, T, T)), resid1=np.ones((T * B, D)), ffn=np.ones((T * B, nhid)),
                resid2=np.ones((T * B, D)))
    with torch.no_grad():
        out = encoder_layer_explicit(x, pad, dict(layer.named_parameters()), H, masks=ones)
    valid = (~pad).T[:, :, None]
    assert normwise(out * valid, ref * valid) < 1e-12


@pytest.mark.parametrize("seed", range(3))
def test_masked_explicit_layer_matches_torch_train_mode(seed):
    """nn.TransformerEncoderLayer in TRAINING mode with dropout1 / dropout / dropout2 replaced by fixed mask
    multipliers == the explicit layer with the same masks, output and every gradient (float64).  The attention
    dropout runs inside torch's fused attention call and cannot be injected; the GPU attention operator test pins it."""
    T, B, D, H, nhid, x, pad = _layer_case(seed)
    p = 0.2
    rng = (1000 + seed, 3)
    masks = dict(resid1=DM.resid1_mask(rng, p, 0, T * B, D), ffn=DM.ffn_mask(rng, p, 0, T * B, nhid),
                 resid2=DM.resid2_mask(rng, p, 0, T * B, D))
    layer = _torch_layer(D, H, nhid, p, seed).train()
    layer.self_attn.dropout = 0.0
    layer.dropout1 = _MaskMul(torch.from_numpy(masks["resid1"]).double())
    layer.dropout = _MaskMul(torch.from_numpy(masks["ffn"]).double())
    layer.dropout2 = _MaskMul(torch.from_numpy(masks["resid2"]).double())
    xr = x.clone().requires_grad_(True)
    ref = layer(xr, src_key_padding_mask=pad)
    valid = (~pad).T[:, :, None].double()
    w = torch.randn(T, B, D, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * valid
    (ref * w).sum().backward()
    params = dict(layer.named_parameters())
    ref_grads = {k: v.grad.clone() for k, v in params.items()}
    for v in params.values():
        v.grad = None
    xe = x.clone().requires_grad_(True)
    out = encoder_layer_explicit(xe, pad, params, H, masks=masks)
    (out * w).sum().backward()
    assert normwise(out * valid, ref * valid) < 1e-12
    assert normwise(xe.grad, xr.grad) < 1e-12
    for k, v in params.items():
        assert normwise(v.grad, ref_grads[k]) < 1e-12, k
    # and the masks did act: the same layer without them is a different function
    plain = encoder_layer_explicit(x, pad, params, H)
    assert normwise(plain * valid, ref * valid) > 1e-2


def test_forward_dense_with_unit_masks_equals_forward_dense():
    cfg = model_config("TINY", dropout=0.2)
    B = 4
    batch = make_batch(cfg, B, seed=3)

    def run(masks):
        oracle = build_oracle_model(cfg).eval()
        synth_weights(oracle, cfg, seed=11)
        oracle.double()
        src = batch["src"].double().requires_grad_(True)
        logits, _, _ = oracle.forward_dense(src, batch["static"].double(), batch["times"].double(), batch["lengths"],
                                            masks=masks)
        F.cross_entropy(logits, batch["y"]).backward()
        g = dict(oracle.named_parameters())
        return logits.detach(), {k: g[k].grad for k in used_param_keys(cfg)}, src.grad

    l0, g0, s0 = run(None)
    l1, g1, s1 = run(DM.ones_masks(cfg, B))
    assert normwise(l1, l0) < 1e-12 and normwise(s1, s0) < 1e-12
    for k in g0:
        assert normwise(g1[k], g0[k]) < 1e-12, k
    l2, _, _ = run(DM.model_masks((5, 1), 0.2, cfg, B))
    assert normwise(l2, l0) > 1e-3            # real masks change the function


def test_dropout_words_at_arbitrary_indices():
    """dropout_words_at / dropout_mask_at (used to spot-check full-size masks) equal the sequential stream."""
    seed, step, site = 0x0123456789ABCDEF, (5 << 32) | 17, 16 + 1
    n = 4 * 777 + 2
    words = DM.dropout_words(seed, step, site, n)
    idx = np.random.default_rng(0).integers(0, n, 500)
    idx = np.concatenate([[0, 1, 2, 3, n - 1], idx])
    assert np.array_equal(DM.dropout_words_at(seed, step, site, idx), words[idx])
    assert np.array_equal(DM.dropout_mask_at(seed, step, site, idx, 0.2), DM.dropout_mask(seed, step, site, n, 0.2)[idx])
    # indices past 2^32 / 4 blocks carry into the counter's second word
    big = np.array([(1 << 34) + 5, (1 << 40) + 2], dtype=np.uint64)
    for i in big:
        blk = DM.philox4x32_10(np.array([int(i >> 2) & 0xFFFFFFFF, int(i >> 2) >> 32, site, step & 0xFFFFFFFF]),
                               np.array([seed & 0xFFFFFFFF, (seed >> 32) ^ (step >> 32)]))
        assert DM.dropout_words_at(seed, step, site, [i])[0] == blk[int(i) & 3]


def _dense_run(cfg, batch, masks, gates=None, stages=None, tf32_model=False):
    oracle = build_oracle_model(cfg).eval()
    synth_weights(oracle, cfg, seed=11)
    oracle.double()
    src = batch["src"].double().requires_grad_(True)
    times = batch["times"].double().requires_grad_(True)
    static = None if batch["static"] is None else batch["static"].double().requires_grad_(True)
    logits, _, _ = oracle.forward_dense(src, static, times, batch["lengths"], stages=stages, masks=masks, gates=gates,
                                        tf32_model=tf32_model)
    F.cross_entropy(logits, batch["y"]).backward()
    g = dict(oracle.named_parameters())
    out = dict(logits=logits.detach(), d_src=src.grad, d_times=times.grad)
    if static is not None:
        out["d_static"] = static.grad
    out.update({k: g[k].grad for k in used_param_keys(cfg)})
    return out


def own_gates(cfg, stages):
    """The gates of every site (forward_dense layout) that the oracle's own ReLU inputs in `stages` imply."""
    T, B = stages["obs"].shape[0], stages["obs"].shape[1]
    N, d_ob = cfg["d_inp"], cfg["d_ob"]
    pre2 = stages["obprop_pre"][1]                                   # [B, N, C] -> obs layout [T, B, N*d_ob]
    return dict(h1=stages["obprop_pre"][0] > 0,
                obs=(pre2 > 0).reshape(B, N, T, d_ob).permute(2, 0, 1, 3).reshape(T, B, N * d_ob),
                ffn=[(f > 0).reshape(T * B, -1) for f in stages["ffn_pre"]], head=stages["head_pre"] > 0)


@pytest.mark.parametrize("tf32_model", [False, True], ids=["plain", "tf32_model"])
@pytest.mark.parametrize("name", ["TINY", "TINY8"])
def test_gate_replay_with_own_gates_is_bitwise(name, tf32_model):
    """forward_dense(gates=...) with the gates the oracle's own ReLU inputs imply is the run without gates, bitwise, in
    the logits, every parameter gradient and the input gradients (float64, CPU); and a flipped gate at each site
    changes the result, so every site is wired."""
    cfg = model_config(name, dropout=0.2)
    B = 5
    batch = make_batch(cfg, B, seed=8)
    masks = DM.model_masks((3, 4), 0.2, cfg, B)
    stages = {}
    ref = _dense_run(cfg, batch, masks, stages=stages, tf32_model=tf32_model)
    gates = own_gates(cfg, stages)
    Df = cfg["d_inp"] * (cfg["d_ob"] + (1 if cfg["static"] else 0)) + 16
    assert len(gates["ffn"]) == cfg["nlayers"] and gates["head"].shape == (B, Df)
    got = _dense_run(cfg, batch, masks, gates=gates, tf32_model=tf32_model)
    assert got.keys() == ref.keys()
    for k in ref:
        assert torch.equal(got[k], ref[k]), k
        assert got[k].view(torch.int64).equal(ref[k].view(torch.int64)), k
    for site in ("h1", "obs", "ffn", "head"):
        flipped = dict(gates)
        if site == "ffn":
            f = gates["ffn"][0].clone()
            f[: f.shape[0] // 2] = ~f[: f.shape[0] // 2]
            flipped["ffn"] = [f] + gates["ffn"][1:]
        else:
            flipped[site] = ~gates[site]
        other = _dense_run(cfg, batch, masks, gates=flipped, tf32_model=tf32_model)
        assert not torch.equal(other["logits"], ref["logits"]), site


def test_chunked_training_reference_equals_one_batch():
    """dense_train_chunked: chunks of 2 samples (masks and gates sliced per chunk) give the one-batch loss, logits and
    gradients up to float64 summation order."""
    from oracle.raindrop_oracle import dense_train_chunked
    cfg = model_config("TINY", dropout=0.2)
    B = 5
    batch = make_batch(cfg, B, seed=9)
    masks = DM.model_masks((3, 5), 0.2, cfg, B)
    stages = {}
    ref = _dense_run(cfg, batch, masks, stages=stages)
    gates = own_gates(cfg, stages)
    oracle = build_oracle_model(cfg).eval()
    synth_weights(oracle, cfg, seed=11)
    oracle.double()
    seen = []
    out = dense_train_chunked(oracle, batch, masks=masks, gates=gates, chunk=2, input_grads=True,
                              on_chunk=lambda sl, st, lg: seen.append((sl.start, sl.stop, st["enc"].shape[1])))
    assert seen == [(0, 2, 2), (2, 4, 2), (4, 5, 1)]
    loss = F.cross_entropy(ref["logits"], batch["y"]).item()
    assert abs(out["loss"] - loss) < 1e-14 * abs(loss)
    assert normwise(out["logits"], ref["logits"]) < 1e-14
    for k in ("d_src", "d_times", "d_static"):
        assert normwise(out[k], ref[k]) < 1e-13, k
    g = dict(oracle.named_parameters())
    for k in used_param_keys(cfg):
        assert normwise(g[k].grad, ref[k]) < 1e-13, k
