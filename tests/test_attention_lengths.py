"""The tensor-core attention kernels (impl 1) across every key length of a launch, with attention dropout 0.2.

The forward draws its dropout decisions only for keys below each sample's length nv = min(length, T), one Philox block
per four keys.  These tests hold the kernels, at every nv, to
  * the float64 restatement (test_encoder_head.attention_reference, with the oracle's dropout mask), for one launch
    whose samples take every length from 0 to T + 1.  Length 0 lies outside the reference's envelope: those samples
    are held to finiteness and to the CUDA-core kernel (impl 2) in the same launch;
  * bitwise equality when the key rows past each sample's length (K and V rows nv <= t < T) hold other finite values.
"""
import pytest
import torch

from helpers import normwise
from test_encoder_head import RNG0, attention_reference, attention_run

gpu = pytest.mark.gpu
P = 0.2
SHAPES = [(60, 76), (60, 96), (64, 76), (64, 96)]


def every_length(T, hd, seed):
    g = torch.Generator().manual_seed(seed * 1000 + T * 100 + hd)
    H, B = 2, T + 2
    D = H * hd
    qkv = torch.randn(T, B, 3 * D, generator=g).cuda()
    dctx = torch.randn(T, B, D, generator=g).cuda()
    lengths = torch.arange(B, dtype=torch.int64).cuda()             # 0 .. T + 1
    return qkv, dctx, lengths, B, H, D


@gpu
@pytest.mark.parametrize("T,hd", SHAPES)
def test_attention_every_length_against_float64(T, hd):
    from oracle.dropout_masks import attention_mask
    qkv, dctx, lengths, B, H, D = every_length(T, hd, 1)
    rng = torch.tensor(RNG0, dtype=torch.int64, device="cuda")
    ctx, dq = attention_run(qkv, dctx, lengths, B, H, T, hd, P, 1, rng)
    assert torch.isfinite(ctx).all() and torch.isfinite(dq).all()
    drop = torch.from_numpy(attention_mask(RNG0, P, 0, B, H, T)).double().cuda()
    keep = torch.arange(1, B, device="cuda")
    ref, dref = attention_reference(qkv[:, keep], dctx[:, keep], lengths[keep], H, hd, drop[keep])
    e = max(normwise(ctx[:, keep], ref), normwise(dq[:, keep], dref))
    print("T %d hd %d: lengths 1..%d against float64 %.3e" % (T, hd, T + 1, e))
    assert e < 2e-5, e
    # length 0: every output of the sample is that of the CUDA-core kernel (zeros)
    ctx2, dq2 = attention_run(qkv, dctx, lengths, B, H, T, hd, P, 2, rng)
    assert torch.equal(ctx[:, 0], ctx2[:, 0]) and torch.equal(dq[:, 0], dq2[:, 0])
    assert float(ctx[:, 0].abs().max()) == 0.0 and float(dq[:, 0].abs().max()) == 0.0


@gpu
@pytest.mark.parametrize("T,hd", SHAPES)
def test_attention_ignores_padded_keys(T, hd):
    qkv, dctx, lengths, B, H, D = every_length(T, hd, 2)
    rng = torch.tensor(RNG0, dtype=torch.int64, device="cuda")
    a = attention_run(qkv, dctx, lengths, B, H, T, hd, P, 1, rng)
    pad = torch.arange(T, device="cuda")[:, None] >= lengths[None, :]           # [T, B]: key rows t >= nv
    g = torch.Generator(device="cuda").manual_seed(T + hd)
    other = qkv.clone()
    noise = 100.0 * torch.randn(T, B, 2 * D, generator=g, device="cuda")
    other[:, :, D:] = torch.where(pad[:, :, None], noise, qkv[:, :, D:])         # K and V rows past the length
    assert not torch.equal(other, qkv)
    b = attention_run(other, dctx, lengths, B, H, T, hd, P, 1, rng)
    for x, y in zip(a, b):
        assert torch.isfinite(x).all()
        assert torch.equal(x, y)
