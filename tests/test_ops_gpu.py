"""GPU parity of the operator-level C-ABI entry points against the CPU oracle (oracle/unet_oracle.py).

Tolerances (floating point; stated per test): GEMM-shaped ops take f16 operands (the reference's diffuser
is f16, src/bin/sample/main.rs:122,241) and accumulate in f32, so inputs are pre-rounded to f16 and the
oracle runs on the SAME rounded values in f32 — what remains is accumulation order (~1e-6 relative) plus,
where the output itself is f16, one output rounding (2^-11 relative).
"""
import math

import numpy as np
import pytest
import torch

from oracle import philox
from oracle import unet_oracle as O
from harness import rel_err

pytestmark = pytest.mark.gpu


def h16(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.float16)


@pytest.mark.parametrize("M,K,N", [(128, 64, 64), (256, 320, 320), (77 * 2, 2048, 2560), (1024, 1280, 3840),
                                   (200, 136, 48), (16, 64, 16), (2048, 640, 640), (300, 1280, 1280)])
def test_linear(ctx, M, K, N):
    g = torch.Generator().manual_seed(M * 7 + K * 3 + N)
    x = h16(torch.randn(M, K, generator=g))
    w = h16(torch.randn(K, N, generator=g) / math.sqrt(K))
    b = h16(torch.randn(N, generator=g) * 0.1)
    res = torch.randn(M, N, generator=g)
    ref = x.float() @ w.float() + b.float() + res
    out = ctx.linear(x, w, b, residual=res)
    assert rel_err(out, ref) < 2e-6
    out16 = ctx.linear(x, w, None, out_f16=True)
    assert rel_err(out16, x.float() @ w.float()) < 6e-4  # one f16 output rounding


@pytest.mark.parametrize("M,C", [(256, 128), (1024, 640), (384, 1280), (130, 64)])
def test_geglu(ctx, M, C):
    g = torch.Generator().manual_seed(M + C)
    x = h16(torch.randn(M, C, generator=g))
    w = h16(torch.randn(C, 8 * C, generator=g) / math.sqrt(C))
    b = h16(torch.randn(8 * C, generator=g) * 0.1)
    wd = {"p/proj/weight": w.float(), "p/proj/bias": b.float()}
    ref = O.geglu(x.float(), wd, "p")
    out = ctx.linear(x, w, b, geglu=True)
    assert out.shape == (M, 4 * C)
    assert rel_err(out, ref) < 6e-4  # f16 output


@pytest.mark.parametrize("B,H,W,Cin,Cout,ks,stride,up", [
    (1, 16, 16, 64, 64, 3, 1, False), (2, 32, 32, 320, 640, 3, 1, False), (2, 8, 8, 128, 256, 3, 1, False),
    (1, 64, 64, 64, 128, 1, 1, False), (2, 32, 32, 320, 320, 3, 2, False), (1, 16, 16, 128, 128, 3, 2, False),
    (2, 16, 16, 256, 256, 3, 1, True), (1, 4, 4, 64, 64, 3, 1, False), (3, 8, 8, 64, 64, 3, 2, False),
    (1, 128, 128, 320, 4, 3, 1, False), (1, 20, 24, 72, 80, 3, 1, False), (1, 128, 128, 64, 64, 3, 1, False)])
def test_conv2d(ctx, B, H, W, Cin, Cout, ks, stride, up):
    g = torch.Generator().manual_seed(B + H + Cin + Cout + ks + stride)
    x = h16(torch.randn(B, Cin, H, W, generator=g)).float()  # values exactly representable in f16
    w = h16(torch.randn(Cout, Cin, ks, ks, generator=g) / math.sqrt(Cin * ks * ks))
    b = h16(torch.randn(Cout, generator=g) * 0.1)
    xin = x
    if up:
        xin = torch.nn.functional.interpolate(x, scale_factor=2, mode="nearest")
    ref = torch.nn.functional.conv2d(xin, w.float(), b.float(), stride=stride, padding=ks // 2)
    out = ctx.conv2d(x.permute(0, 2, 3, 1).contiguous(), w, b, stride=stride, upsample=up)
    assert rel_err(out.permute(0, 3, 1, 2), ref) < 1e-5  # f32 accumulation order only (K up to 2880)


@pytest.mark.parametrize("B,HW,C1,C2,silu", [(2, 1024, 320, 0, True), (1, 4096, 640, 320, True), (2, 256, 1280, 1280, False),
                                             (1, 16384, 320, 0, True), (3, 64, 64, 64, True), (1, 16, 64, 0, False)])
def test_group_norm(ctx, B, HW, C1, C2, silu):
    g = torch.Generator().manual_seed(HW + C1 + C2)
    x1 = torch.randn(B, HW, C1, generator=g) * 1.5 + 0.3
    x2 = torch.randn(B, HW, C2, generator=g) * 0.7 - 0.2 if C2 else None
    C = C1 + C2
    gamma = 1 + 0.1 * torch.randn(C, generator=g)
    beta = 0.1 * torch.randn(C, generator=g)
    xc = x1 if x2 is None else torch.cat([x1, x2], dim=2)
    nchw = xc.permute(0, 2, 1).reshape(B, C, HW, 1)
    ref = O.group_norm(nchw, gamma, beta)
    if silu:
        ref = O.silu(ref)
    ref = ref.reshape(B, C, HW).permute(0, 2, 1)
    out = ctx.group_norm(x1, x2, gamma, beta, silu=silu)
    assert rel_err(out, ref) < 5e-4  # f16 output rounding (2^-11 relative per element)


@pytest.mark.parametrize("B,HW,C,mean,std", [(1, 16384, 320, 50.0, 0.1), (2, 4096, 640, -200.0, 0.5), (1, 1024, 1280, 1000.0, 1.0)])
def test_group_norm_large_mean(ctx, B, HW, C, mean, std):
    """|mean| / sigma up to 1000 (real SDXL activations have groups like this): the variance must come from centred sums
    (reference groupnorm/mod.rs:75-82 centres first), not from E[x^2] - mean^2 in f32."""
    g = torch.Generator().manual_seed(HW + C)
    x = torch.randn(B, HW, C, generator=g) * std + mean
    x += torch.linspace(-3 * std, 3 * std, C)[None, None, :]     # per-channel offsets inside a group
    gamma = 1 + 0.1 * torch.randn(C, generator=g)
    beta = 0.1 * torch.randn(C, generator=g)
    ref = O.group_norm(x.double().permute(0, 2, 1).reshape(B, C, HW, 1), gamma.double(), beta.double()).reshape(B, C, HW).permute(0, 2, 1)
    out = ctx.group_norm(x, None, gamma, beta, silu=False)
    e = rel_err(out, ref)
    print(f"group_norm mean {mean} std {std}: rel err {e:.3e}")
    assert e < 1e-3   # f32 input quantisation of (x - mean) alone is ~|mean| 2^-24 / std


@pytest.mark.parametrize("rows,C", [(1024, 1280), (4096, 640), (100, 128), (33, 256), (7, 64)])
def test_layer_norm(ctx, rows, C):
    g = torch.Generator().manual_seed(rows + C)
    x = torch.randn(rows, C, generator=g) * 2 + 0.5
    gamma = 1 + 0.1 * torch.randn(C, generator=g)
    beta = 0.1 * torch.randn(C, generator=g)
    ref = O.layer_norm(x, gamma, beta)
    out = ctx.layer_norm(x, gamma, beta)
    assert rel_err(out, ref) < 5e-4


@pytest.mark.parametrize("B,T,S,nh", [(1, 256, 256, 2), (2, 1024, 1024, 4), (2, 1024, 77, 20), (1, 4096, 77, 10),
                                      (1, 64, 64, 1), (2, 16, 3, 4), (1, 200, 333, 2), (1, 4096, 4096, 2)])
def test_qkv_attention(ctx, B, T, S, nh):
    g = torch.Generator().manual_seed(T + S + nh)
    C = nh * 64
    q = h16(torch.randn(B, T, C, generator=g))
    k = h16(torch.randn(B, S, C, generator=g))
    v = h16(torch.randn(B, S, C, generator=g))
    ref = O.qkv_attention(q.float(), k.float(), v.float(), None, nh)
    out = ctx.qkv_attention(q, k, v, None, nh)
    # P is rounded to f16 before the PV contraction and the output is f16: ~2^-11 relative each
    e = rel_err(out, ref)
    print(f"attention B={B} T={T} S={S} heads={nh}: rel err {e:.3e}")
    assert e < 1.0e-3
    assert torch.isfinite(out).all()


@pytest.mark.parametrize("scale", [1.5, 3.0, 6.0])
def test_qkv_attention_large_dynamic_range(ctx, scale):
    """Scores whose row maximum grows between 128-key blocks (keys 300 and up are doubled, so the third block takes over):
    score spreads of a few units (scale 1.5), tens (3.0) and hundreds (6.0). The kernel keeps the exact running maximum of
    every key block and rescales the row's O and l registers by exp(m_old - m_new) when it grows — at scale 6 that factor
    underflows to 0 and the earlier blocks drop out — so every probability is <= 1 before its f16 rounding."""
    g = torch.Generator().manual_seed(int(scale * 10))
    B, T, S, nh = 1, 256, 640, 2
    q = h16(torch.randn(B, T, nh * 64, generator=g) * scale)
    k = h16(torch.randn(B, S, nh * 64, generator=g) * scale)
    k[:, 300:] *= 2.0  # later key blocks dominate
    v = h16(torch.randn(B, S, nh * 64, generator=g))
    ref = O.qkv_attention(q.float(), k.float(), v.float(), None, nh)
    out = ctx.qkv_attention(q, k, v, None, nh)
    assert torch.isfinite(out).all()
    e = rel_err(out, ref)
    print(f"attention dynamic range scale {scale}: rel err {e:.3e}")
    assert e < 2e-3


def test_qkv_attention_mask_shape_is_checked(ctx):
    from sdxl_b200 import SdxlError
    q = torch.zeros(1, 8, 64, dtype=torch.float16)
    with pytest.raises(SdxlError):
        ctx.qkv_attention(q, q, q, torch.zeros(4, 8), 1)
    # an all-zero additive mask is the unmasked result (short-sequence kernel vs tensor-core kernel)
    g = torch.Generator().manual_seed(0)
    q, k, v = (torch.randn(2, 40, 128, generator=g).half() for _ in range(3))
    a = ctx.qkv_attention(q, k, v, torch.zeros(40, 40), 2)
    b = ctx.qkv_attention(q, k, v, None, 2)
    assert rel_err(a, b) < 2e-3


def test_timestep_embedding(ctx):
    ts = [0, 1, 249, 499, 749, 999]
    for dim in (320, 256, 64):
        out = ctx.timestep_embedding(ts, dim)
        ref = O.timestep_embedding(torch.tensor(ts), dim)
        assert (out.cpu() - ref).abs().max() < 2e-4  # f32 sin/cos of arguments up to 999 rad


def test_randn_matches_philox_oracle(ctx):
    n = 4 * 4 * 128 * 128 + 3
    out = ctx.randn(n, seed=0x1234_5678_9ABC, subsequence=7).cpu().numpy()
    ref = philox.randn(n, 0x1234_5678_9ABC, 7)
    assert np.abs(out - ref).max() < 1e-4  # identical integer stream; f32 log/sin/cos differ by ulps
    assert abs(out.mean()) < 0.01 and abs(out.std() - 1) < 0.01
