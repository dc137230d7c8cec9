"""GPU parity of the GEMM shapes that run on the 128 x 160 tile (the UNet's 320 * 2^k channel widths).

At 132 SMs the tile picker gives these shapes BN = 160: a Linear at 16 M tiles with N = 1280 (level-2 attention out / proj with
the f32 residual), the same with M not a multiple of 128 (masked last M tile), and the level-0 3x3 conv 320 -> 320 at 128 x 128.
Tolerances as in test_ops_gpu.py: f16 operands pre-rounded, f32 accumulation, so only the summation order differs.
"""
import math

import pytest
import torch
from harness import rel_err

pytestmark = pytest.mark.gpu


def h16(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.float16)


@pytest.mark.parametrize("M,K,N", [(2048, 1280, 1280), (2000, 1280, 1280), (2048, 5120, 1280)])
def test_linear_n160_tile(ctx, M, K, N):
    g = torch.Generator().manual_seed(M + K + N)
    x = h16(torch.randn(M, K, generator=g))
    w = h16(torch.randn(K, N, generator=g) / math.sqrt(K))
    b = h16(torch.randn(N, generator=g) * 0.1)
    res = torch.randn(M, N, generator=g)
    ref = x.float() @ w.float() + b.float() + res
    out = ctx.linear(x, w, b, residual=res)
    assert rel_err(out, ref) < (2e-6 if K <= 2048 else 1e-5)  # f32 accumulation order; both sides sum K products in f32
    out16 = ctx.linear(x, w, None, out_f16=True)
    assert rel_err(out16, x.float() @ w.float()) < 6e-4  # one f16 output rounding


def test_conv2d_n160_tile(ctx):
    B, H, W, C = 1, 128, 128, 320
    g = torch.Generator().manual_seed(320)
    x = h16(torch.randn(B, C, H, W, generator=g)).float()
    w = h16(torch.randn(C, C, 3, 3, generator=g) / math.sqrt(C * 9))
    b = h16(torch.randn(C, generator=g) * 0.1)
    ref = torch.nn.functional.conv2d(x, w.float(), b.float(), padding=1)
    out = ctx.conv2d(x.permute(0, 2, 3, 1).contiguous(), w, b)
    assert rel_err(out.permute(0, 3, 1, 2), ref) < 1e-5  # f32 accumulation order only (K = 2880)
