"""GPU parity of the implicit GEMM's LINEAR epilogue, which loads the bias and residual of 8 or 10 column pairs before their adds.

The cases cover every tile width with a residual (64, 128, 160 and 256), a partial last N tile (some chunks masked part-way), an
odd N (unaligned rows: the scalar load path), a persistent loop with several tiles per CTA, the GEGLU epilogue at level-2 size
and a level-1 3x3 convolution. Tolerances as in test_ops_gpu.py: f16 operands pre-rounded, f32 accumulation, so only the
summation order differs.
"""
import math

import pytest
import torch

from oracle import unet_oracle as O
from harness import rel_err

pytestmark = pytest.mark.gpu


def h16(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.float16)


# 384 x 1280: 3 M tiles; 8192 x 1280: 512 tiles, several per CTA; 2048 x 3840: BN 256; 4096 x 640: BN 160 at level 1;
# 1024 x 1000: no tile width divides N, last tile partial; 512 x 333: odd N; 256 x 128 / 64: BN 128 and 64.
@pytest.mark.parametrize("M,K,N", [(384, 1280, 1280), (8192, 1280, 1280), (2048, 1280, 3840), (4096, 640, 640),
                                   (1024, 320, 1000), (512, 320, 333), (256, 640, 128), (256, 640, 64)])
def test_linear_residual_epilogue(ctx, M, K, N):
    g = torch.Generator().manual_seed(M + K + N)
    x = h16(torch.randn(M, K, generator=g))
    w = h16(torch.randn(K, N, generator=g) / math.sqrt(K))
    b = h16(torch.randn(N, generator=g) * 0.1)
    res = torch.randn(M, N, generator=g)
    ref = x.float() @ w.float() + b.float() + res
    out = ctx.linear(x, w, b, residual=res)
    assert rel_err(out, ref) < 2e-6  # f32 accumulation order; both sides sum K products in f32
    out_nb = ctx.linear(x, w, None, residual=res)
    assert rel_err(out_nb, x.float() @ w.float() + res) < 2e-6
    out16 = ctx.linear(x, w, None, out_f16=True)
    assert rel_err(out16, x.float() @ w.float()) < 6e-4  # one f16 output rounding


def test_geglu_level2(ctx):
    M, C = 2048, 1280
    g = torch.Generator().manual_seed(M + C)
    x = h16(torch.randn(M, C, generator=g))
    w = h16(torch.randn(C, 8 * C, generator=g) / math.sqrt(C))
    b = h16(torch.randn(8 * C, generator=g) * 0.1)
    wd = {"p/proj/weight": w.float(), "p/proj/bias": b.float()}
    ref = O.geglu(x.float(), wd, "p")
    out = ctx.linear(x, w, b, geglu=True)
    assert out.shape == (M, 4 * C)
    assert rel_err(out, ref) < 6e-4  # f16 output


def test_conv2d_level1(ctx):
    B, H, W, C = 1, 64, 64, 640
    g = torch.Generator().manual_seed(640)
    x = h16(torch.randn(B, C, H, W, generator=g)).float()
    w = h16(torch.randn(C, C, 3, 3, generator=g) / math.sqrt(C * 9))
    b = h16(torch.randn(C, generator=g) * 0.1)
    ref = torch.nn.functional.conv2d(x, w.float(), b.float(), padding=1)
    out = ctx.conv2d(x.permute(0, 2, 3, 1).contiguous(), w, b)
    assert rel_err(out.permute(0, 3, 1, 2), ref) < 1e-5  # f32 accumulation order only (K = 5760)
