"""Every implicit-GEMM form of the UNet launch plan, bit for bit on exactly representable operands; GEGLU and the hi/lo head conv
against float64.

PlanBuilder / UNetPlanBuilder (engine_core.h, engine.cu) give igemm_kernel one parameter set per call site: 3x3 convs with a
per-batch bias row, a fused 1x1 skip segment on a second source or an f32 residual, the stride-2 Downsample on a phase-split
input, the upsample conv as four scattered phase convolutions, Linears with f16 or f32 outputs, residuals added in place
(out == res) or into an f16 output, GEGLU, and the 18-segment head conv on GroupNorm's hi / lo split. Each test below builds
its form as the named call site does (repack_conv / repack_upconv / transpose_linear weights, bias_to_f32 biases) at the
plan's real extents: the 128 x 128 latent at B = 2 and the 1216 x 832 bucket (152 x 104) at B = 3 with their lower levels,
small odd images, base widths 320 / 640 / 1280 and refiner widths 384 / 768 / 1536.

Exact arithmetic. Activations are i 2^-3 and weights j 2^-6 with integers |i|, |j| <= 8 (exact in f16), so every product is a
multiple of 2^-9; biases and residuals are f32 multiples of 2^-9 of magnitude <= 2^11 (f16 biases: <= 2047 * 2^-9). Each test
asserts from its operands that sum |x w| + |bias| + |res| < 2^22 * 2^-9: every partial sum is then an integer multiple of
2^-9 below 2^22 of them, exact in f32 whatever the summation order. So an f32 output must equal the exact value and an f16
output its round-to-nearest-even rounding (ties are frequent on this grid), with zero tolerance: a dropped or doubled tap at an
image border, a wrong bias row, a residual added twice or a truncating f16 store all fail. The reference is float64 on the
GPU, one matmul per tap over shifted views of the input (no cuDNN algorithm choice), itself exact in any order. Outputs are
pre-filled with NaN and followed by a NaN guard region that must stay untouched.

GEGLU's gate and the head conv's GroupNorm input are not on a grid: they are bounded elementwise against float64.
"""
import math

import pytest
import torch

from sdxl_b200 import _testing as T
from harness import (DEV, GEGLU, GRID_B, H11, H_SUB, assert_exact, assert_exact_range, bias_f32, check, conv_bound, conv_ref,
                     conv_taps, gen, gn_ref, grid, grid_f32, grid_w, grid_x, guarded, in_place_residual, lin_weights, linear, pad64,
                     plan_upconv, repack3, stride2_taps)

pytestmark = pytest.mark.gpu

U23 = 2.0 ** -23
GEGLU_BN = 256                    # engine.cu geglu_bn_for(4C): 4C is a multiple of 128 at every UNet width
# erf_as (common.cuh): Abramowitz-Stegun 7.1.26 (1.5e-7 absolute) evaluated in f32 with rcp.approx / ex2.approx
E_GELU = 5e-7
HEAD_LO_TOL = 5.5e-5              # normwise error of the hi / lo head conv (test_head_conv_hi_lo)


# ------------------------------------------------------------------------------------------------------------------------------
# convolution forms
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,Cin,Cout", [
    (2, 128, 128, 320, 320), (3, 152, 104, 640, 320), (2, 64, 64, 320, 640), (3, 76, 52, 1280, 640), (2, 32, 32, 2560, 1280),
    (3, 38, 26, 2560, 1280), (3, 5, 7, 960, 320), (3, 12, 12, 1920, 640),
    (2, 32, 32, 3072, 1536),    # the refiner's widest conv_in: K = 9 * 3072 over a concatenated skip
])
def test_resblock_conv_in(ctx, B, H, W, Cin, Cout):
    """UNetPlanBuilder::resblock -> conv3(conv_in): 9 taps; the time embedding folded into a per-batch bias row
    temb_all[b, temb_off:temb_off + Cout] (bias_bstride = temb_total)."""
    g = gen(B, H, W, Cin, Cout)
    x = grid_x(g, B, H, W, Cin)
    w = grid_w(g, Cout, Cin, 3, 3)
    temb_off, temb_total = 640, 640 + Cout + 320
    temb_all = grid_f32(g, B, temb_total)
    Ktot = 9 * pad64(Cin)
    wt = repack3(w, Ktot)
    out, guard = guarded((B, H, W, Cout))
    assert_exact_range("conv_in", conv_bound(x, w), temb_all.abs().max())
    T.igemm(x, (B, H, W, Cin), wt, Cout, Ktot, (W, H, B), conv_taps(pad64(Cin) // 64), out, Cout,
            bias=temb_all.view(-1)[temb_off:], bias_bstride=temb_total)
    ref = conv_ref(x, w) + temb_all[:, temb_off:temb_off + Cout].double()[:, None, None, :]
    assert_exact(out, ref, guard, f"resblock conv_in {B}x{H}x{W} {Cin}->{Cout}")


@pytest.mark.parametrize("B,H,W,C1,C2,Cout", [
    (2, 64, 64, 320, 0, 640), (2, 32, 32, 640, 0, 1280), (2, 128, 128, 320, 320, 320), (3, 152, 104, 640, 320, 320),
    (3, 76, 52, 1280, 640, 640), (3, 38, 26, 1280, 1280, 1280), (3, 5, 7, 640, 320, 320), (3, 12, 12, 1280, 640, 640),
    (2, 32, 32, 1536, 1536, 1536),
])
def test_resblock_conv_out_skip(ctx, B, H, W, C1, C2, Cout):
    """UNetPlanBuilder::resblock with has_skip -> conv3(conv_out, skip): 9 taps on a0 (the second GroupNorm's output) and one 1x1
    segment on a1 = raw, the first GroupNorm's f16(cat(x1, x2)); weights [Cout, 9 Ipad | I2pad], bias = conv bias + skip bias
    (bias_to_f32, then bias_to_f32 accumulate)."""
    g = gen(B, H, W, C1, C2, Cout)
    Cin, HW = C1 + C2, H * W
    x1 = grid_x(g, B, HW, C1).float()
    x2 = grid_x(g, B, HW, C2).float() if C2 else None
    gam = torch.ones(Cin, device=DEV)
    bet = torch.zeros(Cin, device=DEV)
    y = torch.empty(B, HW, Cin, dtype=torch.float16, device=DEV)
    raw = torch.full_like(y, float("nan"))
    T.group_norm(x1, x2, B, HW, 32, gam, bet, 1e-5, True, y, raw, None, T.gn_scratch(B, 32))
    xc = x1 if x2 is None else torch.cat([x1, x2], dim=2)
    assert torch.equal(raw.float(), xc), "GroupNorm raw output of grid inputs must be exact"
    a0 = grid_x(g, B, H, W, Cout)
    w3 = grid_w(g, Cout, Cout, 3, 3)
    ws = grid_w(g, Cout, Cin, 1, 1)
    b3, bias = bias_f32(g, Cout)
    bs = grid(g, (Cout,), GRID_B, 2047)
    T.bias_to_f32(bs, Cout, bias, accumulate=True)
    Ipad, I2pad = pad64(Cout), pad64(Cin)
    Ktot = 9 * Ipad + I2pad
    wt = repack3(w3, Ktot)
    repack3(ws, Ktot, wt, 9 * Ipad)
    out, guard = guarded((B, H, W, Cout))
    assert_exact_range("conv_out + skip", conv_bound(a0, w3), conv_bound(raw, ws), b3.abs().max(), bs.abs().max())
    segs = conv_taps(Ipad // 64) + [(1, 0, 0, 0, I2pad // 64)]
    T.igemm(a0, (B, H, W, Cout), wt, Cout, Ktot, (W, H, B), segs, out, Cout, a1=raw, a1_shape=(B, H, W, Cin), bias=bias)
    ref = conv_ref(a0, w3) + conv_ref(raw.view(B, H, W, Cin), ws) + b3.double() + bs.double()
    assert_exact(out, ref, guard, f"resblock conv_out + skip {B}x{H}x{W} {C1}+{C2}->{Cout}")


@pytest.mark.parametrize("B,H,W,C", [(2, 128, 128, 320), (3, 152, 104, 320), (2, 64, 64, 640), (3, 38, 26, 1280),
                                     (3, 5, 7, 1280), (3, 12, 12, 640), (2, 16, 16, 1536)])
def test_resblock_conv_out_identity(ctx, B, H, W, C):
    """UNetPlanBuilder::resblock without a skip conv -> conv3(conv_out, res = xa): the block input, a separate f32 buffer,
    added in the epilogue (ldr = ldo = C)."""
    g = gen(B, H, W, C, 1)
    a0 = grid_x(g, B, H, W, C)
    w = grid_w(g, C, C, 3, 3)
    b16, b32 = bias_f32(g, C)
    res = grid_f32(g, B, H, W, C)
    Ktot = 9 * pad64(C)
    wt = repack3(w, Ktot)
    out, guard = guarded((B, H, W, C))
    assert_exact_range("conv_out + identity", conv_bound(a0, w), b16.abs().max(), res.abs().max())
    T.igemm(a0, (B, H, W, C), wt, C, Ktot, (W, H, B), conv_taps(pad64(C) // 64), out, C, bias=b32, res=res, ldr=C)
    assert_exact(out, conv_ref(a0, w) + b16.double() + res.double(), guard, f"resblock conv_out + identity {B}x{H}x{W}x{C}")


@pytest.mark.parametrize("B,H,W,C", [(2, 128, 128, 320), (3, 152, 104, 320), (2, 64, 64, 640), (3, 76, 52, 640),
                                     (3, 12, 12, 320), (2, 128, 128, 384), (2, 32, 32, 1536)])
def test_downsample(ctx, B, H, W, C):
    """UNetPlanBuilder encoder, BT_DOWN: phase_split of the f32 input into [4 B, H/2, W/2, C] f16, then the 3x3 stride-2
    conv as 9 segments with batch offsets db = phase * B (stride2_taps)."""
    g = gen(B, H, W, C, 2)
    x = grid_x(g, B, H, W, C).float()
    w = grid_w(g, C, C, 3, 3)
    b16, b32 = bias_f32(g, C)
    ph = torch.empty(4 * B, H // 2, W // 2, C, dtype=torch.float16, device=DEV)
    T.phase_split(x, B, H, W, C, ph)
    Ktot = 9 * pad64(C)
    wt = repack3(w, Ktot)
    H2, W2 = H // 2, W // 2
    out, guard = guarded((B, H2, W2, C))
    assert_exact_range("downsample", conv_bound(x, w), b16.abs().max())
    T.igemm(ph, (4 * B, H2, W2, C), wt, C, Ktot, (W2, H2, B), stride2_taps(B, pad64(C) // 64), out, C, bias=b32)
    assert_exact(out, conv_ref(x, w, stride=2) + b16.double(), guard, f"downsample {B}x{H}x{W}x{C}")


@pytest.mark.parametrize("B,H,W,C", [(2, 32, 32, 1280), (2, 64, 64, 640), (3, 38, 26, 1280), (3, 76, 52, 640),
                                     (3, 5, 7, 640), (2, 16, 16, 1536), (2, 64, 64, 768)])
def test_upsample_conv(ctx, B, H, W, C):
    """PlanBuilder::upconv: repack_upconv's four 2x2 phase kernels (sums of up to four grid taps, exact in f16) and one launch per
    output parity through opix. On this grid each phase convolution is an exact sum, so the result equals nearest-2x upsample
    then the 3x3 conv of the original weights, bit for bit."""
    g = gen(B, H, W, C, 3)
    x = grid_x(g, B, H, W, C)
    w = grid_w(g, C, C, 3, 3)
    b16, b32 = bias_f32(g, C)
    assert_exact_range("upsample conv", conv_bound(x, w), b16.abs().max())
    out, _ = plan_upconv(x, w, b32)      # NaN-filled, every pixel written by one of the four parity launches
    up = x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    assert_exact(out, conv_ref(up, w) + b16.double(), None, f"upsample conv {B}x{H}x{W}x{C}")


# ------------------------------------------------------------------------------------------------------------------------------
# Linear forms (SpatialTransformer, hoisted conditioning, ControlNet zero convs)
# ------------------------------------------------------------------------------------------------------------------------------
# M = B * H * W of a transformer level: 64^2 / 32^2 at B = 2, 76 x 52 / 38 x 26 at B = 3, small odd images, refiner widths
LIN_SHAPES = [(8192, 640), (2048, 1280), (11856, 640), (2964, 1280), (105, 640), (432, 1280), (8192, 768), (2048, 1536)]


@pytest.mark.parametrize("M,C", LIN_SHAPES)
def test_strans_qkv_and_q2(ctx, M, C):
    """UNetPlanBuilder::strans: the fused self-attention QKV (three transpose_linear slices at rows 0, C, 2C of one [3C, Cpad]
    matrix, load_st) and the cross-attention query q2: f16 outputs, no bias."""
    g = gen(M, C, 4)
    x = grid_x(g, M, C)
    wqkv = torch.empty(3 * C * pad64(C), dtype=torch.float16, device=DEV)
    ws = [lin_weights(g, C, C, wt=wqkv, row0=r * C)[0] for r in range(3)]
    w = torch.cat(ws, dim=1)
    out, guard = guarded((M, 3 * C), torch.float16)
    assert_exact_range("qkv", conv_bound(x, w.t()))
    linear(x, wqkv, 3 * C, pad64(C), out, 3 * C)
    assert_exact(out, x.double() @ w.double(), guard, f"strans qkv M={M} C={C} (f16)")
    wq, wqt = lin_weights(g, C, C)
    out, guard = guarded((M, C), torch.float16)
    linear(x, wqt, C, pad64(C), out, C)
    assert_exact(out, x.double() @ wq.double(), guard, f"strans q2 M={M} C={C} (f16)")


@pytest.mark.parametrize("B,K,C", [(2, 2048, 640), (2, 2048, 1280), (3, 2048, 640), (3, 2048, 1280), (2, 1280, 768),
                                   (3, 1280, 1536)])
def test_hoisted_cross_kv(ctx, B, K, C):
    """set_conditioning -> project_kv: every transformer block's cross-attention K / V of the context, one Linear per block
    hoisted out of the step. The [2C, Kpad] matrix is two transpose_linear slices (load_st); f16 output, M = B * 77 (a partial
    M tile); K = 2048 for the base context, 1280 for the refiner's."""
    g = gen(B, K, C, 5)
    M = B * 77
    x = grid_x(g, M, K)
    wkv = torch.empty(2 * C * pad64(K), dtype=torch.float16, device=DEV)
    w = torch.cat([lin_weights(g, K, C, wt=wkv, row0=r * C)[0] for r in range(2)], dim=1)
    out, guard = guarded((M, 2 * C), torch.float16)
    assert_exact_range("hoisted K/V", conv_bound(x, w.t()))
    linear(x, wkv, 2 * C, pad64(K), out, 2 * C)
    assert_exact(out, x.double() @ w.double(), guard, f"hoisted cross K/V B={B} K={K} C={C} (f16)")


@pytest.mark.parametrize("M,C", LIN_SHAPES)
def test_strans_proj_in_proj_out(ctx, M, C):
    """UNetPlanBuilder::strans: proj_in (f32 out + bias into s_tok) and proj_out (f32 out + bias + the block input x, a separate
    residual buffer)."""
    g = gen(M, C, 6)
    x = grid_x(g, M, C)
    for name, res in (("proj_in", None), ("proj_out", grid_f32(g, M, C))):
        w, wt = lin_weights(g, C, C)
        b16, b32 = bias_f32(g, C)
        out, guard = guarded((M, C))
        assert_exact_range(name, conv_bound(x, w.t()), b16.abs().max(), 0 if res is None else res.abs().max())
        linear(x, wt, C, pad64(C), out, C, bias=b32, res=res)
        ref = x.double() @ w.double() + b16.double() + (0 if res is None else res.double())
        assert_exact(out, ref, guard, f"strans {name} M={M} C={C}")


@pytest.mark.parametrize("M,C", LIN_SHAPES)
def test_strans_in_place_residual(ctx, M, C):
    """UNetPlanBuilder::strans: attn1 out, attn2 out (K = C) and ff2 (K = 4C) of every block but the last add into s_tok in
    place: f32 out + bias with out and res the same tensor."""
    g = gen(M, C, 7)
    for name, K in (("out1", C), ("out2", C), ("ff2", 4 * C)):
        x = grid_x(g, M, K)
        w, wt = lin_weights(g, K, C)
        b16, b32 = bias_f32(g, C)
        in_place_residual(g, x, w, wt, b16, b32, f"strans {name} in place M={M} C={C}")


@pytest.mark.parametrize("B,H,W,C", [(2, 128, 128, 320), (3, 152, 104, 320), (2, 64, 64, 640), (3, 38, 26, 1280),
                                     (3, 5, 7, 320)])
def test_controlnet_zero_conv_in_place(ctx, B, H, W, C):
    """UNetPlanBuilder::zero_conv: skip += zero_conv(h), a 1x1 conv (repack_conv, Loader::conv with ks = 1) run as a Linear over
    the B * H * W pixels of the cast ControlNet feature, adding onto the UNet's saved skip in place."""
    g = gen(B, H, W, C, 8)
    M = B * H * W
    x = grid_x(g, M, C)
    wc = grid_w(g, C, C, 1, 1)
    wt = repack3(wc, pad64(C))
    b16, b32 = bias_f32(g, C)
    in_place_residual(g, x, wc.view(C, C).t(), wt, b16, b32, f"zero conv in place {B}x{H}x{W}x{C}")


@pytest.mark.parametrize("M,C", LIN_SHAPES)
def test_strans_last_ff2_f16_out(ctx, M, C):
    """UNetPlanBuilder::strans, last block: ff2's residual add writes the f16 operand of proj_out directly: f16 out (s_a16) +
    bias + f32 residual (s_tok), K = 4C."""
    g = gen(M, C, 9)
    x = grid_x(g, M, 4 * C)
    w, wt = lin_weights(g, 4 * C, C)
    b16, b32 = bias_f32(g, C)
    res = grid_f32(g, M, C)
    out, guard = guarded((M, C), torch.float16)
    assert_exact_range("last ff2", conv_bound(x, w.t()), b16.abs().max(), res.abs().max())
    linear(x, wt, C, pad64(4 * C), out, C, bias=b32, res=res)
    assert_exact(out, x.double() @ w.double() + b16.double() + res.double(), guard, f"strans last ff2 M={M} C={C} (f16 + f32 res)")


@pytest.mark.parametrize("M", [2964, 105])
def test_odd_n_scalar_store(ctx, M):
    """N = 333 (no call site; odd row pitches take the epilogue's scalar load / store path): f32 out + bias + residual, in place
    and separate, and f16 out."""
    g = gen(M, 333)
    N, K = 333, 320
    x = grid_x(g, M, K)
    w, wt = lin_weights(g, K, N)
    b16, b32 = bias_f32(g, N)
    in_place_residual(g, x, w, wt, b16, b32, f"odd N={N} M={M} f32 in place")
    out, guard = guarded((M, N), torch.float16)
    linear(x, wt, N, pad64(K), out, N, bias=b32)
    assert_exact(out, x.double() @ w.double() + b16.double(), guard, f"odd N={N} M={M} (f16)")


# ------------------------------------------------------------------------------------------------------------------------------
# GEGLU
# ------------------------------------------------------------------------------------------------------------------------------
def gelu64(x: torch.Tensor) -> torch.Tensor:
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def geglu_bound(ref, v, gate):
    """f16 output rounding, plus erf_as's absolute error E_GELU passed through value * 0.5 gate."""
    return H11 * ref.abs() + H_SUB + 0.5 * gate.abs() * v.abs() * E_GELU


def test_geglu_every_f16_gate(ctx):
    """UNetPlanBuilder::strans ff1 (IGEMM_GEGLU, geglu_bn = 256) over all 63,488 finite f16 gate values: one-hot A rows pick a
    weight row whose value columns are 1 and whose gate columns are every f16 value (row 1: in reverse order), laid out by
    transpose_linear's GEGLU permutation, so value and gate reach the epilogue exactly. Where erf rounds to 1 in f32 (g >= 6)
    the output must be exactly f16(g)."""
    gates = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.float16)
    gates = gates[torch.isfinite(gates)].to(DEV)
    G = gates.numel()
    assert G == 63488
    N, K = 2 * G, 64
    assert G % (GEGLU_BN // 2) == 0
    w = torch.zeros(K, N, dtype=torch.float16, device=DEV)
    w[0, :G], w[0, G:] = 1.0, gates
    w[1, :G], w[1, G:] = 1.0, gates.flip(0)
    wt = torch.empty(N * K, dtype=torch.float16, device=DEV)
    T.transpose_linear(w, K, N, wt, K, 0, GEGLU_BN)
    x = torch.zeros(2, K, dtype=torch.float16, device=DEV)
    x[0, 0] = x[1, 1] = 1.0
    out, guard = guarded((2, G), torch.float16)
    linear(x, wt, N, K, out, G, mode=GEGLU, geglu_bn=GEGLU_BN)
    gg = torch.stack([gates, gates.flip(0)]).double()
    ref = gelu64(gg)
    nz = gg != 0
    beyond = ((out.double() - ref).abs() - H11 * ref.abs() - H_SUB).clamp_min(0)   # what the f16 rounding does not explain
    worst = float((beyond[nz] / (0.5 * gg[nz].abs())).max())
    print(f"GEGLU gate sweep: worst error beyond the f16 rounding / (0.5 |g|) = {worst:.3e} (E = {E_GELU:.1e})")
    check(out, ref, geglu_bound(ref, torch.ones_like(gg), gg), "GEGLU every f16 gate")
    big = gg >= 6
    assert torch.equal(out[big], gg[big].half()), "GEGLU: gelu(g) must be exactly g where erf(g / sqrt 2) rounds to 1"
    assert bool(guard.isnan().all()), "GEGLU gate sweep: elements after the output were written"


@pytest.mark.parametrize("C", [320, 640, 1280, 384, 768, 1536])
@pytest.mark.parametrize("M", [2048, 2964, 8192])
def test_geglu_plan_widths(ctx, M, C):
    """UNetPlanBuilder::strans ff1 at the UNet's widths: [C, 8C] weights and bias in the geglu_bn layout (transpose_linear,
    bias_to_f32), grid operands so that value and gate are exact; out f16 [M, 4C] = value * gelu(gate)."""
    assert (4 * C) % (GEGLU_BN // 2) == 0
    g = gen(M, C, 10)
    x = grid_x(g, M, C)
    w, wt = lin_weights(g, C, 8 * C, GEGLU_BN)
    b16, b32 = bias_f32(g, 8 * C, GEGLU_BN)
    assert_exact_range("geglu", conv_bound(x, w.t()), b16.abs().max())
    out, guard = guarded((M, 4 * C), torch.float16)
    linear(x, wt, 8 * C, pad64(C), out, 4 * C, bias=b32, mode=GEGLU, geglu_bn=GEGLU_BN)
    z = x.double() @ w.double() + b16.double()
    v, gate = z[:, :4 * C], z[:, 4 * C:]
    ref = v * gelu64(gate)
    check(out, ref, geglu_bound(ref, v, gate), f"GEGLU M={M} C={C}")
    assert bool(guard.isnan().all()), f"GEGLU M={M} C={C}: elements after the output were written"


# ------------------------------------------------------------------------------------------------------------------------------
# the head conv on GroupNorm's hi / lo split
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,C", [(2, 128, 128, 320), (3, 152, 104, 320), (2, 128, 128, 384)])
def test_head_conv_hi_lo(ctx, B, H, W, C):
    """UNetPlanBuilder head (norm_out + conv_out): GroupNorm + SiLU at G = 32 writes y = f16(t) and y_lo = f16(t - y); the conv
    runs 18 segments, 9 taps on y (map 0) and 9 on y_lo (map 1), over weights [W | W] with row pitch 2 Ktot (conv_out_w2),
    N = 4, ldo = 4. Elementwise: f32 accumulation of 18 Ipad products plus the operand error conv(|W|, e32 + 2^-22 |t| +
    2^-25) of y + y_lo. Normwise, the lo half must reach the result: the same launch with only the 9 hi segments leaves the
    f16 rounding of t and must fail the bound the full launch meets.

    On H100 the full launch measures 0.9e-5 - 1.0e-5 normwise, and nearly all of it is the tensor cores' f32 accumulation over
    K = 18 Ipad (printed as "accumulation alone": against the exact conv of the operands y, y_lo), not the operand error
    (~2^-22); the hi-only control measures 1.85e-4 - 2.2e-4. HEAD_LO_TOL = 5.5e-5 sits 5x above the first and 3.4x below the
    second."""
    g = torch.Generator().manual_seed(B * 1000 + H + W + C)
    HW, O = H * W, 4
    x = (torch.randn(B, HW, C, generator=g) * 1.5 + 0.3).to(DEV)
    gam = (1 + 0.1 * torch.randn(C, generator=g)).to(DEV)
    bet = (0.1 * torch.randn(C, generator=g)).to(DEV)
    w = (torch.randn(O, C, 3, 3, generator=g) / math.sqrt(9 * C)).half().to(DEV)
    b16 = (torch.randn(O, generator=g) * 0.1).half().to(DEV)
    b32 = torch.empty(O, dtype=torch.float32, device=DEV)
    T.bias_to_f32(b16, O, b32)
    y = torch.full((B, H, W, C), float("nan"), dtype=torch.float16, device=DEV)
    y_lo = torch.full_like(y, float("nan"))
    T.group_norm(x, None, B, HW, 32, gam, bet, 1e-5, True, y, None, y_lo, T.gn_scratch(B, 32))
    Ipad = pad64(C)
    Ktot = 9 * Ipad
    wt = repack3(w, Ktot).view(O, Ktot)
    w2 = torch.cat([wt, wt], dim=1).contiguous()
    hi, lo = conv_taps(Ipad // 64, 0), conv_taps(Ipad // 64, 1)
    outs = {}
    for name, segs in (("hi + lo", hi + lo), ("hi only", hi)):
        out, guard = guarded((B, H, W, O))
        T.igemm(y, (B, H, W, C), w2, O, 2 * Ktot, (W, H, B), segs, out, O, a1=y_lo, a1_shape=(B, H, W, C), bias=b32)
        assert bool(guard.isnan().all()), f"head conv {name}: elements after the output were written"
        outs[name] = out
    t, e32 = gn_ref(x, None, B, HW, 32, gam, bet, 1e-5, True)
    t = t.view(B, H, W, C)
    ref = conv_ref(t, w) + b16.double()
    mag = conv_ref(y.double().abs() + y_lo.double().abs(), w.abs()) + b16.double().abs()
    ops = conv_ref(y.double() + y_lo.double(), w) + b16.double()       # exact result on the operands the kernel reads
    e_op = conv_ref((e32.view(B, H, W, C) + 2.0 ** -22 * t.abs() + H_SUB), w.abs())
    check(outs["hi + lo"], ref, (18 * Ipad + 1) * U23 * mag + e_op, f"head conv hi/lo {B}x{H}x{W}x{C}")
    rel = {k: float((v.double() - ref).norm() / ref.norm()) for k, v in outs.items()}
    acc = float((outs["hi + lo"].double() - ops).norm() / ref.norm())
    print(f"head conv {B}x{H}x{W}x{C}: normwise rel err hi + lo {rel['hi + lo']:.3e} (accumulation alone {acc:.3e}), "
          f"hi only {rel['hi only']:.3e}")
    assert rel["hi + lo"] < HEAD_LO_TOL, "head conv: the hi / lo split must keep the operand error far below f16's"
    assert rel["hi only"] > HEAD_LO_TOL, "head conv: the hi-only control must fail the bound the hi / lo launch meets"
