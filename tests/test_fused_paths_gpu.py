"""The UNet launch plan's fused kernel forms, launched one kernel at a time and compared with float64 torch.

The operator entry points (test_ops_gpu.py) reach the kernels only through their simplest layouts. Here every kernel gets
the parameter sets the plan (engine_core.h: PlanBuilder, engine.cu: resblock / strans) gives it: the upsample conv as four
scattered 2x2 phase convolutions, a 1x1 skip fused as a second K source, per-batch bias rows, GroupNorm's raw / y_lo outputs
on one shared scratch, attention on column windows of fused QKV / KV matrices with a second (IP-Adapter) source, the
text-encoder attention at every head dim, and the GEMV, first-conv and LoRA-merge kernels. The launchers are reached through
the test-only library libsdxl_b200_testing.so (sdxl_b200._testing).

Every reference is float64 on the very operands the kernel reads (f16 values, or f32 where the kernel reads f32), and every
tolerance is an elementwise bound derived from the kernel's arithmetic:
  - f32 accumulation of n exact products (f16 x f16 fits in f32): |err| <= n * 2^-23 * sum|terms| (one f32 ulp per addition,
    which also covers an adder that truncates);
  - one f16 output rounding: 2^-11 relative (2^-25 absolute below the f16 normal range);
  - attention: P rounded to f16 before the PV contraction, 2^-11 relative per probability.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from sdxl_b200 import SdxlError
from sdxl_b200 import _testing as T
from harness import (DEV, H11, H_SUB, U23, U24, attn_ref, check, conv_taps, f16_round_bound, gn_ref, heads, nchw, pad64,
                     plan_upconv, repack3, to_rows)

pytestmark = pytest.mark.gpu


def f16(t: torch.Tensor) -> torch.Tensor:
    return t.to(DEV, torch.float16).contiguous()


def randn(g, *shape, scale=1.0, shift=0.0):
    return torch.randn(*shape, generator=g) * scale + shift


# ------------------------------------------------------------------------------------------------------------------------------
# implicit GEMM: the plan's convolution forms
# ------------------------------------------------------------------------------------------------------------------------------
def upconv_phase_weights_host(w: torch.Tensor) -> torch.Tensor:
    """repack_upconv_kernel's summed taps, added in f32 in its (kh, kw) order and rounded once: [4 (a, b), O, 4 (th, tw), I]."""
    w = w.float().cpu()
    O, I = w.shape[:2]
    out = torch.zeros(4, O, 4, I, dtype=torch.float16)
    rows = {(0, 0): (0, 0), (0, 1): (1, 2), (1, 0): (0, 1), (1, 1): (2, 2)}   # (parity, tap) -> first, last 3x3 row / column
    for a in range(2):
        for b in range(2):
            for th in range(2):
                for tw in range(2):
                    kh0, kh1 = rows[(a, th)]
                    kw0, kw1 = rows[(b, tw)]
                    acc = torch.zeros(O, I, dtype=torch.float32)
                    for kh in range(kh0, kh1 + 1):
                        for kw in range(kw0, kw1 + 1):
                            acc = acc + w[:, :, kh, kw]
                    out[a * 2 + b, :, th * 2 + tw] = acc.half()
    return out


def phase_conv64(x: torch.Tensor, wph: torch.Tensor) -> torch.Tensor:
    """float64 four-phase convolution: x [B, H, W, I] (any dtype), wph [4, O, 4, I] -> [B, 2H, 2W, O]."""
    B, H, W, I = x.shape
    O = wph.shape[1]
    xd = nchw(x.double())
    out = torch.empty(B, O, 2 * H, 2 * W, dtype=torch.float64, device=x.device)
    for a in range(2):
        for b in range(2):
            k = wph[a * 2 + b].double().reshape(O, 2, 2, I).permute(0, 3, 1, 2)   # [O, I, th, tw]
            xp = F.pad(xd, (1 - b, b, 1 - a, a))    # a = 0: rows i-1, i ; a = 1: rows i, i+1 (same for columns)
            out[:, :, a::2, b::2] = F.conv2d(xp, k)
    return out.permute(0, 2, 3, 1)


@pytest.mark.parametrize("B,H,W,I,O", [(1, 4, 4, 64, 64), (1, 5, 7, 320, 320), (2, 20, 24, 72, 72), (1, 5, 7, 72, 320),
                                       (2, 64, 64, 640, 640)])
def test_upsample_conv_plan_form(ctx, B, H, W, I, O):
    g = torch.Generator().manual_seed(B * 1000 + H * 10 + W + I + O)
    x = randn(g, B, H, W, I).half()
    w = (randn(g, O, I, 3, 3) / math.sqrt(9 * I)).half()
    b = (randn(g, O) * 0.1).half()
    x16, w16, b32 = f16(x), f16(w), b.float().to(DEV)
    out, wup = plan_upconv(x16, w16, b32)
    torch.cuda.synchronize()
    # the phase kernels are the f16 rounding of the f32 sums of the taps that read the same source pixel (bit exact)
    wph = upconv_phase_weights_host(w)
    assert torch.equal(wup[:, :, :, :I].cpu().view(torch.int16), wph.view(torch.int16))
    assert not bool(wup[:, :, :, I:].any()), "padded input channels of the phase kernels must be zero"
    # 1) the GEMM on the operands it reads (x, phase kernels): f32 accumulation of 4 * Ipad products and the bias
    ref = phase_conv64(x16, wph.to(DEV)) + b32.double()
    mag = phase_conv64(x16.abs(), wph.to(DEV).abs()) + b32.double().abs()
    check(out, ref, (4 * I + 1) * U23 * mag, "upconv vs float64 phase convolution")
    # 2) against nearest-2x upsample -> 3x3 conv: the phase kernels' own f16 rounding adds 2^-11 * |x| . |w_phase|
    #    (each phase weight is f16(f32 sum of <= 4 taps): within 2^-11 |sum| + 3 * 2^-24 sum|taps| of the exact sum)
    up = F.interpolate(nchw(x16.double()), scale_factor=2, mode="nearest")
    ref3 = F.conv2d(up, w16.double(), b32.double(), padding=1).permute(0, 2, 3, 1)
    mag3 = F.conv2d(up.abs(), w16.double().abs(), b32.double().abs(), padding=1).permute(0, 2, 3, 1)
    e_plan = (4 * I + 1) * U23 * mag + H11 * mag + 3 * U24 * mag3
    check(out, ref3, e_plan, "upconv vs interpolate + conv2d")
    # 3) the operator entry point (materialised upsample, 3x3 weights: 9 * I products) agrees with the same reference, and
    #    with the plan form within the sum of the two bounds. The phase weights' f16 rounding keeps the two apart by
    #    ~1e-4 normwise, so they are compared elementwise against that bound, not bit for bit.
    op = ctx.conv2d(x.float(), w, b, upsample=True)
    e_op = (9 * I + 1) * U23 * mag3
    check(op, ref3, e_op, "op conv2d(upsample) vs interpolate + conv2d")
    check(out, op.double(), e_plan + e_op, "upconv vs sdxl_op_conv2d(upsample=1)")
    print(f"upconv vs sdxl_op_conv2d(upsample=1): normwise rel diff "
          f"{float((out.double() - op.double()).norm() / op.double().norm()):.3e}")


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 12, 12, 960, 320), (3, 9, 10, 1920, 640), (2, 5, 7, 320, 320)])
def test_resnet_first_conv_per_batch_bias(ctx, B, H, W, Cin, Cout):
    """resblock's first conv: the time embedding is folded into a per-batch bias row temb_all[b, off:off + Cout]."""
    g = torch.Generator().manual_seed(B + H + W + Cin + Cout)
    x16 = f16(randn(g, B, H, W, Cin))
    w16 = f16(randn(g, Cout, Cin, 3, 3) / math.sqrt(9 * Cin))
    off, temb_total = 640, 640 + Cout + 320
    temb_all = (randn(g, B, temb_total)).to(DEV)     # distinct rows per batch
    Ktot = 9 * pad64(Cin)
    wt = repack3(w16, Ktot)
    out = torch.full((B, H, W, Cout), float("nan"), device=DEV)
    T.igemm(x16, (B, H, W, Cin), wt, Cout, Ktot, (W, H, B), conv_taps(pad64(Cin) // 64), out, Cout,
            bias=temb_all.view(-1)[off:], bias_bstride=temb_total)
    bias = temb_all[:, off:off + Cout].double()[:, None, None, :]
    ref = F.conv2d(nchw(x16.double()), w16.double(), padding=1).permute(0, 2, 3, 1) + bias
    mag = F.conv2d(nchw(x16.double().abs()), w16.double().abs(), padding=1).permute(0, 2, 3, 1) + bias.abs()
    check(out, ref, (9 * Cin + 1) * U23 * mag, "first conv + per-batch bias")


@pytest.mark.parametrize("B,H,W,C1,C2,Cout", [(2, 12, 12, 640, 320, 320), (2, 10, 6, 1280, 640, 640), (1, 9, 9, 320, 0, 640)])
def test_resnet_second_conv_fused_skip(ctx, B, H, W, C1, C2, Cout):
    """resblock's second conv with the 1x1 skip conv as a K segment on the second source: the GroupNorm's raw output
    f16(cat(x1, x2)), weights repacked to [Cout, 9 * Ipad | I2pad], bias = conv bias + skip bias."""
    g = torch.Generator().manual_seed(B + H + W + C1 + C2 + Cout)
    Cin = C1 + C2
    HW = H * W
    x1 = (randn(g, B, HW, C1, scale=1.5, shift=0.3)).to(DEV)
    x2 = (randn(g, B, HW, C2, scale=0.7, shift=-0.2)).to(DEV) if C2 else None
    gam, bet = (1 + 0.1 * randn(g, Cin)).to(DEV), (0.1 * randn(g, Cin)).to(DEV)
    y = torch.empty(B, HW, Cin, dtype=torch.float16, device=DEV)
    raw = torch.empty_like(y)
    scratch = T.gn_scratch(B, 32)
    T.group_norm(x1, x2, B, HW, 32, gam, bet, 1e-5, True, y, raw, None, scratch)
    a0 = f16(randn(g, B, H, W, Cout))                         # stands for the second GroupNorm's output
    w3 = f16(randn(g, Cout, Cout, 3, 3) / math.sqrt(9 * Cout))
    ws = f16(randn(g, Cout, Cin, 1, 1) / math.sqrt(Cin))
    b3, bs = f16(randn(g, Cout) * 0.1), f16(randn(g, Cout) * 0.1)
    Ipad, I2pad = pad64(Cout), pad64(Cin)
    Ktot = 9 * Ipad + I2pad
    wt = repack3(w3, Ktot)
    repack3(ws, Ktot, wt, 9 * Ipad)
    bias = torch.empty(Cout, device=DEV)
    T.bias_to_f32(b3, Cout, bias)
    T.bias_to_f32(bs, Cout, bias, accumulate=True)
    out = torch.full((B, H, W, Cout), float("nan"), device=DEV)
    segs = conv_taps(Ipad // 64) + [(1, 0, 0, 0, I2pad // 64)]
    T.igemm(a0, (B, H, W, Cout), wt, Cout, Ktot, (W, H, B), segs, out, Cout, a1=raw.view(B, H, W, Cin),
            a1_shape=(B, H, W, Cin), bias=bias)
    xc = x1 if x2 is None else torch.cat([x1, x2], dim=2)
    assert torch.equal(raw, xc.half()), "GroupNorm raw output must be f16(cat(x1, x2))"
    r64 = raw.double().view(B, H, W, Cin)
    bsum = b3.double() + bs.double()
    ref = (F.conv2d(nchw(a0.double()), w3.double(), padding=1) + F.conv2d(nchw(r64), ws.double())).permute(0, 2, 3, 1) + bsum
    mag = (F.conv2d(nchw(a0.double().abs()), w3.double().abs(), padding=1)
           + F.conv2d(nchw(r64.abs()), ws.double().abs())).permute(0, 2, 3, 1) + b3.double().abs() + bs.double().abs()
    check(out, ref, (9 * Cout + Cin + 2) * U23 * mag, "second conv + fused 1x1 skip")


@pytest.mark.parametrize("B,H,W,C", [(2, 12, 12, 320), (3, 5, 7, 640), (1, 16, 16, 1280)])
def test_resnet_second_conv_identity_residual(ctx, B, H, W, C):
    """resblock's second conv without a skip conv: the block input (f32) is added in the GEMM epilogue (ldr = ldo = C)."""
    g = torch.Generator().manual_seed(B + H + W + C + 7)
    a0 = f16(randn(g, B, H, W, C))
    w3 = f16(randn(g, C, C, 3, 3) / math.sqrt(9 * C))
    b32 = (randn(g, C) * 0.1).half().float().to(DEV)
    res = randn(g, B, H, W, C, scale=2.0).to(DEV)
    Ktot = 9 * pad64(C)
    wt = repack3(w3, Ktot)
    out = torch.full((B, H, W, C), float("nan"), device=DEV)
    T.igemm(a0, (B, H, W, C), wt, C, Ktot, (W, H, B), conv_taps(pad64(C) // 64), out, C, bias=b32, res=res, ldr=C)
    ref = F.conv2d(nchw(a0.double()), w3.double(), padding=1).permute(0, 2, 3, 1) + b32.double() + res.double()
    mag = F.conv2d(nchw(a0.double().abs()), w3.double().abs(), padding=1).permute(0, 2, 3, 1) + b32.double().abs() + res.double().abs()
    check(out, ref, (9 * C + 2) * U23 * mag, "second conv + identity residual")


# ------------------------------------------------------------------------------------------------------------------------------
# GroupNorm
# ------------------------------------------------------------------------------------------------------------------------------
def run_gn(B, HW, C1, C2, G, silu, scratch, g):
    x1 = randn(g, B, HW, C1, scale=1.5, shift=0.3).to(DEV)
    x2 = randn(g, B, HW, C2, scale=0.7, shift=-0.2).to(DEV) if C2 else None
    C = C1 + C2
    gam, bet = (1 + 0.1 * randn(g, C)).to(DEV), (0.1 * randn(g, C)).to(DEV)
    y = torch.full((B, HW, C), float("nan"), dtype=torch.float16, device=DEV)
    raw, y_lo = torch.full_like(y, float("nan")), torch.full_like(y, float("nan"))
    T.group_norm(x1, x2, B, HW, G, gam, bet, 1e-5, silu, y, raw, y_lo, scratch)
    return x1, x2, gam, bet, y, raw, y_lo


def check_gn(B, HW, C1, C2, G, silu, x1, x2, gam, bet, y, raw, y_lo, what):
    xc = x1 if x2 is None else torch.cat([x1, x2], dim=2)
    assert torch.equal(raw.view(torch.int16), xc.half().view(torch.int16)), f"{what}: raw != f16(cat(x1, x2))"
    t, e32 = gn_ref(x1, x2, B, HW, G, gam, bet, 1e-5, silu)
    check(y, t, f16_round_bound(t) + e32, f"{what}: y")
    # y_lo = f16(t32 - y): its own rounding is 2^-11 of |t32 - y| <= 2^-11 |t|, i.e. 2^-22 |t| (2^-25 absolute when the residue
    # is an f16 subnormal); a y_lo that is dropped or has the wrong sign leaves ~2^-12 |t|
    check(y.double() + y_lo.double(), t, e32 + 2.0 ** -22 * t.abs() + H_SUB, f"{what}: y + y_lo")


@pytest.mark.parametrize("B,HW,C1,C2,G,silu", [
    (2, 1024, 640, 320, 32, True),      # the resnet's cat form
    (1, 64, 320, 0, 64, False),         # 5 channels per group: a float4 straddles two groups
    (2, 256, 256, 0, 4, True),
    (1, 100, 128, 64, 8, False),
    (3, 49, 256, 0, 16, True),
    (1, 300, 48, 0, 12, True),          # 4 channels per group
    (1, 37, 1040, 0, 40, True),         # 260-thread stats CTA: the last warp is partial and 8 * 40 lanes > 260
])
def test_group_norm_raw_and_hi_lo(ctx, B, HW, C1, C2, G, silu):
    g = torch.Generator().manual_seed(B * 7 + HW + C1 + C2 + G)
    scratch = T.gn_scratch(B, G)
    out = run_gn(B, HW, C1, C2, G, silu, scratch, g)
    check_gn(B, HW, C1, C2, G, silu, *out, f"gn B={B} HW={HW} C={C1}+{C2} G={G}")


def test_group_norm_shared_scratch():
    """The plan runs every GroupNorm of a step on one scratch initialised once: the last CTA of each sample must leave its
    arrival counter at zero for the next GroupNorm, whatever the previous one's shape (fewer chunks, fewer samples)."""
    g = torch.Generator().manual_seed(11)
    scratch = T.gn_scratch(3, 64)
    shapes = [(3, 4096, 640, 0, 32, True), (1, 3, 320, 320, 64, False), (2, 1, 64, 0, 8, True), (3, 4096, 640, 0, 32, True)]
    runs = [run_gn(*s, scratch, g) for s in shapes]
    torch.cuda.synchronize()
    for s, r in zip(shapes, runs):
        check_gn(*s, *r, f"shared scratch gn {s}")


def test_group_norm_rejects_n_group_not_multiple_of_4(ctx):
    """gn_launch requires n_group % 4 == 0 (its final reduction gives each group 8 lanes of a full-mask warp shuffle); the
    check runs before any launch."""
    g = torch.Generator().manual_seed(3)
    x = randn(g, 1, 16, 48)
    gam, bet = torch.ones(48), torch.zeros(48)
    for n_group in (3, 6, 0):
        with pytest.raises(SdxlError):
            ctx.group_norm(x, None, gam, bet, n_group=n_group)
    out = ctx.group_norm(x, None, gam, bet, n_group=12)
    t, e32 = gn_ref(x.to(DEV), None, 1, 16, 12, gam.to(DEV), bet.to(DEV), 1e-5, False)
    check(out, t, f16_round_bound(t) + e32, "op group_norm n_group=12")


# ------------------------------------------------------------------------------------------------------------------------------
# LayerNorm
# ------------------------------------------------------------------------------------------------------------------------------
def ln_ref(x, gam, bet, eps, unbiased=False):
    """float64 LayerNorm over the last dim of x [rows, C], and the bound on layernorm_kernel's f32 evaluation error (one warp per
    row, NV = ceil(C / 128) float4 per lane, exact two-pass statistics):
      - each warp sum: 4 NV lane-serial additions, then 5 shuffle levels: (4 NV + 5) 2^-24 sum|terms|; mean = sum / C rounds
        once more;
      - q = sum (x - mean32)^2: each centred value rounded (doubled by the square), each square rounded, then the same sum;
        the mean's error d adds C d^2 exactly (sum (x - mean) = 0); var = q / C + eps: two roundings;
      - rstd = 1 / sqrtf(var): half the variance's relative error, plus two roundings;
      - y = (x - mean32) rstd gamma + beta: the mean's error times rstd |gamma|, the relative errors of the centred value and of
        rstd, and three roundings.
    The estimate is first order; a factor 2 covers the second-order terms. unbiased: the sample variance (sum / (C - 1)), a
    reference the bound must reject."""
    xd = x.double()
    C = xd.shape[1]
    n_add = 4 * ((C + 127) // 128) + 5
    mean = xd.mean(dim=1, keepdim=True)
    d = xd - mean
    var = (d * d).sum(dim=1, keepdim=True) / (C - 1 if unbiased else C)
    rstd = 1.0 / torch.sqrt(var + eps)
    ref = d * rstd * gam.double() + bet.double()
    e_mean = (n_add + 1) * U24 * xd.abs().mean(dim=1, keepdim=True)
    rel_var = ((n_add + 6) * U24 * (var + e_mean ** 2) + e_mean ** 2) / (var + eps) + U24
    rel_rstd = 0.5 * rel_var + rel_var ** 2 + 2 * U24
    e32 = 2 * (gam.double().abs() * rstd * (e_mean + d.abs() * (rel_rstd + 4 * U24)) + 2 * U24 * (ref.abs() + bet.double().abs()))
    return ref, e32


def ln_rows(g, kind, rows, C):
    if kind == "N(0.5, 2)":
        return randn(g, rows, C, scale=2.0, shift=0.5)
    if kind == "large mean":        # |mean| / std up to 1e3
        std = torch.exp(randn(g, rows, 1))
        return randn(g, rows, C) * std + (torch.rand(rows, 1, generator=g) * 2 - 1) * 1e3 * std
    if kind == "std 1e-3":          # eps = 1e-5 is ten times the variance
        return randn(g, rows, C, scale=1e-3, shift=0.3)
    # constant rows of multiples of 2^-4: the sums and the mean are exact, so x - mean = 0 and y = beta
    return (torch.randint(-64, 65, (rows, 1), generator=g).float() / 16).expand(rows, C).contiguous()


@pytest.mark.parametrize("C", [64, 100, 320, 384, 640, 768, 1024, 1280, 1536, 1664, 2048])
def test_layer_norm(ctx, C):
    """layernorm_kernel through sdxl_op_layer_norm at every width class (all five NV instantiations; C = 100 and 1664 leave the
    last float4 group of the warp partly empty), row counts that are not a multiple of the 8 warps of a CTA, and four kinds of
    rows: N(0.5, 2), |mean| / std up to 1e3, std 1e-3 (eps comparable to the variance) and constant rows (output exactly
    f16(beta)). At C <= 320 the bound must also reject the unbiased-variance reference (a relative change of 1 / (2C) in rstd)."""
    g = torch.Generator().manual_seed(C)
    gam, bet = 1 + 0.1 * randn(g, C), 0.1 * randn(g, C)
    gd, bd = gam.to(DEV), bet.to(DEV)
    for rows in (1, 7, 154, 2964, 8193):
        for kind in ("N(0.5, 2)", "large mean", "std 1e-3", "constant"):
            x = ln_rows(g, kind, rows, C).to(DEV)
            out = ctx.layer_norm(x, gam, bet, 1e-5)
            ref, e32 = ln_ref(x, gd, bd, 1e-5)
            tol = f16_round_bound(ref) + e32
            check(out, ref, tol, f"layer_norm C={C} rows={rows} {kind}")
            if kind == "constant":
                assert torch.equal(out, bd.half().expand(rows, C)), f"C={C}: a constant row must give exactly f16(beta)"
            if kind == "N(0.5, 2)" and C <= 320:
                ref_u, _ = ln_ref(x, gd, bd, 1e-5, unbiased=True)
                assert bool(((out.double() - ref_u).abs() > tol).any()), \
                    f"C={C} rows={rows}: the bound does not tell the biased from the unbiased variance"


def test_layer_norm_rejects(ctx):
    """layernorm_launch reads rows as float4 and caches at most 16 per lane: C % 4 != 0 (3003) and C > 2048 (3004) are refused."""
    for C, code in ((102, 3003), (2052, 3004), (4096, 3004)):
        x = torch.zeros(3, C)
        with pytest.raises(SdxlError, match=rf"\({code}\)"):
            ctx.layer_norm(x, torch.ones(C), torch.zeros(C))


# ------------------------------------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,T_,nh", [(1, 1, 1), (3, 129, 5), (1, 128, 1), (3, 127, 20), (1, 4096, 5)])
def test_flash_attention_fused_qkv(ctx, B, T_, nh):
    """Self-attention as strans runs it: q, k and v are the column windows 0, C, 2C of one [B*T, 3C] QKV matrix."""
    g = torch.Generator().manual_seed(B + T_ + nh)
    C = nh * 64
    qkv = f16(randn(g, B * T_, 3 * C))
    out = torch.full((B * T_, C), float("nan"), dtype=torch.float16, device=DEV)
    T.attention(qkv, 3 * C, 0, qkv, 3 * C, C, 2 * C, B, T_, T_, nh, out, C)
    ref, tol = attn_ref(heads(qkv, B, T_, 0, nh, 64), heads(qkv, B, T_, C, nh, 64), heads(qkv, B, T_, 2 * C, nh, 64), 0.125)
    ref, tol = to_rows(ref), to_rows(tol)
    check(out, ref, tol + f16_round_bound(ref), f"fused-QKV attention B={B} T={T_} heads={nh}")


@pytest.mark.parametrize("B,T_,S,nh", [(1, 1, 1, 1), (3, 129, 77, 20), (1, 4096, 77, 5), (1, 127, 257, 5),
                                       (3, 128, 128, 1), (1, 129, 127, 5), (3, 1, 129, 5)])
def test_flash_attention_kv_window(ctx, B, T_, S, nh):
    """Cross-attention as strans runs it: K / V are the column windows 0 and C of a [B*S, 2C] matrix. The output is written
    with row pitch 3C; its other columns must be left untouched."""
    g = torch.Generator().manual_seed(B * 3 + T_ + S + nh)
    C = nh * 64
    q = f16(randn(g, B * T_, C))
    kv = f16(randn(g, B * S, 2 * C))
    out = torch.full((B * T_, 3 * C), -7.0, dtype=torch.float16, device=DEV)
    T.attention(q, C, 0, kv, 2 * C, 0, C, B, T_, S, nh, out, 3 * C)
    ref, tol = attn_ref(heads(q, B, T_, 0, nh, 64), heads(kv, B, S, 0, nh, 64), heads(kv, B, S, C, nh, 64), 0.125)
    ref, tol = to_rows(ref), to_rows(tol)
    check(out[:, :C], ref, tol + f16_round_bound(ref), f"KV-window attention B={B} T={T_} S={S} heads={nh}")
    assert bool((out[:, C:] == -7.0).all()), "columns outside the output window were written"


@pytest.mark.parametrize("B,T_,S,S_ip,nh", [(1, 129, 77, 4, 5), (3, 128, 77, 8, 1), (1, 127, 129, 129, 5), (3, 1, 1, 4, 20)])
def test_flash_attention_ip_source(ctx, B, T_, S, S_ip, nh):
    """The IP-Adapter's second key/value source with both windows at non-zero columns (k_ip at C, v_ip at 2C of a
    [B*S_ip, 3C] matrix): out = softmax(q k^T / 8) v + s softmax(q k_ip^T / 8) v_ip."""
    g = torch.Generator().manual_seed(B + T_ + S + S_ip + nh)
    C = nh * 64
    q = f16(randn(g, B * T_, C))
    kv = f16(randn(g, B * S, 2 * C))
    kvip = f16(randn(g, B * S_ip, 3 * C))
    s = torch.tensor([0.7], device=DEV)
    out = torch.full((B * T_, C), float("nan"), dtype=torch.float16, device=DEV)
    T.attention(q, C, 0, kv, 2 * C, 0, C, B, T_, S, nh, out, C, kip=kvip, kip_pitch=3 * C, k_ip_col0=C, v_ip_col0=2 * C,
                S_ip=S_ip, ip_scale=s)
    qh = heads(q, B, T_, 0, nh, 64)
    r1, t1 = attn_ref(qh, heads(kv, B, S, 0, nh, 64), heads(kv, B, S, C, nh, 64), 0.125)
    r2, t2 = attn_ref(qh, heads(kvip, B, S_ip, C, nh, 64), heads(kvip, B, S_ip, 2 * C, nh, 64), 0.125)
    ref = to_rows(r1 + 0.7 * r2)
    # the two normalised sources are combined in f32 (fmaf(s, o_ip / l_ip, o_txt / l_txt)): 2^-23 of |o_txt| + s |o_ip|
    tol = to_rows(t1 + 0.7 * t2 + U23 * (r1.abs() + 0.7 * r2.abs()))
    check(out, ref, tol + f16_round_bound(ref), f"IP attention B={B} T={T_} S={S} S_ip={S_ip} heads={nh}")


def test_flash_attention_large_logits(ctx):
    """|q.k| / 8 around 60, with the later key blocks dominating: the running max of each key block is exact, so no
    probability exceeds 1 before its f16 rounding and nothing overflows."""
    g = torch.Generator().manual_seed(5)
    B, T_, S, nh = 1, 129, 257, 5
    C = nh * 64
    qkv = randn(g, B * T_, 3 * C) * 4.5
    q = f16(qkv[:, :C])
    kv = randn(g, B * S, 2 * C)
    kv[:, :C] *= 4.5
    kv[130:, :C] *= 1.5
    kv = f16(kv)
    out = torch.full((B * T_, C), float("nan"), dtype=torch.float16, device=DEV)
    T.attention(q, C, 0, kv, 2 * C, 0, C, B, T_, S, nh, out, C)
    qh, kh = heads(q, B, T_, 0, nh, 64), heads(kv, B, S, 0, nh, 64)
    logits = (qh @ kh.transpose(-1, -2)).abs() * 0.125
    assert float(logits.amax()) > 60
    ref, tol = attn_ref(qh, kh, heads(kv, B, S, C, nh, 64), 0.125)
    ref, tol = to_rows(ref), to_rows(tol)
    assert bool(torch.isfinite(out).all())
    check(out, ref, tol + f16_round_bound(ref), "attention with large logits")


HEAD_DIMS = [8, 16, 24, 32, 40, 48, 56, 64, 72, 80, 88, 96, 104, 112, 120, 128]


@pytest.mark.parametrize("d", HEAD_DIMS)
def test_attention_small_layouts(ctx, d):
    """The text / vision encoders' attention kernel at every head dim it is instantiated for, with causal alone, an additive
    mask alone and both, in two layouts: the encoders' fused QKV (pitch 3C, windows 0 / C / 2C, S = T = 77) and separate
    q / kv matrices with odd pitches and column offsets (T = 45, S = 77: S is not a multiple of the 32-key chunk). A query
    whose keys are all masked returns exactly 0."""
    nh = 3
    C = nh * d
    g = torch.Generator().manual_seed(d)
    B = 2
    layouts = {
        "fused": dict(T=77, S=77, q_pitch=3 * C, q_col0=0, kv_pitch=3 * C, k_col0=C, v_col0=2 * C),
        "windows": dict(T=45, S=77, q_pitch=C + 16, q_col0=8, kv_pitch=2 * C + 24, k_col0=16, v_col0=C + 24),
    }
    for name, L in layouts.items():
        T_, S = L["T"], L["S"]
        qm = f16(randn(g, B * T_, L["q_pitch"]))
        kvm = qm if name == "fused" else f16(randn(g, B * S, L["kv_pitch"]))
        mask = randn(g, T_, S, scale=2.0)
        dead = 5                                         # query row whose keys are all masked
        mask[dead, :] = float("-inf")
        mask16 = f16(mask)
        for mode in ("causal", "mask", "both"):
            causal = mode != "mask"
            mk = None if mode == "causal" else mask16
            out = torch.full((B * T_, C), float("nan"), dtype=torch.float16, device=DEV)
            T.attention_small(qm, L["q_pitch"], L["q_col0"], kvm, kvm, L["kv_pitch"], L["k_col0"], L["v_col0"], B, T_, S, nh,
                              mk, causal, out, C, d)
            qh = heads(qm, B, T_, L["q_col0"], nh, d)
            kh = heads(kvm, B, S, L["k_col0"], nh, d)
            vh = heads(kvm, B, S, L["v_col0"], nh, d)
            ref, tol = attn_ref(qh, kh, vh, 1.0 / math.sqrt(d), None if mk is None else mk.double(), causal, p_f16=False)
            ref, tol = to_rows(ref), to_rows(tol)
            o = out.view(B, T_, C)
            live = torch.ones(T_, dtype=torch.bool)
            if mk is not None:
                assert bool((o[:, dead] == 0).all()), f"d={d} {name} {mode}: a fully masked query must return 0"
                live[dead] = False
            live = live.repeat(B)
            check(out[live], ref[live], tol[live] + f16_round_bound(ref[live]), f"attention_small d={d} {name} {mode}")


# ------------------------------------------------------------------------------------------------------------------------------
# GEMV, first conv
# ------------------------------------------------------------------------------------------------------------------------------
def silu64(x):
    return x * torch.sigmoid(x)


@pytest.mark.parametrize("Bv", [1, 2, 3, 8])
@pytest.mark.parametrize("K", [1280, 1283])
def test_gemv(ctx, Bv, K):
    """gemv_launch as the plan's embedding GEMVs use it: K-major weights with row pitch ldw > K (transpose_linear's padded
    layout), SiLU on the input and the output, an added row with a batch stride, N = 1003 (not a multiple of the 8 warps of
    a CTA). K = 1280 takes the 128-bit path and K = 1283 the scalar one; K = 1280 is also forced onto the scalar path by a
    misaligned input, and the two must agree."""
    g = torch.Generator().manual_seed(Bv * 10 + K)
    N = 1003
    ldw = pad64(K)
    w_kn = f16(randn(g, K, N) / math.sqrt(K))
    W = torch.empty(N * ldw, dtype=torch.float16, device=DEV)
    T.transpose_linear(w_kn, K, N, W, ldw)
    bias = randn(g, N, scale=0.1).to(DEV)
    in_b, add_b, out_b = K + 8, N + 5, N + 3
    x_rows = randn(g, Bv * in_b, scale=2.0).to(DEV)
    add = randn(g, Bv * add_b).to(DEV)
    Wd = w_kn.double().t()                                              # [N, K]
    for in_silu, out_silu in ((0, 0), (1, 0), (0, 1), (1, 1)):
        outs = []
        for shift in ((0, 1) if K % 8 == 0 else (0,)):                # shift 1: the same input, not 16-byte aligned -> scalar path
            store = torch.empty(shift + Bv * in_b, device=DEV)
            store[shift:] = x_rows
            inp = store[shift:]
            out = torch.full((Bv * out_b,), float("nan"), device=DEV)
            T.gemv(inp, in_b, Bv, K, W, ldw, bias, add, add_b, N, in_silu, out_silu, out, out_b)
            x = inp.view(Bv, in_b)[:, :K].double()
            xe = silu64(x) if in_silu else x
            # silu in f32 (x / (1 + __expf(-x))): 2^-20 (1 + |x|) relative
            ein = 2.0 ** -20 * (1 + x.abs()) * xe.abs() if in_silu else torch.zeros_like(x)
            z = xe @ Wd.t() + bias.double() + add.view(Bv, add_b)[:, :N].double()
            mag = xe.abs() @ Wd.abs().t() + bias.double().abs() + add.view(Bv, add_b)[:, :N].double().abs()
            eacc = (K + 2) * U23 * (mag + ein @ Wd.abs().t())          # accumulation, on the f32 SiLU'd inputs
            ez = eacc + ein @ Wd.abs().t()
            if out_silu:
                ref = silu64(z)
                esil = 2.0 ** -20 * (1 + z.abs()) * ref.abs()
                tol, tol_pair = 1.1 * ez + esil, 2 * (1.1 * eacc + esil)
            else:
                ref, tol, tol_pair = z, ez, 2 * eacc
            o = out.view(Bv, out_b)
            check(o[:, :N], ref, tol, f"gemv Bv={Bv} K={K} silu in/out={in_silu}/{out_silu} shift={shift}")
            assert bool(o[:, N:].isnan().all()), "gemv wrote past N"
            outs.append(o[:, :N])
        if len(outs) == 2:   # same f32 inputs, two summation orders: each within its accumulation bound of the exact sum
            check(outs[1], outs[0].double(), tol_pair, f"gemv vector vs scalar path Bv={Bv} silu in/out={in_silu}/{out_silu}")


@pytest.mark.parametrize("x_f32", [0, 1])
@pytest.mark.parametrize("Cin", [4, 8, 3])
@pytest.mark.parametrize("W", [8, 13])
def test_conv_in(ctx, x_f32, Cin, W):
    """The first conv (CUDA cores, f32): one latent broadcast to B = 4 output images (Bx = 1), plus a ControlNet hint
    embedding added per batch b % n_add (n_add = 2); W = 13 leaves a partial 8-pixel segment. Cin = 3 is the RGB stem of the VAE
    encoder (Cout = 128) and of the ControlNet hint encoder (Cout = 16), and Cout = 512 the decoder's width."""
    for Cout in (16, 128, 512) if Cin == 3 else (320,):
        g = torch.Generator().manual_seed(x_f32 + Cin + W + (Cout if Cin == 3 else 0))
        Bx, B, H, n_add = 1, 4, 6, 2
        x = randn(g, Bx, Cin, H, W)
        x = x.to(DEV) if x_f32 else f16(x)
        w = randn(g, Cout, Cin, 3, 3, scale=1 / math.sqrt(9 * Cin)).to(DEV)
        wk = w.permute(0, 2, 3, 1).contiguous()                             # [Cout][kh][kw][Cin]
        bias = randn(g, Cout, scale=0.1).to(DEV)
        add = randn(g, n_add, H, W, Cout).to(DEV)
        for use_add in (False, True):
            y = torch.full((B, H, W, Cout), float("nan"), device=DEV)
            T.conv_in(x, Bx, B, Cin, H, W, wk, bias, Cout, y, add if use_add else None, n_add)
            xb = x.double()[[b % Bx for b in range(B)]]
            ref = F.conv2d(xb, w.double(), bias.double(), padding=1).permute(0, 2, 3, 1)
            mag = F.conv2d(xb.abs(), w.double().abs(), bias.double().abs(), padding=1).permute(0, 2, 3, 1)
            if use_add:
                a = add.double()[[b % n_add for b in range(B)]]
                ref, mag = ref + a, mag + a.abs()
            # fmaf chain of 9 Cin products onto the bias, then the add: one f32 rounding each
            check(y, ref, (9 * Cin + 2) * U24 * mag, f"conv_in x_f32={x_f32} Cin={Cin} Cout={Cout} W={W} add={use_add}")


# ------------------------------------------------------------------------------------------------------------------------------
# LoRA merge
# ------------------------------------------------------------------------------------------------------------------------------
def geglu_perm(n: torch.Tensor, N: int, bn: int) -> torch.Tensor:
    if bn <= 0:
        return n
    half, hb = N // 2, bn // 2
    gate = (n >= half).long()
    m = n - gate * half
    return (m // hb) * bn + gate * hb + m % hb


def ulp16(v: torch.Tensor) -> torch.Tensor:
    a = v.abs().clamp_min(2.0 ** -14)
    return torch.exp2(torch.floor(torch.log2(a)) - 10)


def lora_terms(g, N, Kd, ranks, scale=0.05):
    terms = []
    for i, r in enumerate(ranks):
        up = f16(randn(g, N, r) * scale)
        down = f16(randn(g, r, Kd) * scale)
        terms.append((up, down, 0.5 + 0.25 * (i % 3) - 0.6 * (i % 2)))
    return terms


def delta64(terms):
    return sum(c * (u.double() @ d.double()) for u, d, c in terms)


@pytest.mark.parametrize("ranks", [[1], [32], [33], [80], [1, 32, 33, 80, 4, 8, 16, 64, 2, 3, 5, 7, 9, 11, 13, 40]])
@pytest.mark.parametrize("form", ["linear_f16", "linear_f32", "geglu", "conv3x3"])
def test_lora_merge(ctx, ranks, form):
    """lora_merge_kernel against f16(f64(W) + sum coef up @ down): ranks across one and several 32-rank chunks, 1 and 16
    terms; f16 and f32 storage, the GEGLU row permutation, and a 3x3 conv slot (taps = 9, Ipad > I) inside a wider matrix.
    Every slot element is within one f16 ulp of the float64 result; a zero delta (row 3: zero up rows) keeps the stored
    bits, -0 included; elements outside the slot are not written."""
    g = torch.Generator().manual_seed(len(ranks) * 100 + sum(ranks) + len(form))
    taps, I, row0, col0, geglu_bn = 1, 136, 0, 0, 0
    N = 200
    if form == "geglu":
        N, geglu_bn = 256, 128
    if form == "conv3x3":
        N, I, taps = 64, 72, 9
    Ipad = pad64(I) if taps == 9 else 0
    Kd = I * taps
    if taps == 9:
        ld, col0, row0 = 9 * Ipad + 64, 0, 2          # conv slot followed by a skip segment, two rows above it
    else:
        ld, row0, col0, Ipad = pad64(I) + 64, 3, 64, pad64(I) + 64
    rows = row0 + N + 2
    f32 = form == "linear_f32"
    W = randn(g, rows, ld, scale=0.05).half()
    W[row0 + 3] = -0.0
    src = (W.float() if f32 else W).to(DEV)
    terms = lora_terms(g, N, Kd, ranks)
    for u, _, _ in terms:
        u[3] = 0.0                                     # delta row n = 3 is exactly zero
    dst = torch.full_like(src, 1234.0)
    T.lora_merge(N, Kd, taps, terms, src, dst, ld, row0, col0, Ipad, geglu_bn)
    torch.cuda.synchronize()
    n = torch.arange(N, device=DEV)
    k = torch.arange(Kd, device=DEV)
    r_idx = (row0 + geglu_perm(n, N, geglu_bn))[:, None]
    c_idx = (col0 + (k % taps) * Ipad + k // taps)[None, :]
    got = dst[r_idx, c_idx].double()
    w0 = src[r_idx, c_idx].double()
    ref = w0 + delta64(terms)
    err = (got - ref).abs()
    assert bool((err <= ulp16(ref)).all()), f"{form} ranks={ranks}: max err / ulp {float((err / ulp16(ref)).max()):.2f}"
    row3 = dst[r_idx[3, 0], c_idx[0]]
    assert torch.equal(row3.view(torch.int32) if f32 else row3.view(torch.int16),
                       src[r_idx[3, 0], c_idx[0]].view(torch.int32) if f32 else src[r_idx[3, 0], c_idx[0]].view(torch.int16)), \
        "a zero delta must keep the weight's bits (-0 included)"
    written = torch.zeros_like(dst, dtype=torch.bool)
    written[r_idx, c_idx] = True
    assert bool((dst[~written] == 1234.0).all()), "elements outside the slot were written"


@pytest.mark.parametrize("O,I,ranks", [(64, 64, [8]), (72, 72, [33, 4]), (320, 320, [80])])
def test_lora_upconv_merge(ctx, O, I, ranks):
    """An upsample conv's LoRA: the f32 3x3 delta (delta_out of lora_merge_kernel) summed into the four 2x2 phase kernels with
    repack_upconv's tap sets, against a float64 four-phase sum; padded input channels are not written."""
    g = torch.Generator().manual_seed(O + I + sum(ranks))
    Ipad = pad64(I)
    w = f16(randn(g, O, I, 3, 3) / math.sqrt(9 * I))
    wup = torch.empty(4 * O * 4 * Ipad, dtype=torch.float16, device=DEV)
    T.repack_upconv(w, O, I, wup, Ipad)
    terms = lora_terms(g, O, I * 9, ranks)
    delta = torch.full((O, I * 9), float("nan"), device=DEV)
    T.lora_merge(O, I * 9, 9, terms, wup, wup, 4 * Ipad, 0, 0, Ipad, 0, delta_out=delta)
    d64 = delta64(terms)
    mag = sum(abs(c) * (u.double().abs() @ dd.double().abs()) for u, dd, c in terms)
    check(delta, d64, (sum(ranks) + len(ranks)) * U23 * mag, "upconv LoRA f32 delta")
    dst = torch.full_like(wup, 1234.0)
    T.lora_upconv_merge(wup, delta, O, I, dst, Ipad)
    dd = d64.view(O, I, 3, 3)
    rows = {(0, 0): (0, 0), (0, 1): (1, 2), (1, 0): (0, 1), (1, 1): (2, 2)}
    ref = wup.view(4, O, 4, Ipad)[..., :I].double().clone()
    for a in range(2):
        for b in range(2):
            for th in range(2):
                for tw in range(2):
                    kh0, kh1 = rows[(a, th)]
                    kw0, kw1 = rows[(b, tw)]
                    ref[a * 2 + b, :, th * 2 + tw] += dd[:, :, kh0:kh1 + 1, kw0:kw1 + 1].sum(dim=(2, 3))
    got = dst.view(4, O, 4, Ipad)
    err = (got[..., :I].double() - ref).abs()
    assert bool((err <= ulp16(ref)).all()), f"upconv merge: max err / ulp {float((err / ulp16(ref)).max()):.2f}"
    assert bool((got[..., I:] == 1234.0).all()), "padded input channels were written"
