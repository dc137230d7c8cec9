"""Helpers the tests share: the relative error they bound, the reference's probe input, f16 rounding, the tiny-config CFG
conditioning, a report of where two tensors differ, the UNet's plan-build counter, and the kernel-level pieces of the implicit-GEMM and GroupNorm tests (elementwise
bound check, the plan's conv tap segments and weight repacks, float64 GroupNorm)."""
import numpy as np
import torch

from sdxl_b200 import TINY, TINY_REFINER
from sdxl_b200 import _testing as T

U24 = 2.0 ** -24      # f32 unit roundoff
H11 = 2.0 ** -11      # f16 unit roundoff
H_SUB = 2.0 ** -25    # half the f16 subnormal spacing
DEV = "cuda"


def rel_err(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def arb(*dims):
    """arb_tensor(dims) = sin(arange(prod(dims))) — the reference's probe input (src/bin/test/main.rs:51-54)."""
    n = int(np.prod(dims))
    return torch.sin(torch.arange(n, dtype=torch.float32)).reshape(*dims)


def h16f(t):
    return t.to(torch.float16).float()


def tiny_conditioning(B=2, n_ctx=7, res=(128, 128), cfg=TINY, refiner=False):
    """Conditioning keyword arguments drawn from arb: cfg's context_full and channel_context with their unconditional rows, and with
    refiner=True also TINY_REFINER's context_open_clip and channel_context_refiner, so one conditioning serves the base and the
    refiner."""
    kw = dict(context_full=h16f(arb(B, n_ctx, cfg.context_dim) * 0.9), unconditional_context_full=h16f(arb(n_ctx, cfg.context_dim).cos()),
              channel_context=h16f(arb(B, cfg.adm_in_channels)), unconditional_channel_context=h16f(arb(cfg.adm_in_channels).cos()),
              resolution=res)
    if refiner:
        r = TINY_REFINER
        kw.update(context_open_clip=h16f(arb(B, n_ctx, r.context_dim) * 0.8),
                  unconditional_context_open_clip=h16f(arb(n_ctx, r.context_dim).cos()),
                  channel_context_refiner=h16f(arb(B, r.adm_in_channels) * 0.5),
                  unconditional_channel_context_refiner=h16f(arb(r.adm_in_channels).cos()))
    return kw


def first_difference(a: torch.Tensor, b: torch.Tensor) -> str:
    """Where b differs bit for bit from a: how many elements, the non-finite counts of each, and the largest |a - b| with its index
    (a NaN or an infinity on either side counts as the largest)."""
    if a.shape != b.shape or a.dtype != b.dtype:
        return f"shape / dtype {tuple(a.shape)} {a.dtype} vs {tuple(b.shape)} {b.dtype}"
    a64, b64 = a.double(), b.double()
    d = (a64 - b64).abs().nan_to_num(nan=float("inf"))
    d[a64 == b64] = 0
    i = int(d.flatten().argmax())
    idx = tuple(int(k) for k in torch.unravel_index(torch.tensor(i), a.shape))
    return (f"{int((a64 != b64).sum())} of {a.numel()} elements differ; non-finite: {int((~torch.isfinite(a64)).sum())} vs "
            f"{int((~torch.isfinite(b64)).sum())}; max |delta| {float(d.flatten()[i]):.3e} at {idx} "
            f"({float(a64.flatten()[i])!r} vs {float(b64.flatten()[i])!r})")


def plan_builds(d):
    """How many times the Diffuser d has built its UNet plan (sdxl_unet_plan_builds)."""
    return int(d.ctx.lib.sdxl_unet_plan_builds(d.h))


def pad64(k: int) -> int:
    return (k + 63) // 64 * 64


def check(out: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor, what: str) -> None:
    err = (out.double() - ref).abs()
    bad = err > tol
    worst = float((err / tol.clamp_min(1e-300)).max())
    print(f"{what}: max err {float(err.max()):.3e}, worst err / bound {worst:.3f}")
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements outside the bound (worst err / bound {worst:.2f})"


def f16_round_bound(ref: torch.Tensor) -> torch.Tensor:
    return ref.abs() * H11 + H_SUB


def nchw(x: torch.Tensor) -> torch.Tensor:
    return x.permute(0, 3, 1, 2)


def conv_taps(nkb: int, map_: int = 0):
    return [(map_, kw - 1, kh - 1, 0, nkb) for kh in range(3) for kw in range(3)]


def plan_upconv(x16: torch.Tensor, w: torch.Tensor, b32: torch.Tensor):
    """PlanBuilder::upconv: repack_upconv's phase kernels, then one launch per output parity (a, b) writing the pixels
    (2i + a, 2j + b) of the upsampled output through opix_row = 4W, opix_w = 2, opix_off = a * 2W + b."""
    B, H, W, I = x16.shape
    O = w.shape[0]
    Ipad = pad64(I)
    Ktot = 4 * Ipad
    wup = torch.empty(4 * O * Ktot, dtype=torch.float16, device=DEV)
    T.repack_upconv(w, O, I, wup, Ipad)
    out = torch.full((B, 2 * H, 2 * W, O), float("nan"), dtype=torch.float32, device=DEV)
    for pa in range(2):
        for pb in range(2):
            segs = [(0, tw - 1 if pb == 0 else tw, th - 1 if pa == 0 else th, 0, Ipad // 64) for th in range(2) for tw in range(2)]
            wp = wup[(pa * 2 + pb) * O * Ktot:(pa * 2 + pb + 1) * O * Ktot]
            T.igemm(x16, (B, H, W, I), wp, O, Ktot, (W, H, B), segs, out, O, bias=b32, opix=(4 * W, 2, pa * 2 * W + pb))
    return out, wup.view(4, O, 4, Ipad)


def repack3(w: torch.Tensor, Ktot: int, wt: torch.Tensor = None, col0: int = 0) -> torch.Tensor:
    O, I, kh, _ = w.shape
    if wt is None:
        wt = torch.zeros(O * Ktot, dtype=torch.float16, device=DEV)
    T.repack_conv(w, O, I, kh, kh, wt, Ktot, col0, pad64(I))
    return wt


def gn_ref(x1, x2, B, HW, G, gam, bet, eps, silu):
    """float64 GroupNorm (+SiLU) of cat(x1, x2): returns t, and the bound on the kernel's f32 evaluation error of t."""
    xc = (x1 if x2 is None else torch.cat([x1, x2], dim=2)).double()
    C = xc.shape[2]
    xg = xc.view(B, HW, G, C // G)
    mean = xg.mean(dim=(1, 3), keepdim=True)
    var = ((xg - mean) ** 2).mean(dim=(1, 3), keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    sc = (rstd * gam.double().view(1, 1, G, C // G))
    n = ((xg - mean) * sc).view(B, HW, C) + bet.double()
    # y = fmaf(x, sc, sh), sc = f32(rstd) * gamma, sh = fmaf(-mean, sc, beta), mean / rstd rounded from double to f32:
    # a few f32 roundings of the terms |x sc|, |mean sc|, |beta|
    e32 = 8 * U24 * ((xg.abs() * sc.abs()).view(B, HW, C) + (mean.abs() * sc.abs()).expand_as(xg).reshape(B, HW, C) + bet.double().abs())
    if not silu:
        return n, e32
    t = n * torch.sigmoid(n)
    # x / (1 + __expf(-x)) in f32: __expf's error grows with |x| (2^-21 + |x| 2^-23 relative); the f32 error of n passes
    # through silu' <= 1.1
    return t, 1.1 * e32 + 2.0 ** -20 * (1 + n.abs()) * t.abs()
