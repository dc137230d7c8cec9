"""Helpers the tests share: the relative error they bound, the reference's probe input, f16 rounding, the tiny-config CFG
conditioning, a report of where two tensors differ, the UNet's plan-build counter, and the kernel-level pieces of the implicit-GEMM and GroupNorm tests (elementwise
bound check, the plan's conv tap segments and weight repacks, float64 GroupNorm, and the exact-arithmetic GEMM checks: operands
on the 2^-3 / 2^-6 / 2^-9 grid, NaN-guarded outputs, the float64 conv reference)."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from sdxl_b200 import TINY, TINY_REFINER
from sdxl_b200 import _testing as T

U23 = 2.0 ** -23      # one f32 ulp (relative)
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


def check(out: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor, what: str) -> float:
    """Every element of out within tol of ref; a NaN in out, ref or tol counts as outside. Returns the worst err / bound."""
    err = (out.double() - ref).abs()
    bad = ~(err <= tol)
    worst = float((err / tol.clamp_min(1e-300)).nan_to_num(nan=float("inf")).max())
    print(f"{what}: max err {float(err.max()):.3e}, worst err / bound {worst:.3f}")
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements outside the bound (worst err / bound {worst:.2f})"
    return worst


def f16_round_bound(ref: torch.Tensor) -> torch.Tensor:
    return ref.abs() * H11 + H_SUB


def nchw(x: torch.Tensor) -> torch.Tensor:
    return x.permute(0, 3, 1, 2)


# ------------------------------------------------------------------------------------------------------------------------------
# attention (test_fused_paths_gpu.py, test_attention_plans_gpu.py): head views of the plan's row-major matrices, float64 softmax
# ------------------------------------------------------------------------------------------------------------------------------
def heads(m: torch.Tensor, B: int, rows: int, col0: int, nh: int, d: int) -> torch.Tensor:
    """[B * rows, pitch] -> [B, nh, rows, d] float64 view of the column window starting at col0."""
    return m.view(B, rows, -1)[:, :, col0:col0 + nh * d].double().reshape(B, rows, nh, d).permute(0, 2, 1, 3)


def attn_ref(q, k, v, scale, mask=None, causal=False, p_f16=True):
    """float64 softmax(q k^T scale + mask) v, and the bound on the kernel's error before its f16 output rounding:
    - the f32 score: (d + 1) 2^-23 sum_i |q_i k_i| scale, plus exp's argument rounding and its approximation 2^-21
      (relative error of each p, and of l);
    - P rounded to f16 (flash kernel): 2^-11 p, or 2^-25 absolute for a subnormal p (p <= 1, so l >= 1);
    - f32 accumulation of S terms of p v and of l."""
    d, S = q.shape[-1], k.shape[-2]
    s = q @ k.transpose(-1, -2) * scale
    sabs = q.abs() @ k.abs().transpose(-1, -2) * scale
    if mask is not None:
        s = s + mask
    if causal:
        T_ = q.shape[-2]
        s = s.masked_fill(torch.ones(T_, S, dtype=torch.bool, device=s.device).triu(1), float("-inf"))
    m = s.amax(dim=-1, keepdim=True)
    P = torch.softmax(s, dim=-1)
    ref = P @ v
    pv = P @ v.abs()
    eps_s = ((d + 1) * U23 * sabs.amax(dim=-1, keepdim=True) + 2 * U24 * (s.abs().masked_fill(s.isinf(), 0).amax(dim=-1, keepdim=True)
             + m.abs().nan_to_num(0)) + 2.0 ** -21)
    tol = (2 * eps_s + S * U23) * pv + (eps_s + S * U24) * ref.abs()
    if p_f16:
        tol = tol + H11 * pv + H_SUB * v.abs().sum(dim=-2, keepdim=True)
    return ref, tol


def to_rows(x: torch.Tensor) -> torch.Tensor:
    """[B, nh, rows, d] -> [B * rows, nh * d]"""
    B, nh, rows, d = x.shape
    return x.permute(0, 2, 1, 3).reshape(B * rows, nh * d)


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


# ------------------------------------------------------------------------------------------------------------------------------
# exact GEMM checks (test_igemm_forms_gpu.py, test_igemm_plans_gpu.py): operands on a grid whose every partial sum is exact in f32
# ------------------------------------------------------------------------------------------------------------------------------
GRID_X, GRID_W, GRID_B = 2.0 ** -3, 2.0 ** -6, 2.0 ** -9
EXACT_SUM = 2.0 ** 22 * GRID_B    # below this, every sum of multiples of 2^-9 is exact in f32
GUARD = 4096                      # elements after each output that must stay NaN
LINEAR, GEGLU = 0, 1              # kernels.h: IgemmMode


def gen(*key) -> torch.Generator:
    return torch.Generator(device=DEV).manual_seed(sum((i + 1) * 7919 * int(k) for i, k in enumerate(key)) % (2 ** 31))


def grid(g, shape, step, lim, dtype=torch.float16) -> torch.Tensor:
    """Random integers in [-lim, lim] times step, exact in dtype."""
    return (torch.randint(-lim, lim + 1, tuple(shape), generator=g, device=DEV).double() * step).to(dtype)


def grid_x(g, *shape):
    return grid(g, shape, GRID_X, 8)


def grid_w(g, *shape):
    return grid(g, shape, GRID_W, 8)


def grid_f32(g, *shape):
    """Bias / residual values: f32 multiples of 2^-9 with magnitude <= 2^11."""
    return grid(g, shape, GRID_B, 2 ** 20, torch.float32)


def bias_f32(g, N, geglu_bn=0):
    """A grid f16 bias (magnitude <= 2047 * 2^-9, exact in f16) and its plan copy: bias_to_f32 (Loader::vec_f32)."""
    b16 = grid(g, (N,), GRID_B, 2047)
    b32 = torch.empty(N, dtype=torch.float32, device=DEV)
    T.bias_to_f32(b16, N, b32, geglu_bn=geglu_bn)
    return b16, b32


def guarded(shape, dtype=torch.float32, fill=None):
    """An output of `shape`, NaN-filled (or holding `fill`), followed by GUARD NaN elements: (output view, guard view)."""
    n = math.prod(shape)
    buf = torch.full((n + GUARD,), float("nan"), dtype=dtype, device=DEV)
    if fill is not None:
        buf[:n] = fill.reshape(-1)
    return buf[:n].view(shape), buf[n:]


def assert_exact_range(what, *bounds) -> None:
    """bounds: upper bounds of sum |x w| per output and of every added |bias| / |res|, taken from the operands."""
    tot = sum(float(b) for b in bounds)
    assert tot < EXACT_SUM, f"{what}: operands reach {tot} >= 2^22 * 2^-9, partial sums would not be exact in f32"


def conv_bound(x, w) -> float:
    """max |x| * max_o sum |w[o]|: bounds sum |x w| of every output of a conv (or Linear, w [N, K]) of x with w."""
    return float(x.abs().max()) * float(w.double().abs().reshape(w.shape[0], -1).sum(dim=1).max())


def assert_exact(out, ref, guard, what) -> None:
    """out (f32 or f16) equals the exact float64 value ref rounded once (f32(ref) is exact, so f16(f32(ref)) is RN-even); the
    guard after it (if any) is still NaN."""
    want = ref.float() if out.dtype == torch.float32 else ref.float().half()
    bad = out != want
    n_bad = int(bad.sum())
    first = tuple(bad.nonzero()[0].tolist()) if n_bad else None
    print(f"{what}: {bad.numel() - n_bad} / {bad.numel()} exact")
    assert n_bad == 0, (f"{what}: {n_bad} elements differ from the exact value, first at {first}: "
                        f"{float(out[first])} != {float(want[first])}")
    assert guard is None or bool(guard.isnan().all()), f"{what}: elements after the output were written"


def conv_ref(x, w, stride=1):
    """Exact float64 conv (padding k // 2) of x [B, H, W, I] with w [O, I, k, k]: one matmul per tap over a shifted (strided)
    view of the zero-padded input. [B, Ho, Wo, O]."""
    B, H, W, I = x.shape
    O, _, k, _ = w.shape
    p = k // 2
    xp = F.pad(x.double(), (0, 0, p, p, p, p))
    Ho, Wo = (H + 2 * p - k) // stride + 1, (W + 2 * p - k) // stride + 1
    wd = w.double()
    out = torch.zeros(B, Ho, Wo, O, dtype=torch.float64, device=x.device)
    for kh in range(k):
        for kw in range(k):
            out += xp[:, kh:kh + stride * (Ho - 1) + 1:stride, kw:kw + stride * (Wo - 1) + 1:stride] @ wd[:, :, kh, kw].t()
    return out


def linear(x16, wt, N, Kpad, out, ldo, bias=None, res=None, mode=LINEAR, geglu_bn=0) -> None:
    """PlanBuilder::linear: x [M, K] as a (1, 1, M, K) image, one 1x1 segment over the padded K."""
    M, K = x16.shape
    T.igemm(x16, (1, 1, M, K), wt, N, Kpad, (M, 1, 1), [(0, 0, 0, 0, Kpad // 64)], out, ldo, bias=bias, res=res,
            ldr=ldo if res is not None else 0, mode=mode, geglu_bn=geglu_bn)


def lin_weights(g, K, N, geglu_bn=0, wt=None, row0=0):
    """A grid Linear weight [K, N] (stored [in, out]) and its plan layout (Loader::lin_into): transpose_linear's K-major
    [N, Kpad], rows from row0 of wt (a fused matrix) or of a new one."""
    w = grid_w(g, K, N)
    if wt is None:
        wt = torch.empty(N * pad64(K), dtype=torch.float16, device=DEV)
    T.transpose_linear(w, K, N, wt, pad64(K), row0, geglu_bn)
    return w, wt


def stride2_taps(Bn: int, nkb: int):
    """engine_core.h stride2_taps: tap (kh, kw) reads phase (kh != 1, kw != 1) of the phase split, one row / column back
    for kh / kw = 0."""
    return [(0, -1 if kw == 0 else 0, -1 if kh == 0 else 0, ((kh != 1) * 2 + (kw != 1)) * Bn, nkb)
            for kh in range(3) for kw in range(3)]


def in_place_residual(g, x, w, wt, b16, b32, what) -> None:
    """out == res: the f32 residual stream updated in place, against the exact value and, bit for bit, against the same launch
    writing a separate output."""
    M, N = x.shape[0], w.shape[1]
    res = grid_f32(g, M, N)
    assert_exact_range(what, conv_bound(x, w.t()), b16.abs().max(), res.abs().max())
    inplace, guard = guarded((M, N), fill=res)
    linear(x, wt, N, pad64(x.shape[1]), inplace, N, bias=b32, res=inplace)
    sep, _ = guarded((M, N))
    linear(x, wt, N, pad64(x.shape[1]), sep, N, bias=b32, res=res)
    assert_exact(inplace, x.double() @ w.double() + b16.double() + res.double(), guard, what)
    assert torch.equal(inplace, sep), f"{what}: the in-place launch differs from the one with a separate output"
