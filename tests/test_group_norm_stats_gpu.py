"""GroupNorm per element at every shape the plans build and at adversarial group statistics, against float64.

gn_stats_kernel (norm.cu) sums each group in a fixed order: a thread walks L = ceil(ceil(HW / nchunk) / R) rows of its float4
column (R and nchunk as gn_launch picks them), the CTA folds its R * cpg thread partials per group, and the last CTA merges the
nchunk chunk partials in double. The tests below bound every output element of gn_apply_kernel by

  f16 rounding of t  +  the apply pass's f32 roundings (harness.gn_ref's e32)  +  |gamma| (rstd dm + |xhat| dr)   (x 1.1 with SiLU)

where xhat = (x - mean) rstd, and dm, dr are the kernel's statistics errors (mean absolute, rstd relative), derived from its
summation order with u = 2^-24 and u_d = 2^-53, for a group of n = cpg HW elements with mean mu and standard deviation sigma:

  mean: each thread re-centres on its running mean after every merge, so what it adds are deviations from the mean, not
        values (the re-centring itself keeps its rounding exactly while |offset| <= |centre|, and within one rounding of a
        deviation otherwise): an f32 chain of L + 8 additions of terms whose mean magnitude is at most 3 sigma (Cauchy-Schwarz over
        the group; the running centre of a thread's first rows averages to within 2 sigma of the group over all its threads),
        i.e. 3 (L + 8) u sigma. The thread mean, the chunk mean and the final mean are each stored in f32: 3 u |mu|. The CTA
        fold (R cpg terms) and the chunk merge (nchunk terms) run in double: (R cpg + nchunk) u_d (|mu| + sigma).
          dm = 3 u |mu| + 3 (L + 8) u sigma + (R cpg + nchunk) u_d (|mu| + sigma)
  m2:   the thread's m2 is an f32 sum of non-negative terms (each block's two-pass m2 over its 6 or 8 rows, and one Chan cross
        term per block): at most L + 16 additions on any path, (L + 16) u relative, plus 3 u for the rounding of each deviation and its square. A mean stored in
        f32 moves the centred cross terms count * (mean - m)^2 of the next level by 2 u |mu| sqrt(n M2) at most, i.e. 2 u |mu| /
        sigma relative, at the fold and at the chunk merge. The chunk m2 is stored in f32 (u), the fold and merge add u_d terms.
          dv = (L + 20) u + 4 u |mu| / sigma + (R cpg + nchunk) u_d
        and rstd = 1 / sqrt(m2 / n + eps) carries half of it, plus one f32 rounding: dr = dv / 2 + u.
Both are first-order bounds; a factor 2 covers the second-order terms. Neither depends on where an outlier sits or on which
element a thread reads first: the adversarial inputs put outliers exactly there. The 4 u |mu| / sigma term comes from the f32
storage of the thread and chunk means: at |mean| / sigma = 1e4 it allows rstd to be off by ~2.4e-3 relative, so those cases
check that the kernel gets the mean's scale right, not that its variance is better than that (at 1e2 the term is 2.4e-5).
With sigma = 0 (a constant group) dm is 3 u |mu| and rstd = 1 / sqrt(eps) comes out within dr.

Shapes: the base UNet / ControlNet and refiner GroupNorms (block_program's resnet GroupNorms with their concatenation splits,
the transformers' GroupNorm, the output head) at the 1024^2 latent extents and the 1216x832 bucket with B = 2; the VAE
decoder's and encoder's GroupNorms at a 1024^2 image (B = 1, eps 1e-6); and, through the operator entry point, 1 to 5
channels per group and HW in {1, 3, R - 1}.
"""

import pytest
import torch

from sdxl_b200 import SDXL_BASE, SDXL_REFINER
from sdxl_b200 import _testing as T
from sdxl_b200.config import block_program
from harness import DEV, H11, H_SUB, U24

pytestmark = pytest.mark.gpu

UD = 2.0 ** -53


def cdiv(a, b):
    return (a + b - 1) // b


def gn_order(HW, C, G):
    """gn_launch's R and nchunk, and the resulting per-thread chain length L and CTA fold length R * cpg."""
    R = min(max(512 // (C // 4), 1), 16)
    nchunk = min(132, cdiv(HW, R))
    L = cdiv(cdiv(HW, nchunk), R)
    return R, nchunk, L, R * (C // G)


# ------------------------------------------------------------------------------------------------------------------------------
# reference and bound
# ------------------------------------------------------------------------------------------------------------------------------
def check_gn_stats(x1, x2, G, gam, bet, eps, silu, y, raw=None, y_lo=None, what="", slice_ch=64):
    """Every element of y (and raw, y_lo when given) against the float64 GroupNorm of cat(x1, x2) under the bound of the module
    docstring. Statistics are taken over whole groups in float64; the elementwise check runs over slices of slice_ch channels so
    that a 1024^2 x 256 input does not need its float64 copy all at once. Returns the worst err / bound."""
    B, HW, C1 = x1.shape
    C2 = 0 if x2 is None else x2.shape[2]
    C = C1 + C2
    cpg = C // G
    R, nchunk, L, F = gn_order(HW, C, G)
    n = cpg * HW

    def cols(c0, c1):   # channels [c0, c1) of cat(x1, x2) as float64
        parts = []
        if c0 < C1:
            parts.append(x1[:, :, c0:min(c1, C1)])
        if c1 > C1:
            parts.append(x2[:, :, max(c0, C1) - C1:c1 - C1])
        return torch.cat(parts, dim=2).double() if len(parts) > 1 else parts[0].double()

    mean = torch.empty(B, G, dtype=torch.float64, device=DEV)
    var = torch.empty_like(mean)
    gstep = max(1, slice_ch // cpg)
    for g0 in range(0, G, gstep):
        g1 = min(G, g0 + gstep)
        xg = cols(g0 * cpg, g1 * cpg).view(B, HW, g1 - g0, cpg)
        m = xg.mean(dim=(1, 3))
        mean[:, g0:g1] = m
        var[:, g0:g1] = ((xg - m[:, None, :, None]) ** 2).mean(dim=(1, 3))
        del xg
    rstd = 1.0 / torch.sqrt(var + eps)
    sd = var.sqrt()
    mu = mean.abs()
    dm = 2 * (3 * U24 * mu + 3 * (L + 8) * U24 * sd + (F + nchunk) * UD * (mu + sd))
    kappa = torch.where(sd > 0, mu / sd.clamp_min(1e-300), torch.zeros_like(mu))
    dv = (L + 20) * U24 + 4 * U24 * kappa + (F + nchunk) * UD
    dr = 2 * (dv / 2 + U24)
    worst = 0.0
    worst_lo = 0.0
    nbad = 0
    for c0 in range(0, C, gstep * cpg):
        c1 = min(C, c0 + gstep * cpg)
        x = cols(c0, c1)
        gidx = torch.arange(c0, c1, device=DEV) // cpg
        m, r = mean[:, gidx][:, None, :], rstd[:, gidx][:, None, :]
        ga, be = gam[c0:c1].double(), bet[c0:c1].double()
        xhat = (x - m) * r
        nrm = xhat * ga + be
        sc = r * ga
        e32 = 8 * U24 * (x.abs() * sc.abs() + m.abs() * sc.abs() + be.abs())
        es = ga.abs() * (r * dm[:, gidx][:, None, :] + xhat.abs() * dr[:, gidx][:, None, :])
        if silu:
            t = nrm * torch.sigmoid(nrm)
            tol = 1.1 * (e32 + es) + 2.0 ** -20 * (1 + nrm.abs()) * t.abs()
        else:
            t, tol = nrm, e32 + es
        got = y[:, :, c0:c1].double()
        err = (got - t).abs()
        bound = t.abs() * H11 + H_SUB + tol
        worst = max(worst, float((err / bound).max()))
        nbad += int((err > bound).sum())
        if raw is not None:
            assert torch.equal(raw[:, :, c0:c1].view(torch.int16), x.half().view(torch.int16)), f"{what}: raw != f16(cat(x1, x2))"
        if y_lo is not None:
            # y_lo = f16(t32 - y): its own rounding is 2^-22 |t| (see test_fused_paths_gpu.check_gn)
            err_lo = (got + y_lo[:, :, c0:c1].double() - t).abs()
            bound_lo = tol + 2.0 ** -22 * t.abs() + H_SUB
            worst_lo = max(worst_lo, float((err_lo / bound_lo).max()))
            nbad += int((err_lo > bound_lo).sum())
        del x, xhat, nrm, t, err, bound
    print(f"{what}: L={L} R*cpg={F} nchunk={nchunk}; worst err / bound {worst:.3f}"
          + (f", y + y_lo {worst_lo:.3f}" if y_lo is not None else ""))
    assert nbad == 0, f"{what}: {nbad} elements outside the bound (worst err / bound y {worst:.2f}, y + y_lo {worst_lo:.2f})"
    return max(worst, worst_lo)


# ------------------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------------------
def chain_first_pixel(HW, C):
    """A pixel that is the first row of some thread's chain other than chunk 0 / row 0: chunk 1's row 1 (or its row 0)."""
    R, nchunk, _, _ = gn_order(HW, C, 32)
    per = cdiv(HW, nchunk)
    return min(HW - 1, per + (1 if R > 1 else 0))


def make_input(kind, B, HW, C1, C2, G, gen):
    """cat sources x1 [B, HW, C1], x2 [B, HW, C2] (None when C2 = 0) of one of the statistics below, float32 on the device."""
    C = C1 + C2
    cpg = C // G

    def rn(*shape):
        return torch.randn(*shape, generator=gen, device=DEV)

    x = rn(B, HW, C)
    if kind == "normal":
        pass
    elif kind.startswith("mean"):                  # mean{k}_sd{s}: |mean| / sigma = k, sigma = s, sign alternating per group
        k, s = kind[4:].split("_sd")
        k, s = float(k), float(s)
        sign = torch.where(torch.arange(C, device=DEV) // cpg % 2 == 0, 1.0, -1.0)
        x = x * s + sign * k * s
    elif kind == "chan_offsets":                   # per-channel offsets inside every group, up to 10 sigma apart
        x += torch.linspace(-5.0, 5.0, cpg, device=DEV).repeat(G)
    elif kind == "cat_means":                      # the two sources at different means and scales
        if C2:
            x[:, :, :C1] = x[:, :, :C1] * 0.5 + 40.0
            x[:, :, C1:] = x[:, :, C1:] * 3.0 - 25.0
        else:
            x[:, :, :C // 2] += 40.0
    elif kind == "pivots":                         # the old kernel's four samples of each group at +-1e3 sigma
        c0 = torch.arange(G, device=DEV) * cpg
        for c in (c0, c0 + cpg // 2):
            for p, sgn in ((0, 1.0), (HW // 2, -1.0)):
                x[:, p, c] = sgn * 1e3
    elif kind == "px0":                            # one outlier pixel (every channel) at pixel 0
        x[:, 0, :] = 1e3
    elif kind == "pxmid":
        x[:, HW // 2, :] = -1e3
    elif kind == "px_pair800":                     # +800 at pixel 0 and HW / 2 in every channel
        x[:, 0, :] += 800.0
        x[:, HW // 2, :] += 800.0
    elif kind == "chain_first":                    # the first element of a thread's chain, and chunk 0's first, as outliers
        x[:, chain_first_pixel(HW, C), :] = 1e3
        x[:, 0, ::2] = -1e3
    elif kind == "const":                          # sigma = 0: eps decides rstd; one all-zero group
        x = (torch.arange(C, device=DEV) // cpg).float().mul(0.37).sub(3.0).expand(B, HW, C).contiguous()
        x[:, :, :cpg] = 0.0
    elif kind == "tiny_var":                       # sigma^2 comparable to eps, at an offset
        x = x * 3e-3 + 2.0
    elif kind == "adversarial":                    # what the plan shapes get: several of the above at once
        x += torch.linspace(-3.0, 3.0, cpg, device=DEV).repeat(G)
        x[:, :, C1:] += 7.0
        x[:, 0, :] = 1e3
        x[:, HW // 2, ::3] = -5e2
        x[:, chain_first_pixel(HW, C), 1::2] = 8e2
    else:
        raise ValueError(kind)
    x1 = x[:, :, :C1].contiguous()
    x2 = x[:, :, C1:].contiguous() if C2 else None
    return x1, x2


def affine(C, gen):
    gam = 1 + 0.1 * torch.randn(C, generator=gen, device=DEV)
    bet = 0.1 * torch.randn(C, generator=gen, device=DEV)
    return gam, bet


def run(x1, x2, G, gam, bet, eps, silu, scratch, lo=True):
    B, HW, C1 = x1.shape
    C = C1 + (0 if x2 is None else x2.shape[2])
    y = torch.full((B, HW, C), float("nan"), dtype=torch.float16, device=DEV)
    raw = torch.full_like(y, float("nan"))
    y_lo = torch.full_like(y, float("nan")) if lo else None
    T.group_norm(x1, x2, B, HW, G, gam, bet, eps, silu, y, raw, y_lo, scratch)
    return y, raw, y_lo


# ------------------------------------------------------------------------------------------------------------------------------
# the plans' GroupNorm forms
# ------------------------------------------------------------------------------------------------------------------------------
def unet_gn_forms(cfg, hws):
    """(C1, C2, HW) of every GroupNorm a UNet of cfg runs (resnet GroupNorms with their skip concatenation, the transformers'
    GroupNorm, the output head), with hws[level] pixels at each level."""
    ins, mid, outs = block_program(cfg)
    forms = set()
    level = 0
    for blk in ins[1:]:
        if blk.kind == "downsample":
            level += 1
            continue
        forms.add((blk.c_in, 0, hws[level]))
        forms.add((blk.c_out, 0, hws[level]))
    forms.add((mid.c_in, 0, hws[-1]))
    skips = [ins[0].c_out] + [b.c_out for b in ins[1:]]
    level = len(hws) - 1
    for blk in outs:
        c_skip = skips.pop()
        forms.add((blk.c_in - c_skip, c_skip, hws[level]))
        forms.add((blk.c_out, 0, hws[level]))
        if blk.kind.endswith("upsample"):
            level -= 1
    forms.add((cfg.model_channels, 0, hws[0]))
    return sorted(forms)


def latent_hws(h, w, n_levels):
    hw = []
    for _ in range(n_levels):
        hw.append(h * w)
        h, w = (h + 1) // 2, (w + 1) // 2
    return hw


BASE_FORMS = sorted(set(unet_gn_forms(SDXL_BASE, latent_hws(128, 128, 3)) + unet_gn_forms(SDXL_BASE, latent_hws(152, 104, 3))))
REFINER_FORMS = sorted(set(unet_gn_forms(SDXL_REFINER, latent_hws(128, 128, 4))
                           + unet_gn_forms(SDXL_REFINER, latent_hws(152, 104, 4))))


def test_plan_forms_cover_the_issue_shapes():
    """The enumerated forms include the decoder concatenations and the refiner's straddling 768 + 384."""
    base = {(c1, c2) for c1, c2, _ in BASE_FORMS}
    assert {(1280, 1280), (1280, 640), (640, 640), (640, 320), (320, 320)} <= base
    assert {c1 + c2 for c1, c2 in base} >= {320, 640, 960, 1280, 1920, 2560}
    assert {hw for _, _, hw in BASE_FORMS} >= {16384, 4096, 1024, 15808, 3952, 988}
    ref = {(c1, c2) for c1, c2, _ in REFINER_FORMS}
    assert (768, 384) in ref and (1536, 1536) in ref and (384, 0) in ref


@pytest.mark.parametrize("C1,C2,HW", BASE_FORMS)
@pytest.mark.parametrize("kind", ["normal", "adversarial"])
def test_base_unet_forms(C1, C2, HW, kind):
    gen = torch.Generator(device=DEV).manual_seed(C1 * 7 + C2 * 3 + HW)
    G, B = 32, 2
    x1, x2 = make_input(kind, B, HW, C1, C2, G, gen)
    gam, bet = affine(C1 + C2, gen)
    silu = kind == "normal"
    y, raw, y_lo = run(x1, x2, G, gam, bet, 1e-5, silu, T.gn_scratch(B, G))
    check_gn_stats(x1, x2, G, gam, bet, 1e-5, silu, y, raw, y_lo, f"base C={C1}+{C2} HW={HW} {kind}")


@pytest.mark.parametrize("C1,C2,HW", REFINER_FORMS)
@pytest.mark.parametrize("kind", ["normal", "adversarial"])
def test_refiner_forms(C1, C2, HW, kind):
    gen = torch.Generator(device=DEV).manual_seed(C1 * 5 + C2 * 11 + HW)
    G, B = 32, 2
    x1, x2 = make_input(kind, B, HW, C1, C2, G, gen)
    gam, bet = affine(C1 + C2, gen)
    y, raw, y_lo = run(x1, x2, G, gam, bet, 1e-5, True, T.gn_scratch(B, G))
    check_gn_stats(x1, x2, G, gam, bet, 1e-5, True, y, raw, y_lo, f"refiner C={C1}+{C2} HW={HW} {kind}")


# VAE decoder (and encoder, the same (C, HW) set in reverse) at a 1024^2 image: 512 at 128^2 .. 256^2 .. 512^2, 256 at 512^2 and
# 1024^2, 128 at 1024^2; the mid-block attention's GroupNorm is the 512 at 128^2 one without SiLU.
VAE_FORMS = [(512, 128 * 128), (512, 256 * 256), (512, 512 * 512), (256, 512 * 512), (256, 1024 * 1024), (128, 1024 * 1024),
             (128, 512 * 512), (256, 256 * 256)]


@pytest.mark.parametrize("C,HW", VAE_FORMS)
@pytest.mark.parametrize("kind", ["normal", "pivots", "px_pair800", "chain_first", "mean1000_sd1"])
def test_vae_forms(C, HW, kind):
    gen = torch.Generator(device=DEV).manual_seed(C + HW)
    G = 32
    x1, _ = make_input(kind, 1, HW, C, 0, G, gen)
    gam, bet = affine(C, gen)
    y, raw, _ = run(x1, None, G, gam, bet, 1e-6, True, T.gn_scratch(1, G), lo=False)
    check_gn_stats(x1, None, G, gam, bet, 1e-6, True, y, raw, None, f"vae C={C} HW={HW} {kind}")


# ------------------------------------------------------------------------------------------------------------------------------
# every statistic at the base decoder's 640 + 320 and the refiner's 768 + 384 concatenations (cpg = 30 and 36: group 21
# straddles the two sources in both) and at 320 + 0
# ------------------------------------------------------------------------------------------------------------------------------
STATS = ["normal", "chan_offsets", "cat_means", "pivots", "px0", "pxmid", "chain_first", "const", "tiny_var"] + \
        [f"mean{k:g}_sd{s:g}" for k in (1e2, 1e3, 1e4) for s in (1e-3, 1.0, 30.0)]


@pytest.mark.parametrize("kind", STATS)
@pytest.mark.parametrize("C1,C2,HW,silu", [(640, 320, 4096, True), (768, 384, 4096, False), (320, 0, 16384, True)])
def test_statistics(kind, C1, C2, HW, silu):
    gen = torch.Generator(device=DEV).manual_seed(sum(map(ord, kind)) * 1000 + C1 + C2)
    G, B = 32, 2
    x1, x2 = make_input(kind, B, HW, C1, C2, G, gen)
    gam, bet = affine(C1 + C2, gen)
    y, raw, y_lo = run(x1, x2, G, gam, bet, 1e-5, silu, T.gn_scratch(B, G))
    check_gn_stats(x1, x2, G, gam, bet, 1e-5, silu, y, raw, y_lo, f"C={C1}+{C2} HW={HW} {kind} silu={silu}")


# ------------------------------------------------------------------------------------------------------------------------------
# through the operator entry point: 1 to 5 channels per group, tiny HW
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,G", [(32, 32), (64, 32), (96, 32), (48, 12), (320, 64), (16, 16)])
@pytest.mark.parametrize("hw", ["1", "3", "R-1", "4096"])
@pytest.mark.parametrize("kind", ["normal", "chan_offsets"])
def test_op_channels_per_group(ctx, C, G, hw, kind):
    """cpg = 1 puts four groups in one float4 column; cpg = 2, 3, 5 put two. With per-channel offsets a statistic summed
    around another group's values is off by many sigma."""
    R = gn_order(1, C, G)[0]
    HW = {"1": 1, "3": 3, "R-1": max(R - 1, 1), "4096": 4096}[hw]
    gen = torch.Generator(device=DEV).manual_seed(C * 131 + G + HW)
    x1, _ = make_input(kind, 2, HW, C, 0, G, gen)
    if kind == "chan_offsets":
        x1 += 10.0 * torch.arange(C, device=DEV)     # every channel its own mean, 10 sigma apart
    gam, bet = affine(C, gen)
    y = ctx.group_norm(x1, None, gam, bet, n_group=G, silu=False)
    check_gn_stats(x1, None, G, gam, bet, 1e-5, False, y, what=f"op C={C} G={G} HW={HW} {kind}")


# ------------------------------------------------------------------------------------------------------------------------------
# invariance, bit for bit
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C1,C2,HW", [(640, 320, 4096), (1280, 0, 988), (128, 0, 512 * 512)])
def test_batch_run_and_scratch_invariance(C1, C2, HW):
    """Sample b of a B = 3 call equals the B = 1 call on that sample (chunking depends on HW only), a second run gives the same
    bits, and a scratch initialised for a larger (B, G) gives the same bits."""
    gen = torch.Generator(device=DEV).manual_seed(HW + C1)
    G = 32
    x1, x2 = make_input("adversarial", 3, HW, C1, C2, G, gen)
    gam, bet = affine(C1 + C2, gen)
    y3, _, lo3 = run(x1, x2, G, gam, bet, 1e-5, True, T.gn_scratch(3, G))
    y3b, _, lo3b = run(x1, x2, G, gam, bet, 1e-5, True, T.gn_scratch(3, G))
    assert torch.equal(y3.view(torch.int16), y3b.view(torch.int16)) and torch.equal(lo3.view(torch.int16), lo3b.view(torch.int16))
    big = T.gn_scratch(5, 64)
    for b in range(3):
        xb1 = x1[b:b + 1].contiguous()
        xb2 = None if x2 is None else x2[b:b + 1].contiguous()
        for scratch in (T.gn_scratch(1, G), big):
            y1, _, lo1 = run(xb1, xb2, G, gam, bet, 1e-5, True, scratch)
            assert torch.equal(y1.view(torch.int16), y3[b:b + 1].view(torch.int16)), f"sample {b}: B = 1 differs from B = 3"
            assert torch.equal(lo1.view(torch.int16), lo3[b:b + 1].view(torch.int16)), f"sample {b}: y_lo differs"
