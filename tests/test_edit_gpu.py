"""GPU tests of instruction-based editing (sdxl_unet_set_edit_image, DESIGN.md §21), tiny configs: the image-guidance forms of the three
step kernels against float64, edit forwards and CFG samples of every sampler family against the oracle chains (tests/edit_oracle.py),
the bit-exact properties (a zero source image, rewrites in place, detach and attach, no_cfg as a one-row chain, the plan builds), every
refusal, and bit-identity under fresh-memory fills, eager launches and no PDL (tests/edit_invariance_worker.py)."""
import ctypes as C
import math
from dataclasses import replace
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from sdxl_b200 import (TINY, TINY_EDIT, Conditioning, ControlNet, ControlNetConfig, Diffuser, IPAdapter, SdxlError, T2IAdapter, T2IAdapterConfig,
                       _lib, _testing, build_pack, synth_weights)
from sdxl_b200.engine import _cfg_struct
from sdxl_b200.ip_adapter import synth_ip_adapter
from sdxl_b200.schedulers import Schedule, alphas_cumprod
from oracle import unet_oracle as O
import deepcache_oracle as DO
import edit_oracle as EO
import prediction_oracle as PR
import scheduler2_oracle as S2
import scheduler_oracle as SO
from harness import first_difference, plan_builds, rel_err, tiny_conditioning

pytestmark = pytest.mark.gpu
KERNEL_TOL = 1e-6
STATS_TOL = 1e-7
FWD_TOL = 2e-3
SAMPLE_TOL = 5e-3
S_TEXT, S_IMG = 5.0, 1.5
ZSNR = alphas_cumprod(TINY_EDIT.n_steps, zero_terminal_snr=True)


def gen(seed):
    return torch.Generator().manual_seed(seed)


def _equal(got, want, what):
    assert torch.equal(got, want), f"{what}: {first_difference(want, got)}"


# ---- kernels ----------------------------------------------------------------------------------------------------------------------
def _rows(Bimg, Cc, HW, ld, seed):
    """NHWC eps rows [cond | img | uncond] of [3 * Bimg, HW, ld], correlated as a UNet's are, NaN in the pitch padding."""
    eps = torch.randn(3 * Bimg, HW, ld, generator=gen(seed))
    eps[Bimg:] = eps[Bimg:] * 0.8 + eps[:Bimg].repeat(2, 1, 1) * 0.5
    eps[:, :, Cc:] = float("nan")
    return eps


def _g64(eps, Bimg, Cc, factor=None):
    e = eps.double().permute(0, 2, 1)[:, :Cc]
    g = EO.combine(e[:Bimg], e[Bimg:2 * Bimg], e[2 * Bimg:], S_TEXT, S_IMG)
    return g if factor is None else g * factor.double().reshape(Bimg, 1, 1)


@pytest.mark.parametrize("HW", [37 * 5, 64 * 64, 128 * 128], ids=["one_block", "blocks", "max_blocks"])
def test_guidance_stats_img_kernel(ctx, HW):
    """The per-image rescale factor of the image-guidance combine against float64 on the kernel's own f32 combine."""
    Bimg, Cc, ld, phi = 2, 4, 8, 0.7
    eps = _rows(Bimg, Cc, HW, ld, HW)
    e = eps.permute(0, 2, 1)[:, :Cc]
    c, i, u = e[:Bimg], e[Bimg:2 * Bimg], e[2 * Bimg:]
    g = ((u + S_TEXT * (c - i)).double() + S_IMG * (i - u).double()).float()   # within an ulp of the kernel's fused f32
    want = phi * c.double().reshape(Bimg, -1).std(dim=1) / g.double().reshape(Bimg, -1).std(dim=1) + (1 - phi)
    want64 = phi * c.double().reshape(Bimg, -1).std(dim=1) / _g64(eps, Bimg, Cc).reshape(Bimg, -1).std(dim=1) + (1 - phi)
    scratch = _testing.guidance_stats_scratch(Bimg)
    runs = []
    for _ in range(2):
        f = torch.full((Bimg,), float("nan"), device="cuda")
        _testing.guidance_stats_img(eps.cuda(), ld, Bimg, Cc, HW, S_TEXT, S_IMG, phi, scratch, f)
        runs.append(f.cpu())
    err = float(((runs[0].double() - want64).abs() / want64).max())
    print(f"guidance_stats img HW={HW}: factors {runs[0].tolist()}, rel err vs float64 {err:.2e} "
          f"(vs the f32 combine {float(((runs[0].double() - want).abs() / want).max()):.2e})")
    assert err <= STATS_TOL
    _equal(runs[1], runs[0], "second run")


@pytest.mark.parametrize("v", [False, True], ids=["eps", "v"])
@pytest.mark.parametrize("rescale", [False, True], ids=["plain", "rescale"])
def test_cfg_ddim_img_kernel(ctx, v, rescale):
    Bimg, Cc, HW, ld = 2, 4, 37 * 5, 8
    eps = _rows(Bimg, Cc, HW, ld, 5)
    x0 = torch.randn(Bimg, Cc, HW, generator=gen(6))
    factor = torch.tensor([0.8, 1.3]) if rescale else None
    a, ap = float(ZSNR[749]), float(ZSNR[499])
    sa, s1, sap, s1p = (float(np.float32(math.sqrt(q))) for q in (a, 1 - a, ap, 1 - ap))
    g = _g64(eps, Bimg, Cc, factor)
    xd = x0.double()
    want = sap * (sa * xd - s1 * g) + s1p * (sa * g + s1 * xd) if v else sap * (xd - s1 * g) / sa + s1p * g
    x = x0.clone().cuda()
    _testing.cfg_ddim_img(eps.cuda(), ld, Bimg, Cc, HW, S_TEXT, S_IMG, sa, s1, sap, s1p, x, v, None if factor is None else factor.cuda())
    err = rel_err(x, want)
    print(f"cfg_ddim img v={v} rescale={rescale}: rel err vs float64 {err:.2e}")
    assert err <= KERNEL_TOL


@pytest.mark.parametrize("v", [False, True], ids=["eps", "v"])
@pytest.mark.parametrize("rescale", [False, True], ids=["plain", "rescale"])
@pytest.mark.parametrize("two_row", [False, True], ids=["one_row", "two_row"])
def test_guided_step_img_kernel(ctx, v, rescale, two_row):
    Bimg, Cc, HW, ld, sigma = 2, 4, 37 * 5, 8, 3.7
    eps = _rows(Bimg, Cc, HW, ld, 7)
    g0 = gen(8)
    xh0, hist0, h20, xs0, z = (torch.randn(Bimg, Cc, HW, generator=g0) for _ in range(5))
    factor = torch.tensor([1.2, 0.7]) if rescale else None
    g = _g64(eps, Bimg, Cc, factor)
    xd = xh0.double()
    if v:
        dx, de = (float(np.float32(q)) for q in (1 / (sigma * sigma + 1), sigma / math.sqrt(sigma * sigma + 1)))
        D = dx * xd - de * g
    else:
        D = xd - float(np.float32(sigma)) * g
    xh, hist, x_in = xh0.clone().cuda(), hist0.clone().cuda(), torch.empty_like(xh0).cuda()
    f = None if factor is None else factor.cuda()
    if two_row:
        coef, rows = (0.3, 0.4, 0.7, 0.2, -0.6, 0.9, 0.5), (0.1, 0.2, 0.3, 0.4, 0.5)
        cx, cs, cd, ch, ch2, cn, c_in = coef
        h1, h2, xs = hist0.double(), h20.double(), xs0.double()
        want = cx * xd + cs * xs + cd * D + ch * h1 + ch2 * h2 + cn * z.double()
        want_xs = 0.1 * xd + 0.2 * xs + 0.3 * D + 0.4 * h1 + 0.5 * h2
        h2d, xsd = h20.clone().cuda(), xs0.clone().cuda()
        _testing.guided_step_img(eps.cuda(), ld, Bimg, Cc, HW, S_TEXT, S_IMG, sigma, coef, xh, x_in, hist, True, z.cuda(), v=v, factor=f,
                                 rows=rows, h2=h2d, xs=xsd, write_xs=True, shift=True)
        err = max(rel_err(xsd, want_xs), rel_err(h2d, h1))
    else:
        coef = (0.3, 0.7, 0.2, 0.9, 0.5)
        cx, cd, ch, cn, c_in = coef
        want = cx * xd + cd * D + ch * hist0.double() + cn * z.double()
        _testing.guided_step_img(eps.cuda(), ld, Bimg, Cc, HW, S_TEXT, S_IMG, sigma, coef, xh, x_in, hist, True, z.cuda(), v=v, factor=f)
        err = 0.0
    err = max(err, rel_err(xh, want), rel_err(x_in, want * c_in), rel_err(hist, D))
    print(f"guided_step img v={v} rescale={rescale} two_row={two_row}: rel err vs float64 {err:.2e}")
    assert err <= KERNEL_TOL


# ---- engine ---------------------------------------------------------------------------------------------------------------------------
class Setup:
    def __init__(self, ctx):
        self.ctx = ctx
        self.w = synth_weights(TINY_EDIT, seed=0)
        self.wf = O.to_f32(self.w)
        self.d = Diffuser(ctx, TINY_EDIT, self.w)
        self.noise = torch.randn(2, 4, 16, 16, generator=gen(0))
        self.L = 0.5 * torch.randn(2, 4, 16, 16, generator=gen(1))
        self.cond = Conditioning(**tiny_conditioning(cfg=TINY_EDIT))
        self.oc = O.OracleConditioning(**tiny_conditioning(cfg=TINY_EDIT))
        self.loaded = np.array([self.d.alpha(i) for i in range(TINY_EDIT.n_steps)])


@pytest.fixture(scope="module")
def S(ctx):
    s = Setup(ctx)
    yield s
    s.d.close()


@pytest.fixture(autouse=True)
def detach(S):
    S.d.set_edit_image(S.L[:1], S_IMG)
    yield
    S.d.set_prediction()
    S.d.set_pag(None)
    S.d.set_deepcache(None)
    S.d.set_edit_image(None)


@pytest.mark.parametrize("n", [1, 2], ids=["n1", "nB"])
def test_forward_vs_oracle(S, n):
    """A direct forward of B = 2 rows: row r reads image r % n."""
    L = S.L[:n]
    S.d.set_edit_image(L, S_IMG)
    x = 0.7 * torch.randn(2, 4, 16, 16, generator=gen(2))
    ctx, y = S.oc.context_full, S.oc.channel_context
    out = S.d.unet_forward(x, [499], ctx, y).cpu()
    ref = O.unet_forward(TINY_EDIT, S.wf, x, torch.tensor([499]), ctx, y, O.Attach(concat=L))
    e = rel_err(out, ref)
    print(f"edit forward n={n}: rel err vs oracle {e:.2e}")
    assert e <= FWD_TOL


# every case samples a batch of 2 images: with one source image (row b reads image b % 1), and with two in "batch2_n2"
SAMPLE_CASES = ["ddim", "euler_ancestral/karras", "dpmpp_2m/karras", "unipc/karras", "heun_discrete/karras", "v_zsnr/trailing",
                "deepcache3", "batch2_n2"]


@pytest.mark.parametrize("case", SAMPLE_CASES)
def test_cfg_sample_vs_oracle(S, case):
    L, phi, v, alphas = S.L[:1], 0.0, False, S.loaded
    if case == "batch2_n2":
        L = S.L
    S.d.set_edit_image(L, S_IMG)
    cache = None
    if case == "deepcache3":
        S.d.set_deepcache(3, 2)
        cache = DO.Cache(TINY_EDIT, 3, 2)
    if case == "v_zsnr/trailing":
        phi, v, alphas = 0.7, True, ZSNR
        S.d.set_prediction("v_prediction", phi, zero_terminal_snr=True)
    f = EO.model_fn(TINY_EDIT, S.wf, S.oc, L, S_TEXT, S_IMG, phi, cache=cache)
    if case in ("ddim", "deepcache3", "batch2_n2"):
        got = S.d.sample_latent(S.cond, S_TEXT, 4, noise=S.noise).cpu()
        ref = PR.ddim(f, alphas, S.noise.double(), 4, v=False)
    else:
        sampler, spacing = ("dpmpp_2m", "trailing") if v else case.split("/")
        sch = Schedule(sampler, spacing, 4)
        k = sch.n_noise(False)
        steps = torch.randn(max(k, 1), 2, 4, 16, 16, generator=gen(9))
        got = S.d.sample_latent(S.cond, S_TEXT, 4, noise=S.noise, step_noise=steps if k else None, schedule=sch).cpu()
        t, sig = SO.schedule(spacing, 4, alphas)
        it = iter(steps.double())
        x0 = S.noise.double() * (sig[0] ** 2 + 1) ** 0.5
        if sampler in S2.SAMPLERS2:
            ref = S2.sample2(f, sampler, t, sig, x0, lambda: next(it), where=torch.where)
        else:
            ref = PR.sample(f, sampler, t, sig, x0, lambda: next(it), v=v)
    e = rel_err(got, ref)
    print(f"edit {case}: rel err vs oracle {e:.2e}")
    assert bool(torch.isfinite(got).all()) and e <= SAMPLE_TOL


def _dpm(S, **kw):
    return S.d.sample_latent(S.cond, S_TEXT, 4, noise=S.noise, schedule=Schedule("dpmpp_2m", "karras", 4), **kw).cpu()


def test_zero_image_reduces_to_text_guidance(S):
    """With L = 0 the img and uncond rows are the same forward bit for bit, so s_img * (i - u) is zero and g = u + s (c - u) whatever
    s_img is."""
    zero = torch.zeros(1, 4, 16, 16)
    S.d.set_edit_image(zero, 1.5)
    a = _dpm(S)
    S.d.set_edit_image(zero, 7.0)
    _equal(_dpm(S), a, "L = 0, s_img 7 vs 1.5")


def test_rewrite_detach_and_plan_builds(S):
    S.d.set_edit_image(S.L[1:], S_IMG)
    fresh = _dpm(S)
    b0 = plan_builds(S.d)
    S.d.set_edit_image(S.L[:1], 3.0)
    _dpm(S)
    S.d.set_edit_image(S.L[1:], S_IMG)   # the same shape: rewritten in place, plan and graph kept
    _equal(_dpm(S), fresh, "rewrite in place")
    assert plan_builds(S.d) == b0
    S.d.set_edit_image(S.L[1:], 2.5)     # s_img only
    moved = _dpm(S)
    assert plan_builds(S.d) == b0 and not torch.equal(moved, fresh)
    S.d.set_edit_image(None)
    S.d.set_edit_image(S.L[1:], S_IMG)
    _equal(_dpm(S), fresh, "detach then attach")
    assert plan_builds(S.d) == b0 + 1
    S.d.set_edit_image(S.L, S_IMG)       # a new n: a new plan
    _dpm(S)
    assert plan_builds(S.d) == b0 + 2


def test_no_cfg_is_a_one_row_forward_chain(S):
    """The no_cfg Euler loop against the same loop driven by hand: direct forwards of the two rows, each reading its image, and the
    step kernel with the coefficients the engine takes."""
    S.d.set_edit_image(S.L, S_IMG)
    sch = Schedule("euler", "leading", 4, no_cfg=True)
    got = S.d.sample_latent(S.cond, S_TEXT, 4, noise=S.noise, schedule=sch).cpu()
    t, sig = SO.schedule("leading", 4, S.loaded)
    z = S.noise.reshape(2, 4, 256).cuda()
    xh, x_in, hist = torch.zeros_like(z), torch.empty_like(z), torch.zeros_like(z)
    s0 = float(sig[0])
    _testing.guided_step(None, 4, 2, 4, 256, False, False, 0.0, 0.0, 0.0, (0.0, 0.0, 0.0, math.sqrt(s0 * s0 + 1), 1 / math.sqrt(s0 * s0 + 1)),
                         xh, x_in, z=z)
    ctx, y = S.oc.context_full, S.oc.channel_context
    for k in range(4):
        st = _testing.step_stages(S.loaded, sch.to_struct(), k, t, sig, min(k, 2))[0]
        eps = S.d.unet_forward(x_in.reshape(2, 4, 16, 16), [st["t"]], ctx if k == 0 else None, y if k == 0 else None)
        rows = eps.permute(0, 2, 3, 1).reshape(2, 256, 4).contiguous()
        _testing.guided_step(rows, 4, 2, 4, 256, False, False, 0.0, 0.0, st["sigma"], (st["cx"], st["cd"], st["ch"], st["cn"], st["c_in"]),
                             xh, x_in, hist, int(st["hist"]) % 2 == 1)
    _equal(got, xh.reshape(2, 4, 16, 16).cpu(), "no_cfg vs hand-driven chain")


def _code(fn, code, what):
    with pytest.raises(SdxlError, match=rf"\({code}\)"):
        fn()
    print(f"{what}: refused with {code}")


def test_refusals_leave_the_previous_state(S, ctx):
    want = _dpm(S)
    d = S.d
    keep = torch.zeros(1, 4, 16, 16)

    def raw(**kw):   # sdxl_unet_set_edit_image on a host image, fields overridden by kw
        s = _lib.EditImage()
        s.latent, s.on_host, s.n, s.height, s.width, s.image_guidance = keep.data_ptr(), 1, 1, 128, 128, 1.5
        for k, v in kw.items():
            setattr(s, k, v)
        d.ctx.call("sdxl_unet_set_edit_image", d.ctx.lib.sdxl_unet_set_edit_image, d.h, C.byref(s))
    _code(lambda: raw(latent=None), 5711, "null latent")
    _code(lambda: raw(n=0), 5712, "n = 0")
    _code(lambda: raw(height=12), 5713, "height 12")
    _code(lambda: raw(image_guidance=float("nan")), 5714, "image_guidance NaN")
    _code(lambda: raw(n=1 << 28), 5715, "a 1 TiB image buffer")   # cudaMalloc refuses it; nothing is copied
    _equal(_dpm(S), want, "after set_edit_image refusals")
    # the forward's and the sampler's
    d.set_edit_image(torch.zeros(1, 4, 8, 8), S_IMG)
    _code(lambda: _dpm(S), 5721, "image of another size")
    d.set_edit_image(torch.zeros(3, 4, 16, 16), S_IMG)
    _code(lambda: _dpm(S), 5722, "batch not a multiple of n")
    d.set_edit_image(None)
    _code(lambda: _dpm(S), 5720, "nothing attached")
    _code(lambda: d.unet_forward(S.noise, [499], S.oc.context_full, S.oc.channel_context), 5720, "forward, nothing attached")
    d.set_edit_image(S.L[:1], S_IMG)
    d.set_pag("mid", 3.0)
    _code(lambda: _dpm(S), 5723, "PAG")
    d.set_pag(None)
    t2i = T2IAdapter(ctx, T2IAdapterConfig(TINY_EDIT), synth_weights(T2IAdapterConfig(TINY_EDIT), seed=1))
    d.set_t2i_adapters([(t2i, torch.rand(1, 3, 128, 128, generator=gen(2)), 1.5)])
    _code(lambda: _dpm(S), 5725, "T2I-Adapter")
    d.set_t2i_adapters([])
    t2i.close()
    ip = IPAdapter(ctx, TINY_EDIT, 32, synth_ip_adapter(TINY_EDIT, 32, seed=3))
    d.set_image_prompt(ip, torch.randn(1, 1, 32, generator=gen(2)), 0.8)
    _code(lambda: _dpm(S), 5726, "image prompt")
    d.set_image_prompt(None)
    ip.close()
    # a ControlNet of a plain 8-channel cfg passes the cfg match (edit_layout is not compared) and is refused at the forward
    ncfg8 = ControlNetConfig(replace(TINY, in_channels=8), hint_block_channels=(8, 16, 24, 32))
    net = ControlNet(ctx, ncfg8, synth_weights(ncfg8, seed=7))
    d.set_controls([(net, torch.rand(1, 3, 128, 128, generator=gen(4)), 0.8)])
    _code(lambda: _dpm(S), 5724, "ControlNet")
    d.set_controls([])
    net.close()
    mask = torch.ones(2, 4, 16, 16, dtype=torch.bool)
    _code(lambda: d.sample_latent_with_inpainting(S.cond, S_TEXT, 4, S.noise, mask, init_noise=S.noise), 5727, "inpaint_ref (DDIM)")
    _code(lambda: d.sample_latent_with_inpainting(S.cond, S_TEXT, 4, S.noise, mask, init_noise=S.noise, schedule=Schedule("euler", "karras", 4)),
          5727, "inpaint_ref (scheduled)")
    _equal(_dpm(S), want, "after the refusals")
    # a ControlNet cannot be built on an edit cfg; the cfg rules
    ncfg = ControlNetConfig(TINY_EDIT, hint_block_channels=(8, 16, 24, 32))
    _code(lambda: ControlNet(ctx, ncfg, synth_weights(ControlNetConfig(TINY, hint_block_channels=(8, 16, 24, 32)), seed=7)), 5703, "ControlNet")
    for cfg, code in ((replace(TINY_EDIT, in_channels=9), 5701), (replace(TINY_EDIT, is_refiner=True), 5702)):
        _code(lambda: Diffuser(ctx, cfg, synth_weights(replace(cfg, is_edit=False, is_refiner=False), seed=0)), code, f"cfg {code}")
    cs = _cfg_struct(TINY_EDIT)
    cs.edit_layout = 2
    pack, h = build_pack(synth_weights(TINY_EDIT, seed=0)), C.c_void_p()
    _code(lambda: ctx.call("sdxl_unet_load", ctx.lib.sdxl_unet_load, ctx.h, C.byref(cs), pack.data_ptr(), pack.numel(), 0, C.byref(h)), 5700,
          "edit_layout = 2")
    plain = Diffuser(ctx, TINY, synth_weights(TINY, seed=0))
    _code(lambda: plain.set_edit_image(S.L[:1]), 5710, "a UNet without the edit layout")
    plain.close()


# ---- the sample() front end ----------------------------------------------------------------------------------------------------------
MINI = os.path.join(os.path.dirname(__file__), "golden", "mini_bpe")


def test_pipeline_sample(ctx):
    """sample(..., edit_image=) with tiny text encoders, VAE and edit UNet: the source latent prepare_edit_latent makes is the oracle's
    unscaled posterior mean (quant_conv's mean channels, no scaling factor); the image equals, bit for bit, the library calls it stands
    for (set_edit_image, sample_latent, latent_to_image), with CFG and, for image_guidance < 1 and guidance <= 1, as diffusers switches
    CFG off, with the no_cfg Euler loop on the reference spacing; the image is detached after each call."""
    import torch.nn.functional as F
    from oracle import vae_oracle as VO
    from sdxl_b200 import TINY_CLIP, TINY_OPEN_CLIP, TINY_VAE, ClipTextEncoder, Embedder, LatentDecoder, OpenClipTokenizer, UNetConfig, sample
    from sdxl_b200.pipeline import prepare_edit_latent
    ca, cb = TINY_CLIP, TINY_OPEN_CLIP
    ucfg = UNetConfig(adm_in_channels=cb.embed_dim + 6 * 256, model_channels=64, channel_mults=(1, 2, 4), transformer_depths=(0, 1, 1),
                      context_dim=ca.n_state + cb.n_state, in_channels=8, is_edit=True)
    wa, wb, wu, wv = (synth_weights(cfg, seed=s) for cfg, s in ((ca, 1), (cb, 2), (ucfg, 3), (TINY_VAE, 0)))
    tok = OpenClipTokenizer(os.path.join(MINI, "mini_merges.txt"), os.path.join(MINI, "mini_vocab.txt"))
    emb = Embedder(ctx, ClipTextEncoder(ctx, ca, wa), ClipTextEncoder(ctx, cb, wb), tok, tok)
    dif = Diffuser(ctx, ucfg, wu)
    vae = LatentDecoder(ctx, TINY_VAE, wv)
    text = "make it winter"
    rgb = torch.randint(0, 256, (1, 32, 32, 3), dtype=torch.uint8, generator=gen(1))
    noise = torch.randn(1, 4, 8, 8, generator=gen(0))
    wvf = O.to_f32(wv)
    image = rgb.permute(0, 3, 1, 2).float() / 255.0 * 2.0 - 1.0
    mean = F.conv2d(VO.encoder_forward(TINY_VAE, wvf, image), wvf["quant_conv/weight"], wvf["quant_conv/bias"])[:, :4]
    L = prepare_edit_latent(vae, rgb)
    e = rel_err(L, mean)
    print(f"prepare_edit_latent: rel err vs the oracle's unscaled posterior mean {e:.2e}")
    assert e <= FWD_TOL
    cond = emb.text_to_conditioning(text, [32, 32], [0, 0], [32, 32])
    cond.resolution = (8 * L.shape[2], 8 * L.shape[3])   # the latent follows the source image's (TINY_VAE downsamples by 4)
    for guidance, s_img in ((5.0, 1.5), (5.0, 0.9), (1.0, 1.5)):
        img = sample(emb, dif, vae, text, guidance=guidance, n_steps=4, noise=noise, edit_image=rgb, image_guidance=s_img)
        with pytest.raises(SdxlError, match=r"\(5720\)"):   # detached after the call
            dif.sample_latent(cond, guidance, 4, noise=noise)
        dif.set_edit_image(L, s_img)
        sch = None if guidance > 1 and s_img >= 1 else Schedule("euler", "reference", 4, no_cfg=True)
        lat = dif.sample_latent(cond, guidance, 4, noise=noise, schedule=sch)
        dif.set_edit_image(None)
        _equal(img.cpu(), vae.latent_to_image(lat).cpu(), f"sample() guidance {guidance} image_guidance {s_img}")
    for o in (emb.clip, emb.open_clip, dif, vae):
        o.close()


WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "edit_invariance_worker.py")
SWITCHES = ("SDXL_B200_FILL", "SDXL_B200_NO_GRAPH", "SDXL_B200_NO_PDL")
CONFIGS = {"base": {}, "nan": {"SDXL_B200_FILL": "0xff"}, "big": {"SDXL_B200_FILL": "0x7b"}, "eager": {"SDXL_B200_NO_GRAPH": "1"},
           "nopdl": {"SDXL_B200_NO_PDL": "1"}}


def _run_worker(name, out_dir):
    env = {k: v for k, v in os.environ.items() if k not in SWITCHES}
    env.update(CONFIGS[name])
    out = os.path.join(out_dir, f"{name}.pt")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [WORKER, out]
    p = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, f"worker [{name}] exited with {p.returncode}:\n{p.stderr[-6000:]}"
    return torch.load(out, weights_only=True)


def test_fills_graphs_and_pdl_change_nothing(tmp_path):
    base = _run_worker("base", str(tmp_path))
    assert all(bool(torch.isfinite(v).all()) for v in base.values())
    for name in ("nan", "big", "eager", "nopdl"):
        got = _run_worker(name, str(tmp_path))
        for k in base:
            _equal(got[k], base[k], f"{name}: {k}")
