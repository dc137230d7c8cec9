"""GPU tests of the v prediction, zero-terminal SNR and guidance rescale (sdxl_unet_set_prediction, DESIGN.md §18), tiny configs: the
statistics kernel and both step kernels against float64, the epsilon setting and a detach bit-identical to never attaching, v samples
on the zero-SNR table against the oracle chains (tests/prediction_oracle.py), no_cfg and the refiner ignoring phi, the hand-driven
loop, the plan builds, the refusals, the pipeline's per-call phi, from_diffusers_dir's scheduler config, DeepCache with v, and
bit-identity under fresh-memory fills, eager launches and no PDL (tests/prediction_invariance_worker.py, one subprocess per
configuration)."""
import ctypes as C
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from sdxl_b200 import TINY, TINY_INPAINT, TINY_REFINER, Conditioning, Diffuser, SdxlError, _lib, _testing, pag_layer_mask, synth_weights
from sdxl_b200.schedulers import Schedule, alphas_cumprod
from oracle import unet_oracle as O
import deepcache_oracle as DO
import pag_oracle as PO
import prediction_oracle as PR
import scheduler_oracle as SO
from harness import first_difference, plan_builds, rel_err, tiny_conditioning

pytestmark = pytest.mark.gpu
SAMPLE_TOL = 5e-3
KERNEL_TOL = 1e-6
ZSNR = alphas_cumprod(TINY.n_steps, zero_terminal_snr=True)


def gen(seed):
    return torch.Generator().manual_seed(seed)


def _equal(got, want, what):
    assert torch.equal(got, want), f"{what}: {first_difference(want, got)}"


# ---- kernels ----------------------------------------------------------------------------------------------------------------------
def _rows(groups, Bimg, Cc, HW, ld, seed, mean=0.0):
    """NHWC eps rows [groups * Bimg, HW, ld] with NaN in the pitch padding; mean: added to every row."""
    g = gen(seed)
    eps = torch.randn(groups * Bimg, HW, ld, generator=g)
    eps[Bimg:] = eps[Bimg:] * 0.8 + eps[:Bimg].repeat(groups - 1, 1, 1) * 0.5   # correlated rows, as a UNet's are
    eps = eps + mean
    eps[:, :, Cc:] = float("nan")
    return eps


def _f32_guided(eps, Bimg, Cc, use_pag, s, p_t):
    """(c, g) NCHW f32 as the kernels compute them: u + (c - u) * s and g + p_t * (c - ptb), each one fused multiply-add."""
    e = eps.permute(0, 2, 1)[:, :Cc]
    c, u = e[:Bimg], e[Bimg:2 * Bimg]
    g = ((c - u).double() * s + u.double()).float()
    if use_pag:
        g = ((c - e[2 * Bimg:3 * Bimg]).double() * p_t + g.double()).float()
    return c, g


@pytest.mark.parametrize("use_pag", [False, True])
@pytest.mark.parametrize("HW, mean", [(37 * 5, 0.0), (64 * 64, 0.0), (128 * 128, 0.0), (64 * 64, 1e3)],
                         ids=["one_block", "blocks", "max_blocks", "mean_1e3"])
def test_guidance_stats_kernel(ctx, use_pag, HW, mean):
    """The per-image factor against float64 on the kernels' own f32 values, one block and several per image, an input whose mean is
    a thousand times its spread, and two runs on one scratch (the arrival counters reset) giving the same bits."""
    Bimg, Cc, ld, s, p_t, phi = 2, 4, 8, 7.5, 2.25, 0.7
    eps = _rows(3 if use_pag else 2, Bimg, Cc, HW, ld, HW + use_pag, mean)
    c, g = _f32_guided(eps, Bimg, Cc, use_pag, s, p_t)
    sc = c.double().reshape(Bimg, -1).std(dim=1)
    sg = g.double().reshape(Bimg, -1).std(dim=1)
    want = phi * sc / sg + (1 - phi)
    scratch = _testing.guidance_stats_scratch(Bimg)
    runs = []
    for _ in range(2):
        f = torch.full((Bimg,), float("nan"), device="cuda")
        _testing.guidance_stats(eps.cuda(), ld, Bimg, Cc, HW, use_pag, s, p_t, phi, scratch, f)
        runs.append(f.cpu())
    e = float(((runs[0].double() - want).abs() / want).max())
    print(f"guidance_stats pag={use_pag} HW={HW} mean={mean:g}: factors {runs[0].tolist()}, rel err vs float64 {e:.2e}")
    assert e <= KERNEL_TOL
    _equal(runs[1], runs[0], "second run")
    flat = torch.zeros(2 * Bimg, HW, ld)   # std(g) = 0: the factor is 1
    f = torch.empty(Bimg, device="cuda")
    _testing.guidance_stats(flat.cuda(), ld, Bimg, Cc, HW, False, s, p_t, phi, scratch, f)
    assert torch.equal(f.cpu(), torch.ones(Bimg))


def _factor_ref(factor, Bimg):
    return factor.double().reshape(Bimg, 1, 1)


@pytest.mark.parametrize("v", [False, True], ids=["eps", "v"])
@pytest.mark.parametrize("rescale", [False, True], ids=["plain", "rescale"])
@pytest.mark.parametrize("use_pag", [False, True], ids=["cfg", "pag"])
def test_cfg_ddim_kernel(ctx, v, rescale, use_pag):
    Bimg, Cc, HW, ld, s, p_t = 2, 4, 37 * 5, 8, 7.5, 2.25
    eps = _rows(3 if use_pag else 2, Bimg, Cc, HW, ld, 5)
    x0 = torch.randn(Bimg, Cc, HW, generator=gen(6))
    factor = torch.tensor([0.8, 1.3]) if rescale else None
    a, ap = float(ZSNR[749]), float(ZSNR[499])
    sa, s1, sap, s1p = (float(np.float32(math.sqrt(q))) for q in (a, 1 - a, ap, 1 - ap))
    e = eps.double().permute(0, 2, 1)[:, :Cc]
    g = e[Bimg:2 * Bimg] + (e[:Bimg] - e[Bimg:2 * Bimg]) * s
    if use_pag:
        g = g + p_t * (e[:Bimg] - e[2 * Bimg:])
    if rescale:
        g = g * _factor_ref(factor, Bimg)
    xd = x0.double()
    if v:
        want = sap * (sa * xd - s1 * g) + s1p * (sa * g + s1 * xd)
    else:
        want = sap * (xd - s1 * g) / sa + s1p * g
    x = x0.clone().cuda()
    _testing.cfg_ddim_pred(eps.cuda(), ld, Bimg, Cc, HW, True, s, sa, s1, sap, s1p, x, use_pag, p_t, v, None if factor is None else factor.cuda())
    err = rel_err(x, want)
    print(f"cfg_ddim v={v} rescale={rescale} pag={use_pag}: rel err vs float64 {err:.2e}")
    assert err <= KERNEL_TOL


@pytest.mark.parametrize("v", [False, True], ids=["eps", "v"])
@pytest.mark.parametrize("rescale", [False, True], ids=["plain", "rescale"])
@pytest.mark.parametrize("use_pag, inpaint", [(False, False), (True, False), (False, True)], ids=["cfg", "pag", "inpaint"])
def test_guided_step_kernel(ctx, v, rescale, use_pag, inpaint):
    Bimg, Cc, HW, ld, s, p_t, sigma = 2, 4, 37 * 5, 8, 7.5, 2.25, 3.7
    coef = (0.3, 0.7, 0.2, 0.9, 0.5)
    eps = _rows(3 if use_pag else 2, Bimg, Cc, HW, ld, 7)
    g0 = gen(8)
    xh0, hist0, z, zb, ref = (torch.randn(Bimg, Cc, HW, generator=g0) for _ in range(5))
    mask = (torch.rand(Bimg, Cc, HW, generator=g0) < 0.5).to(torch.uint8)
    factor = torch.tensor([1.2, 0.7]) if rescale else None
    e = eps.double().permute(0, 2, 1)[:, :Cc]
    g = e[Bimg:2 * Bimg] + (e[:Bimg] - e[Bimg:2 * Bimg]) * s
    if use_pag:
        g = g + p_t * (e[:Bimg] - e[2 * Bimg:])
    if rescale:
        g = g * _factor_ref(factor, Bimg)
    xd = xh0.double()
    if v:
        dx, de = (float(np.float32(q)) for q in (1 / (sigma * sigma + 1), sigma / math.sqrt(sigma * sigma + 1)))
        D = dx * xd - de * g
    else:
        D = xd - float(np.float32(sigma)) * g
    cx, cd, ch, cn, c_in = coef
    want = cx * xd + cd * D + ch * hist0.double() + cn * z.double()
    if inpaint:
        want = torch.where(mask.bool(), want, ref.double() + 1.5 * zb.double())
    xh, hist, x_in = xh0.clone().cuda(), hist0.clone().cuda(), torch.empty_like(xh0).cuda()
    _testing.guided_step_pred(eps.cuda(), ld, Bimg, Cc, HW, True, use_pag, s, p_t, sigma, coef, xh, x_in, hist, True, z.cuda(),
                              zb.cuda() if inpaint else None, mask=mask.cuda() if inpaint else None, ref=ref.cuda() if inpaint else None,
                              sigma_blend=1.5, v=v, factor=None if factor is None else factor.cuda())
    err = max(rel_err(xh, want), rel_err(x_in, want * c_in), rel_err(hist, D))
    print(f"guided_step v={v} rescale={rescale} pag={use_pag} inpaint={inpaint}: rel err vs float64 {err:.2e}")
    assert err <= KERNEL_TOL


# ---- engine ---------------------------------------------------------------------------------------------------------------------------
class Setup:
    def __init__(self, ctx):
        self.ctx = ctx
        self.w = synth_weights(TINY, seed=0)
        self.wf = O.to_f32(self.w)
        self.d = Diffuser(ctx, TINY, self.w)
        self.noise = torch.randn(2, 4, 16, 16, generator=gen(0))
        self.cond = Conditioning(**tiny_conditioning(refiner=True))
        self.oc = O.OracleConditioning(**tiny_conditioning(refiner=True))
        self.loaded = np.array([self.d.alpha(i) for i in range(TINY.n_steps)])


@pytest.fixture(scope="module")
def S(ctx):
    s = Setup(ctx)
    yield s
    s.d.close()


@pytest.fixture(autouse=True)
def detach(S):
    yield
    S.d.set_prediction()
    S.d.set_pag(None)
    S.d.set_deepcache(None)


def _raw(d, type_, phi, table=None):
    """sdxl_unet_set_prediction with a non-null struct (the C ABI, not Diffuser.set_prediction's detach)."""
    s = _lib.Prediction()
    s.type, s.guidance_rescale = type_, phi
    keep = None
    if table is not None:
        keep = np.ascontiguousarray(table, dtype=np.float64)
        s.n_alphas, s.alphas_cumprod_host = keep.size, keep.ctypes.data
    return d.ctx.lib.sdxl_unet_set_prediction(d.h, C.byref(s))


SAMPLE_CASES = ["ddim", "inpainting", "pag"] + [f"{s}/{m}" for s in ("euler", "euler_ancestral", "dpmpp_2m", "lcm") for m in ("cfg", "no_cfg")]


def _sample(S, case):
    if case == "ddim":
        return S.d.sample_latent(S.cond, 7.5, 4, noise=S.noise).cpu()
    if case == "pag":
        return S.d.sample_latent(S.cond, 7.5, 4, noise=S.noise, schedule=Schedule("dpmpp_2m", "karras", 4)).cpu()
    if case == "inpainting":
        mask = torch.zeros(2, 4, 16, 16, dtype=torch.bool)
        mask[:, :, :6] = True
        ref = torch.randn(2, 4, 16, 16, generator=gen(3))
        return S.d.sample_latent_with_inpainting(S.cond, 7.5, 4, ref, mask, init_noise=S.noise, seed=4).cpu()
    sampler, mode = case.split("/")
    sch = Schedule(sampler, "karras" if sampler != "lcm" else "lcm", 4, no_cfg=mode == "no_cfg")
    return S.d.sample_latent(S.cond, 7.5, 4, noise=S.noise, seed=5, schedule=sch).cpu()


# ---- 1. the epsilon setting and a detach are the plain calls ------------------------------------------------------------------------
@pytest.mark.parametrize("case", SAMPLE_CASES)
def test_epsilon_and_detach_are_bit_identical(S, case):
    if case == "pag":
        S.d.set_pag("mid", 3.0)
    plain = _sample(S, case)
    assert _raw(S.d, 0, 0.0) == 0
    _equal(_sample(S, case), plain, f"{case}, epsilon phi 0")
    assert _raw(S.d, 0, 0.0, S.loaded) == 0   # the loaded table passed back in
    _equal(_sample(S, case), plain, f"{case}, epsilon phi 0, the loaded table")
    S.d.set_prediction("v_prediction", 0.7, zero_terminal_snr=True)
    moved = _sample(S, case)
    S.d.set_prediction()
    _equal(_sample(S, case), plain, f"{case}, detached")
    assert not torch.equal(moved, plain)


def test_epsilon_and_detach_inpainting_unet_and_refiner(ctx):
    w = synth_weights(TINY_INPAINT, seed=0)
    d = Diffuser(ctx, TINY_INPAINT, w)
    d.set_inpaint_condition(torch.rand(1, 5, 16, 16, generator=gen(6)))
    cond, noise = Conditioning(**tiny_conditioning(refiner=True)), torch.randn(2, 4, 16, 16, generator=gen(0))
    plain = d.sample_latent(cond, 7.5, 4, noise=noise).cpu()
    assert _raw(d, 0, 0.0) == 0
    _equal(d.sample_latent(cond, 7.5, 4, noise=noise).cpu(), plain, "inpainting UNet, epsilon phi 0")
    d.set_prediction("v_prediction", 0.5, zero_terminal_snr=True)
    d.set_prediction()
    _equal(d.sample_latent(cond, 7.5, 4, noise=noise).cpu(), plain, "inpainting UNet, detached")
    d.close()
    r = Diffuser(ctx, TINY_REFINER, synth_weights(TINY_REFINER, seed=1))
    latent, rn = torch.randn(2, 4, 16, 16, generator=gen(5)), torch.randn(2, 4, 16, 16, generator=gen(7))
    plain = r.refine_latent(latent, cond, 7.5, 800, 50, noise=rn).cpu()
    assert _raw(r, 0, 0.0) == 0
    _equal(r.refine_latent(latent, cond, 7.5, 800, 50, noise=rn).cpu(), plain, "refiner, epsilon phi 0")
    r.set_prediction("v_prediction", 0.5)
    r.set_prediction()
    _equal(r.refine_latent(latent, cond, 7.5, 800, 50, noise=rn).cpu(), plain, "refiner, detached")
    r.close()


# ---- 2. v on the zero-SNR table against the oracle chains ----------------------------------------------------------------------------
V_CASES = [("ddim", 0.0), ("ddim", 0.7), ("euler_ancestral/trailing", 0.7), ("dpmpp_2m/trailing", 0.7), ("lcm/lcm", 0.7), ("pag", 0.7)]


@pytest.mark.parametrize("case, phi", V_CASES, ids=[f"{c}-phi{p}" for c, p in V_CASES])
def test_v_zero_snr_vs_oracle(S, case, phi):
    """Each of the batch's two images has its own rescale factor: the oracle's std is per image. The schedules are the ones v models
    are sampled with (trailing or LCM spacing): a 4-step Karras schedule from sigma = 4096 jumps to 444 and 17 and amplifies the
    forwards' f16 error about four times as much (6e-3 here, DESIGN.md §18)."""
    att = None
    if case == "pag":
        S.d.set_pag("mid", 3.0)
        att = PO.attach(TINY, PO.paths_of_mask(TINY, pag_layer_mask(TINY, "mid")), 3.0)
    S.d.set_prediction("v_prediction", phi, zero_terminal_snr=True)
    f = PR.model_fn(TINY, S.wf, S.oc, 7.5, phi, att)
    if case == "ddim":
        got = S.d.sample_latent(S.cond, 7.5, 4, noise=S.noise).cpu()
        ref = PR.ddim(f, ZSNR, S.noise.double(), 4)
    else:
        sampler, spacing = ("dpmpp_2m", "trailing") if case == "pag" else case.split("/")
        sch = Schedule(sampler, spacing, 4)
        steps = torch.randn(max(sch.n_noise(False), 1), 2, 4, 16, 16, generator=gen(9))
        got = S.d.sample_latent(S.cond, 7.5, 4, noise=S.noise, step_noise=steps if sch.n_noise(False) else None, schedule=sch).cpu()
        t, sig = SO.schedule(spacing, 4, ZSNR)
        it = iter(steps.double())
        ref = PR.sample(f, sampler, t, sig, S.noise.double() * (sig[0] ** 2 + 1) ** 0.5, lambda: next(it))
    e = rel_err(got, ref)
    print(f"v zero-SNR {case} phi={phi}: rel err vs oracle {e:.2e}")
    assert bool(torch.isfinite(got).all()) and e <= SAMPLE_TOL


# ---- 3. no_cfg and the refiner ignore phi -----------------------------------------------------------------------------------------------
def test_no_cfg_and_refiner_ignore_rescale(S, ctx):
    sch = Schedule("euler", "trailing", 4, no_cfg=True)
    S.d.set_prediction("v_prediction", 0.0, zero_terminal_snr=True)
    want = S.d.sample_latent(S.cond, 7.5, 4, noise=S.noise, schedule=sch).cpu()
    S.d.set_prediction("v_prediction", 0.9, zero_terminal_snr=True)
    _equal(S.d.sample_latent(S.cond, 7.5, 4, noise=S.noise, schedule=sch).cpu(), want, "no_cfg, phi 0.9")
    r = Diffuser(ctx, TINY_REFINER, synth_weights(TINY_REFINER, seed=1))
    latent, rn = torch.randn(2, 4, 16, 16, generator=gen(5)), torch.randn(2, 4, 16, 16, generator=gen(7))
    rs = Schedule("dpmpp_2m", "trailing", 5, first_step=2, renoise=True)
    outs = []
    for phi in (0.0, 0.9):
        r.set_prediction("v_prediction", phi, zero_terminal_snr=True)
        outs.append((r.refine_latent(latent, S.cond, 7.5, 800, 50, noise=rn).cpu(),
                     r.refine_latent(latent, S.cond, 7.5, 0, 5, noise=rn, schedule=rs).cpu()))
    r.close()
    _equal(outs[1][0], outs[0][0], "refiner DDIM, phi 0.9")
    _equal(outs[1][1], outs[0][1], "refiner scheduled, phi 0.9")


# ---- 4. the hand-driven loop ----------------------------------------------------------------------------------------------------------
def test_hand_driven_steps_are_sample_latent(S):
    S.d.set_prediction("v_prediction", 0.7, zero_terminal_snr=True)
    want = S.d.sample_latent(S.cond, 7.5, 5, noise=S.noise).cpu()
    S.d.sampler_begin(S.cond, 7.5)
    S.d.sampler_set_latent(S.noise)
    ts = list(range(999, -1, -200))
    for t in ts:
        S.d.sampler_step(t, t - 200 if t >= 200 else -1)
    _equal(S.d.sampler_get_latent(S.noise).cpu(), want, "hand-driven loop")
    host = S.noise.clone()
    S.d.sampler_begin(S.cond, 7.5)
    for t in ts:
        S.d.sampler_step_host(t, t - 200 if t >= 200 else -1, host)
    _equal(host, want, "hand-driven host loop")


# ---- 5. DeepCache with v ----------------------------------------------------------------------------------------------------------------
def test_deepcache_interval_3_with_v(S):
    S.d.set_deepcache(3, 2)
    S.d.set_prediction("v_prediction", 0.0, zero_terminal_snr=True)
    sch = Schedule("dpmpp_2m", "trailing", 5)
    got = S.d.sample_latent(S.cond, 7.5, 5, noise=S.noise, schedule=sch).cpu()
    t, sig = SO.schedule("trailing", 5, ZSNR)
    ref = PR.sample(DO.eps_fn(TINY, S.wf, S.oc, 7.5, 3, 2), "dpmpp_2m", t, sig, S.noise.double() * (sig[0] ** 2 + 1) ** 0.5)
    e = rel_err(got, ref)
    print(f"DeepCache interval 3, v zero-SNR DPM++ 2M: rel err vs oracle {e:.2e}")
    assert e <= SAMPLE_TOL


# ---- 6. the table, plan builds and refusals ---------------------------------------------------------------------------------------------
def test_table_and_plan_builds(S):
    S.d.sample_latent(S.cond, 7.5, 3, noise=S.noise)
    n = plan_builds(S.d)
    S.d.set_prediction("v_prediction", 0.7, zero_terminal_snr=True)
    assert [S.d.alpha(i) for i in (0, 500, 999)] == [float(ZSNR[i]) for i in (0, 500, 999)] and S.d.alpha(999) == 2.0 ** -24
    S.d.sample_latent(S.cond, 7.5, 3, noise=S.noise)
    S.d.sample_latent(S.cond, 7.5, 3, noise=S.noise, schedule=Schedule("dpmpp_2m", "trailing", 3))
    S.d.set_prediction("v_prediction", 0.2)   # the loaded table again
    assert np.array_equal(np.array([S.d.alpha(i) for i in range(TINY.n_steps)]), S.loaded)
    S.d.sample_latent(S.cond, 7.5, 3, noise=S.noise)
    S.d.set_prediction()
    assert np.array_equal(np.array([S.d.alpha(i) for i in range(TINY.n_steps)]), S.loaded)
    assert plan_builds(S.d) == n


def test_refusals_leave_the_previous_state(S):
    S.d.set_prediction("v_prediction", 0.7, zero_terminal_snr=True)
    want = _sample(S, "dpmpp_2m/cfg")
    lib = S.ctx.lib
    bad_up = ZSNR.copy()
    bad_up[500] = bad_up[499]
    bad_range = ZSNR.copy()
    bad_range[-1] = 0.0
    for args, field in (((2, 0.0), "type"), ((-1, 0.0), "type"), ((1, float("nan")), "guidance_rescale"), ((1, 1.5), "guidance_rescale"),
                        ((1, -0.1), "guidance_rescale"), ((1, 0.5, ZSNR[:10]), "n_alphas"), ((1, 0.5, bad_up), "alphas_cumprod_host[500]"),
                        ((1, 0.5, bad_range), "alphas_cumprod_host[999]")):
        assert _raw(S.d, *args) != 0
        assert field in lib.sdxl_last_error(S.ctx.h).decode()
        assert S.d.alpha(999) == 2.0 ** -24
        _equal(_sample(S, "dpmpp_2m/cfg"), want, f"after refusing {field}")
    s = _lib.Prediction()
    s.type, s.guidance_rescale, s.n_alphas, s.alphas_cumprod_host = 1, 0.5, TINY.n_steps, None
    assert lib.sdxl_unet_set_prediction(S.d.h, C.byref(s)) != 0
    assert "alphas_cumprod_host" in lib.sdxl_last_error(S.ctx.h).decode()
    _equal(_sample(S, "dpmpp_2m/cfg"), want, "after refusing a null table")
    with pytest.raises(SdxlError, match="prediction"):
        S.d.set_prediction("sample")


# ---- 7. the pipeline's per-call phi and from_diffusers_dir ----------------------------------------------------------------------------
def test_pipeline_guidance_rescale_is_for_the_call(ctx):
    from sdxl_b200 import TINY_CLIP, TINY_OPEN_CLIP, TINY_VAE, ClipTextEncoder, Embedder, LatentDecoder, OpenClipTokenizer, UNetConfig
    from sdxl_b200.pipeline import sample
    mini = os.path.join(os.path.dirname(__file__), "golden", "mini_bpe")
    ca, cb = TINY_CLIP, TINY_OPEN_CLIP
    ucfg = UNetConfig(adm_in_channels=cb.embed_dim + 6 * 256, model_channels=64, channel_mults=(1, 2, 4), transformer_depths=(0, 1, 1),
                      context_dim=ca.n_state + cb.n_state)
    tok = OpenClipTokenizer(os.path.join(mini, "mini_merges.txt"), os.path.join(mini, "mini_vocab.txt"))
    emb = Embedder(ctx, ClipTextEncoder(ctx, ca, synth_weights(ca, seed=1)), ClipTextEncoder(ctx, cb, synth_weights(cb, seed=2)), tok, tok)
    dif = Diffuser(ctx, ucfg, synth_weights(ucfg, seed=3))
    vae = LatentDecoder(ctx, TINY_VAE, synth_weights(TINY_VAE, seed=0))
    kw = dict(guidance=5.0, n_steps=4, resolution=(64, 64), seed=0, sampler="dpmpp_2m", spacing="trailing")
    dif.set_prediction("v_prediction", 0.0, zero_terminal_snr=True)
    plain = sample(emb, dif, vae, "a photo of a cat", **kw)
    rescaled = sample(emb, dif, vae, "a photo of a cat", guidance_rescale=0.7, **kw)
    pred, phi, table = dif.prediction
    assert pred == "v_prediction" and phi == 0.0 and np.array_equal(table, alphas_cumprod(ucfg.n_steps, zero_terminal_snr=True))
    dif.set_prediction("v_prediction", 0.7, zero_terminal_snr=True)
    same = sample(emb, dif, vae, "a photo of a cat", **kw)
    dif.set_prediction("v_prediction", 0.0, zero_terminal_snr=True)
    assert torch.equal(rescaled, same) and not torch.equal(rescaled, plain)
    assert torch.equal(sample(emb, dif, vae, "a photo of a cat", **kw), plain)   # phi restored after the call
    dif.close()


def _pipeline_dir(root, scheduler_config):
    from lora_cases import write_safetensors
    from test_inpaint_cpu import TINY_JSON, to_diffusers
    unet = os.path.join(root, "unet")
    os.makedirs(unet)
    with open(os.path.join(unet, "config.json"), "w") as f:
        json.dump(TINY_JSON, f)
    write_safetensors(os.path.join(unet, "diffusion_pytorch_model.safetensors"), to_diffusers(TINY, synth_weights(TINY, seed=0)))
    if scheduler_config is not None:
        os.makedirs(os.path.join(root, "scheduler"))
        with open(os.path.join(root, "scheduler", "scheduler_config.json"), "w") as f:
            json.dump(scheduler_config, f)
    return unet


def test_from_diffusers_dir_reads_the_scheduler_config(ctx, tmp_path, S):
    base = dict(_class_name="EulerDiscreteScheduler", beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                num_train_timesteps=1000, timestep_spacing="trailing")
    cases = {"none": None, "eps": dict(base, prediction_type="epsilon"),
             "v": dict(base, prediction_type="v_prediction", rescale_betas_zero_snr=True)}
    outs = {}
    for name, sc in cases.items():
        d = Diffuser.from_diffusers_dir(ctx, _pipeline_dir(str(tmp_path / name), sc))
        pred, phi, table = d.prediction
        if name == "v":
            assert pred == "v_prediction" and phi == 0.0 and d.alpha(999) == 2.0 ** -24
            assert np.array_equal(np.array([d.alpha(i) for i in range(TINY.n_steps)]), ZSNR)
        else:
            assert pred == "epsilon" and table is None
            assert np.array_equal(np.array([d.alpha(i) for i in range(TINY.n_steps)]), S.loaded)
        outs[name] = d.sample_latent(S.cond, 7.5, 4, noise=S.noise, schedule=Schedule("dpmpp_2m", "trailing", 4)).cpu()
        d.close()
    _equal(outs["eps"], outs["none"], "epsilon config")
    S.d.set_prediction("v_prediction", 0.0, zero_terminal_snr=True)
    _equal(outs["v"], S.d.sample_latent(S.cond, 7.5, 4, noise=S.noise, schedule=Schedule("dpmpp_2m", "trailing", 4)).cpu(), "v config")
    with pytest.raises(SdxlError, match="prediction_type"):
        Diffuser.from_diffusers_dir(ctx, _pipeline_dir(str(tmp_path / "sample"), dict(base, prediction_type="sample")))
    with pytest.raises(SdxlError, match="beta_schedule"):
        Diffuser.from_diffusers_dir(ctx, _pipeline_dir(str(tmp_path / "linear"), dict(base, prediction_type="v_prediction",
                                                                                        beta_schedule="linear")))


# ---- 8. fresh-memory fills, graphs and PDL ---------------------------------------------------------------------------------------------
WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "prediction_invariance_worker.py")
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
        assert got.keys() == base.keys()
        for k in base:
            _equal(got[k], base[k], f"{name}: {k}")
