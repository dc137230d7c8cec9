"""The scheduled samplers with each kind of attachment, and the `sample()` front end: a scheduled sample on a Karras schedule
(fractional timesteps) against the oracle chain built from oracle/unet_oracle.py's guided noise with the attachment and
tests/scheduler_oracle.py; the T2I-Adapter window derived from the schedule; sample(..., sampler=, spacing=, no_cfg=) with and
without a refiner; Euler against the DDIM kernel on one step; the step kernel's remaining paths."""
import ctypes as C

import numpy as np
import pytest
import torch

import sdxl_b200
from sdxl_b200 import (TINY, TINY_CONTROLNET, TINY_INPAINT, TINY_REFINER, TINY_T2I_ADAPTER, Conditioning, ControlNet, Diffuser, IPAdapter,
                       SdxlError, T2IAdapter, _testing, schedulers, synth_weights)
from sdxl_b200.ip_adapter import synth_ip_adapter
from sdxl_b200.lora import merge_into
from sdxl_b200.schedulers import Schedule
from oracle import unet_oracle as O
import freeu_oracle as FO
import ip_adapter_oracle as IPO
import scheduler_oracle as SO
import t2i_adapter_oracle as TA
from lora_cases import layer_paths, make_adapter
from test_schedulers_gpu import LAT, Setup, noises  # noqa: F401
from harness import arb, rel_err, tiny_conditioning

pytestmark = pytest.mark.gpu
SAMPLE_TOL = 5e-3
G = 7.5


@pytest.fixture(scope="module")
def S(ctx):
    s = Setup(ctx)
    yield s
    s.d.close()


def guided_eps(cfg, w, oc, att):
    """The guided noise prediction with the attachment att(t) at timestep t."""
    return lambda x_in, t: O.forward_diffuser(cfg, w, x_in.float(), torch.tensor([float(t)]), oc, G, att(t))


def chain(S, sch, eps, z):
    t, sig = SO.schedule(sch.spacing, sch.n_steps, S.a64)
    return SO.sample(eps, sch.sampler, t, sig, z * (sig[0] ** 2 + 1) ** 0.5)


def check(name, got, ref, plain):
    e, moved = rel_err(got, ref), rel_err(got, plain)
    print(f"{name}: scheduled sample rel err vs oracle chain {e:.2e}; the attachment moves the latent by {moved:.2e}")
    assert e <= SAMPLE_TOL and moved > 3 * e


SCH = Schedule("euler", "karras", 4)


@pytest.fixture(scope="module")
def plain(S):
    return S.d.sample_latent(S.cond, G, 4, noise=noises(1)[0], schedule=SCH)


# ---- one test per attachment kind ------------------------------------------------------------------------------------------------
def test_controlnet(S, ctx, plain):
    wc = synth_weights(TINY_CONTROLNET, seed=7)
    net = ControlNet(ctx, TINY_CONTROLNET, wc)
    hint = torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(4))
    z = noises(1)[0]
    S.d.set_controls([(net, hint, 0.8)])
    try:
        got = S.d.sample_latent(S.cond, G, 4, noise=z, schedule=SCH)
    finally:
        S.d.set_controls([])
        net.close()
    att = O.Attach(controls=[(TINY_CONTROLNET, O.to_f32(wc), hint, 0.8)])
    ref = chain(S, SCH, guided_eps(TINY, S.wf, S.oc, lambda t: att), z)
    check("ControlNet", got, ref, plain)


def test_image_prompt(S, ctx, plain):
    D = 32
    wa = synth_ip_adapter(TINY, D, seed=3)
    ad = IPAdapter(ctx, TINY, D, wa)
    e = torch.randn(1, 2, D, generator=torch.Generator().manual_seed(20))
    z = noises(1)[0]
    S.d.set_image_prompt(ad, e, 0.9)
    try:
        got = S.d.sample_latent(S.cond, G, 4, noise=z, schedule=SCH)
    finally:
        S.d.set_image_prompt(None)
        ad.close()
    att = IPO.attach(O.to_f32(wa), e, None, IPO.uniform_scales(TINY, 0.9))
    check("image prompt", got, chain(S, SCH, guided_eps(TINY, S.wf, S.oc, lambda t: att), z), plain)


@pytest.mark.parametrize("spacing, factor", [("karras", 0.25), ("karras", 0.5), ("karras", 1.0), ("leading", 1.0), ("trailing", 0.5)])
def test_t2i_adapter_window_follows_the_schedule(S, ctx, spacing, factor):
    """The window closes after int(n * factor) steps of THIS schedule (on Karras between two fractional timesteps); at factor 1 the
    adapter acts on every step, also on leading's t = 1 and Karras's t = 0 that a DDIM-derived t_min would cut off."""
    sch = Schedule("euler", spacing, 4)
    wa = synth_weights(TINY_T2I_ADAPTER, seed=1)
    ad = T2IAdapter(ctx, TINY_T2I_ADAPTER, wa)
    hint = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(10))
    t, _ = schedulers.build(S.a64, sch)
    t_min = schedulers.t2i_t_min(S.a64, sch, factor)
    k = int(4 * factor)
    on = [int(np.rint(v)) >= t_min for v in t]
    assert on == [i < k for i in range(4)], (t, t_min)
    z = noises(1)[0]
    S.d.set_t2i_adapters([(ad, hint, 3.0)], t_min=t_min)
    try:
        got = S.d.sample_latent(S.cond, G, 4, noise=z, schedule=sch)
    finally:
        S.d.set_t2i_adapters([])
        ad.close()
    att = O.Attach(t2i=(TA.summed_features([(TINY_T2I_ADAPTER, O.to_f32(wa), hint, 3.0)]), 0))
    first = set(float(v) for v in SO.schedule(spacing, 4, S.a64)[0][:k])
    ref = chain(S, sch, guided_eps(TINY, S.wf, S.oc, lambda tk: att if float(tk) in first else None), z)
    always = chain(S, sch, guided_eps(TINY, S.wf, S.oc, lambda tk: att), z) if k < 4 else None
    e = rel_err(got, ref)
    print(f"T2I-Adapter, {spacing}, factor {factor} (t = {np.round(t, 2)}, t_min {t_min}): rel err vs oracle chain {e:.2e}"
          + (f"; vs the chain with the window never closing {rel_err(got, always):.2e}" if always is not None else ""))
    assert e <= SAMPLE_TOL
    # an adapter that stays on for the late steps too moves the latent by less than the f16 noise of the sample, so only the window that
    # closes after the first step tells the two chains apart here; test_t2i_window_compares_the_rounded_timestep pins the rest exactly
    assert k != 1 or rel_err(got, always) > 3 * e


def test_t2i_window_compares_the_rounded_timestep(S, ctx):
    """Karras, 4 steps: t = 999, 690.14, 152.39, 0. The device adds the features where lround(t) >= t_min: every t_min in (152, 690]
    gives the same run bit for bit, 691 switches step 1 off and 152 switches step 2 on."""
    sch = Schedule("euler", "karras", 4)
    t, _ = schedulers.build(S.a64, sch)
    assert [int(np.rint(v)) for v in t] == [999, 690, 152, 0]
    ad = T2IAdapter(ctx, TINY_T2I_ADAPTER, synth_weights(TINY_T2I_ADAPTER, seed=1))
    hint = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(10))
    z = noises(1)[0]
    out = {}
    try:
        for t_min in (152, 153, 690, 691):
            S.d.set_t2i_adapters([(ad, hint, 1.0)], t_min=t_min)
            out[t_min] = S.d.sample_latent(S.cond, G, 4, noise=z, schedule=sch)
    finally:
        S.d.set_t2i_adapters([])
        ad.close()
    assert torch.equal(out[153], out[690])
    assert not torch.equal(out[690], out[691]) and not torch.equal(out[152], out[153])


def test_inpainting_unet_condition(S, ctx):
    w = synth_weights(TINY_INPAINT, seed=0)
    d = Diffuser(ctx, TINY_INPAINT, w)
    g = torch.Generator().manual_seed(11)
    mask = (torch.rand(2, 1, 16, 16, generator=g) < 0.4).float()
    cond = torch.cat([mask, torch.randn(2, 4, 16, 16, generator=g) * (1 - mask)], dim=1)
    other = torch.cat([1 - mask, torch.randn(2, 4, 16, 16, generator=g) * mask], dim=1)
    z = noises(1)[0]
    c, oc = Conditioning(**tiny_conditioning(refiner=True)), O.OracleConditioning(**tiny_conditioning(refiner=True))
    try:
        d.set_inpaint_condition(other)
        plain = d.sample_latent(c, G, 4, noise=z, schedule=SCH)
        d.set_inpaint_condition(cond)
        got = d.sample_latent(c, G, 4, noise=z, schedule=SCH)
    finally:
        d.close()
    wf = O.to_f32(w)
    ref = chain(S, SCH, guided_eps(TINY_INPAINT, wf, oc, lambda t: O.Attach(concat=cond)), z)
    check("inpainting UNet condition", got, ref, plain)


def test_freeu(S, plain):
    z = noises(1)[0]
    S.d.set_freeu(*FO.RECOMMENDED_SDXL)
    try:
        got = S.d.sample_latent(S.cond, G, 4, noise=z, schedule=SCH)
    finally:
        S.d.set_freeu(None)
    att = O.Attach(freeu=FO.RECOMMENDED_SDXL)
    check("FreeU", got, chain(S, SCH, guided_eps(TINY, S.wf, S.oc, lambda t: att), z), plain)


def test_merged_lora(S, plain):
    ad = make_adapter(TINY, layer_paths(TINY), rank=4, seed=5)
    z = noises(1)[0]
    S.d.set_adapters([(ad, 0.5)])
    try:
        got = S.d.sample_latent(S.cond, G, 4, noise=z, schedule=SCH)
    finally:
        S.d.set_adapters([])
    wf = O.to_f32(merge_into(S.w, ad, 0.5))
    eps = lambda x_in, t: O.forward_diffuser(TINY, wf, x_in.float(), torch.tensor([float(t)]), S.oc, G)   # noqa: E731
    check("merged LoRA", got, chain(S, SCH, eps, z), plain)
    assert torch.equal(S.d.sample_latent(S.cond, G, 4, noise=z, schedule=SCH), plain)   # restored


# ---- sample() ------------------------------------------------------------------------------------------------------------------------
class FixedEmbedder:
    """sample() needs text_to_conditioning only; the text encoders have their own tests."""
    def text_to_conditioning(self, prompt, size, crop, ar):
        return Conditioning(**tiny_conditioning(B=1, res=tuple(size), refiner=True))


class LatentOut:
    def latent_to_image(self, latent):
        return latent


def test_sample_with_a_schedule_and_a_refiner(S, ctx):
    """sample(..., sampler=, spacing=, no_cfg=): the base model on the whole schedule, then the refiner from the first step below
    t = 200 with the base latent re-noised to that step's sigma by seed + 1's stream."""
    wr = synth_weights(TINY_REFINER, seed=1)
    refiner = Diffuser(ctx, TINY_REFINER, wr)
    oc = O.OracleConditioning(**tiny_conditioning(B=1, refiner=True))
    z = noises(1, seed=6)[0][:1]
    kw = dict(guidance=G, n_steps=6, resolution=(128, 128), noise=z, seed=3)
    try:
        base = sdxl_b200.sample(FixedEmbedder(), S.d, LatentOut(), "x", sampler="dpmpp_2m", spacing="karras", **kw)
        both = sdxl_b200.sample(FixedEmbedder(), S.d, LatentOut(), "x", refiner=refiner, sampler="dpmpp_2m", spacing="karras", **kw)
        nocfg = sdxl_b200.sample(FixedEmbedder(), S.d, LatentOut(), "x", no_cfg=True, **kw)   # defaults: Euler, leading
        with pytest.raises(SdxlError, match="no step is below"):   # 999, 749, 499, 249: the hand-off point does not exist
            sdxl_b200.sample(FixedEmbedder(), S.d, LatentOut(), "x", refiner=refiner, spacing="reference", guidance=G, n_steps=4,
                             resolution=(128, 128), noise=z)
    finally:
        refiner.close()
    t, sig = SO.schedule("karras", 6, S.a64)
    eps_b = lambda x_in, tk: O.forward_diffuser(TINY, S.wf, x_in.float(), torch.tensor([float(tk)]), oc, G)   # noqa: E731
    ref_base = SO.sample(eps_b, "dpmpp_2m", t, sig, z * (sig[0] ** 2 + 1) ** 0.5)
    e_base = rel_err(base, ref_base)
    k0 = next(k for k in range(6) if t[k] < 200)
    assert 0 < k0 < 6
    zr = ctx.randn(z.numel(), 4, 0).cpu().reshape(z.shape)
    wrf = O.to_f32(wr)
    eps_r = lambda x_in, tk: O.forward_diffuser(TINY_REFINER, wrf, x_in.float(), torch.tensor([float(tk)]), oc, G)   # noqa: E731
    ref_both = SO.sample(eps_r, "dpmpp_2m", t, sig, ref_base + sig[k0] * zr, k0=k0)
    e_both = rel_err(both, ref_both)
    tl, sl = SO.schedule("leading", 6, S.a64)
    eps_c = lambda x_in, tk: O.unet_forward(TINY, S.wf, x_in.float(), torch.tensor([float(tk)]), oc.context_full, oc.channel_context)   # noqa: E731
    e_nocfg = rel_err(nocfg, SO.sample(eps_c, "euler", tl, sl, z * (sl[0] ** 2 + 1) ** 0.5))
    print(f"sample(): DPM++ 2M Karras 6 steps {e_base:.2e}; with the refiner from step {k0} {e_both:.2e}; no_cfg Euler leading {e_nocfg:.2e}"
          f" (the refiner moves the latent by {rel_err(both, base):.2e})")
    assert max(e_base, e_both, e_nocfg) <= SAMPLE_TOL and rel_err(both, base) > 1e-2


def test_sample_derives_the_t2i_window_from_the_schedule(S, ctx):
    """sample(..., t2i_adapters=, spacing='leading') at factor 1 equals an attachment that is never switched off."""
    wa = synth_weights(TINY_T2I_ADAPTER, seed=1)
    ad = T2IAdapter(ctx, TINY_T2I_ADAPTER, wa)
    hint = torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(10))
    z = noises(1, seed=6)[0][:1]
    try:
        got = sdxl_b200.sample(FixedEmbedder(), S.d, LatentOut(), "x", guidance=G, n_steps=4, resolution=(128, 128), noise=z,
                               t2i_adapters=[(ad, hint, 1.0)], spacing="leading")
        S.d.set_t2i_adapters([(ad, hint, 1.0)], t_min=0)
        want = S.d.sample_latent(Conditioning(**tiny_conditioning(B=1, refiner=True)), G, 4, noise=z,
                                 schedule=Schedule("euler", "leading", 4))
        S.d.set_t2i_adapters([(ad, hint, 1.0)], t_min=sdxl_b200.t2i_t_min(4, 1.0))   # the DDIM loop's window: cuts t = 1 off
        cut = S.d.sample_latent(Conditioning(**tiny_conditioning(B=1, refiner=True)), G, 4, noise=z,
                                schedule=Schedule("euler", "leading", 4))
    finally:
        S.d.set_t2i_adapters([])
        ad.close()
    assert torch.equal(got, want) and not torch.equal(got, cut)


# ---- Euler is DDIM, on the device ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("use_cfg", [False, True])
def test_one_euler_step_is_the_ddim_kernel(ctx, use_cfg):
    """The same eps rows through cfg_ddim_kernel (VP latent) and guided_step_kernel (xh = x / sqrt(a)) with step_coef's Euler
    coefficients: the next model inputs agree to f32 rounding, which a wrong coefficient would not."""
    a64 = SO.sdxl_alphas(1000, f16=True)
    worst = 0.0
    for spacing, n, k in (("reference", 10, 0), ("reference", 10, 6), ("reference", 10, 9), ("trailing", 16, 3), ("leading", 7, 6)):
        sch = Schedule("euler", spacing, n)
        t, sig = schedulers.build(a64, sch)
        coef = (C.c_float * 5)()
        s = sch.to_struct()
        _testing.load().sdxl_test_step_coef(C.byref(s), k, t.ctypes.data, sig.ctypes.data, 1, coef)
        Bimg, Cc, HW, ld = 2, 4, 16 * 16, 4
        g = torch.Generator().manual_seed(k)
        eps = torch.randn((2 if use_cfg else 1) * Bimg, HW, ld, generator=g).cuda()
        x0 = torch.randn(Bimg, Cc, HW, generator=g)
        a, ap = a64[int(t[k])], (a64[int(t[k + 1])] if k + 1 < n else 1.0)
        x = x0.clone().cuda()
        _testing.cfg_ddim(eps, ld, Bimg, Cc, HW, use_cfg, G, a ** 0.5, (1 - a) ** 0.5, ap ** 0.5, (1 - ap) ** 0.5, x)
        xh = (x0.double() * (sig[k] ** 2 + 1) ** 0.5).float().cuda()
        x_in = torch.empty_like(xh)
        _testing.guided_step(eps, ld, Bimg, Cc, HW, use_cfg, False, G, 0.0, float(sig[k]), list(coef), xh, x_in)
        torch.cuda.synchronize()
        worst = max(worst, rel_err(x_in, x))
    print(f"one Euler step vs cfg_ddim_kernel (cfg={use_cfg}): worst rel L2 {worst:.2e}")
    assert worst <= 2e-6


# ---- the step kernel's remaining paths -----------------------------------------------------------------------------------------------
def test_step_kernel_blend_with_eps_rows_and_in_kernel_blend_noise(ctx):
    """CFG rows, sampler noise and blend noise both generated in the kernel from their own subsequences, history written with
    ch = 0 (DPM++ 2M's first step)."""
    Bimg, Cc, HW, ld = 2, 4, 45, 8
    g = torch.Generator().manual_seed(8)
    eps = torch.randn(2 * Bimg, HW, ld, generator=g)
    xh0, ref = (torch.randn(Bimg, Cc, HW, generator=g) for _ in range(2))
    mask = (torch.rand(Bimg, Cc, HW, generator=g) > 0.5).to(torch.uint8)
    n = xh0.numel()
    z, zb = (ctx.randn(n, 99, s).cpu().reshape(xh0.shape).double() for s in (4, 5))
    xh, x_in, hist = xh0.clone().cuda(), torch.empty_like(xh0).cuda(), torch.full_like(xh0, 7.0).cuda()
    coef = (0.3, 0.7, 0.0, 0.9, 0.5)
    _testing.guided_step(eps.cuda(), ld, Bimg, Cc, HW, True, False, G, 0.0, 2.0, coef, xh, x_in, hist, True, seed=99, z_subseq=4,
                         zb_subseq=5, mask=mask.cuda(), ref=ref.cuda(), sigma_blend=1.5)
    torch.cuda.synchronize()
    e = eps.double().permute(0, 2, 1)[:, :Cc]
    guided = e[Bimg:] + (e[:Bimg] - e[Bimg:]) * G
    Dd = xh0.double() - 2.0 * guided
    want = torch.where(mask.bool(), 0.3 * xh0.double() + 0.7 * Dd + 0.9 * z, ref.double() + 1.5 * zb)
    assert rel_err(xh, want) < 1e-6 and rel_err(x_in, want * 0.5) < 1e-6 and rel_err(hist, Dd) < 1e-6


def test_seeded_inpainting_takes_blend_noise_before_sampler_noise(S):
    """A seeded inpainting run equals the run with sdxl_randn's tensors injected in the documented order."""
    sch = Schedule("euler_ancestral", "trailing", 4)
    ref, mask = arb(*LAT) * 0.5, noises(1, seed=12)[0] > 0.1
    seeded = S.d.sample_latent_with_inpainting(S.cond, G, 4, ref, mask, seed=21, schedule=sch)
    k = sch.n_noise(initial=True, inpainting=True)
    assert k == 1 + 4 + 3
    z = torch.stack([S.ctx.randn(int(np.prod(LAT)), 21, i).reshape(LAT) for i in range(k)])
    injected = S.d.sample_latent_with_inpainting(S.cond, G, 4, ref, mask, init_noise=z[0], step_noise=z[1:], schedule=sch)
    assert torch.equal(seeded, injected)
    swapped = z.clone()
    swapped[[1, 2]] = z[[2, 1]]
    assert not torch.equal(S.d.sample_latent_with_inpainting(S.cond, G, 4, ref, mask, init_noise=swapped[0], step_noise=swapped[1:],
                                                             schedule=sch), seeded)

