"""GPU tests of the scheduled samplers (sdxl_sample_latent_scheduled, guided_step_kernel, the float timestep): the kernels against
float64, the Euler path against sdxl_sample_latent's DDIM, every sampler against the oracle chain (oracle/unet_oracle.py forward +
tests/scheduler_oracle.py), the CFG-free layout, partial schedules, the inpainting blend, seeded noise, PAG, and the plan-build counts."""
import ctypes as C

import numpy as np
import pytest
import torch

import sdxl_b200
from sdxl_b200 import TINY, Conditioning, Diffuser, SdxlError, _testing, pag_layer_mask, schedulers, synth_weights
from sdxl_b200.schedulers import SAMPLERS, Schedule
from oracle import unet_oracle as O
import pag_oracle as PO
import scheduler_oracle as SO
from harness import arb, h16f, plan_builds, rel_err, tiny_conditioning

pytestmark = pytest.mark.gpu
SAMPLE_TOL = 5e-3
LAT = (2, 4, 16, 16)


def noises(n, seed=0):
    return torch.randn(n, *LAT, generator=torch.Generator().manual_seed(seed))


class Setup:
    def __init__(self, ctx):
        self.ctx = ctx
        self.w = synth_weights(TINY, seed=0)
        self.wf = O.to_f32(self.w)
        self.d = Diffuser(ctx, TINY, self.w)
        self.alphas = sdxl_b200.alphas_cumprod(TINY.n_steps)
        self.a64 = np.array([O.get_alpha(self.alphas, i) for i in range(TINY.n_steps)])
        self.cond = Conditioning(**tiny_conditioning(refiner=True))
        self.oc = O.OracleConditioning(**tiny_conditioning(refiner=True))

    def eps_fn(self, guidance, no_cfg=False):
        def f(x_in, t):
            ts = torch.tensor([float(t)], dtype=torch.float32)
            if no_cfg:
                return O.unet_forward(TINY, self.wf, x_in.float(), ts, self.oc.context_full, self.oc.channel_context)
            return O.forward_diffuser(TINY, self.wf, x_in.float(), ts, self.oc, guidance)
        return f

    def oracle(self, sch, z, guidance=7.5, init=None, blend=None):
        """The chain in float32 tensors with float64 scalars; z: the call's noise tensors in its documented order."""
        t, sig = SO.schedule(sch.spacing, sch.n_steps, self.a64, sch.karras_rho or 7.0)
        it = iter(z)
        k0, k1 = sch.first_step, sch.last_step or sch.n_steps
        if init is None:
            x = next(it) * (sig[0] ** 2 + 1) ** 0.5
        else:
            x = init + (sig[k0] * next(it) if sch.renoise else 0.0)
        return SO.sample(self.eps_fn(guidance, sch.no_cfg), sch.sampler, t, sig, x, lambda: next(it), k0, k1, sch.eta or 1.0, sch.s_noise or 1.0,
                         blend, torch.where)


@pytest.fixture(scope="module")
def S(ctx):
    s = Setup(ctx)
    yield s
    s.d.close()


# ---- kernels -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("use_cfg, use_pag", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("coef", [(0.4, 0.6, 0.0, 0.0, 0.8), (0.3, 0.7, 0.0, 0.9, 0.5), (0.2, 1.3, -0.5, 0.0, 0.7), (1e-4, 0.99, 0.0, 2.5, 0.3),
                                  (0.0, 1.0, 0.0, 0.0, 1.0)])
@pytest.mark.parametrize("HW", [37 * 5, 64])
def test_guided_step_kernel(ctx, use_cfg, use_pag, coef, HW):
    """Every sampler's row shape (Euler, ancestral, DPM++ 2M with history, LCM, the step to sigma 0) x the four row layouts, with
    injected and with in-kernel noise, a padded eps pitch holding NaN, and an extent that is not a multiple of the 4-wide blocks."""
    Bimg, Cc, ld = 3, 4, 8
    groups = 1 + use_cfg + use_pag
    g = torch.Generator().manual_seed(HW + groups)
    eps = torch.randn(groups * Bimg, HW, ld, generator=g)
    eps[:, :, Cc:] = float("nan")
    xh0, hist0, z = (torch.randn(Bimg, Cc, HW, generator=g) for _ in range(3))
    s, p_t, sigma = 7.5, 2.25, 3.7
    cx, cd, ch, cn, c_in = coef
    e = eps.double().permute(0, 2, 1)[:, :Cc]
    c = e[:Bimg]
    guided = e[Bimg:2 * Bimg] + (c - e[Bimg:2 * Bimg]) * s if use_cfg else c
    if use_pag:
        guided = guided + p_t * (c - e[(groups - 1) * Bimg:])
    Dd = xh0.double() - sigma * guided
    worst = 0.0
    for injected in (True, False):
        zz = z if injected else ctx.randn(xh0.numel(), 11, 5).cpu().reshape(xh0.shape)
        xh, hist, x_in = xh0.clone().cuda(), hist0.clone().cuda(), torch.empty_like(xh0).cuda()
        _testing.guided_step(eps.cuda(), ld, Bimg, Cc, HW, use_cfg, use_pag, s, p_t, sigma, coef, xh, x_in, hist, ch != 0.0,
                             z.cuda() if injected else None, seed=11, z_subseq=5)
        torch.cuda.synchronize()
        want = cx * xh0.double() + cd * Dd + ch * hist0.double() + cn * zz.double()
        worst = max(worst, rel_err(xh, want), rel_err(x_in, want * c_in))
        assert rel_err(hist, Dd if ch != 0.0 else hist0) < 1e-6
    print(f"guided_step cfg={use_cfg} pag={use_pag} coef={coef} HW={HW}: rel err vs float64 {worst:.2e}")
    assert worst < 1e-6


@pytest.mark.parametrize("n", [4 * 16 * 16, 3 * 185, 7])
def test_in_kernel_noise_is_randn_bit_for_bit(ctx, n):
    xh, x_in = torch.zeros(1, 1, n).cuda(), torch.empty(1, 1, n).cuda()
    _testing.guided_step(None, 0, 1, 1, n, False, False, 1.0, 0.0, 0.0, (0.0, 0.0, 0.0, 1.0, 1.0), xh, x_in, seed=1234567890123, z_subseq=3)
    torch.cuda.synchronize()
    want = ctx.randn(n, 1234567890123, 3)
    assert torch.equal(xh.flatten(), want) and torch.equal(x_in.flatten(), want)


def test_blend_and_entry_in_the_step_kernel(ctx):
    """mask ? xh' : ref + sigma_blend * zb, and the entry form without a model output (xh = latent + sigma z)."""
    g = torch.Generator().manual_seed(5)
    lat, z, zb, ref = (torch.randn(2, 4, 45, generator=g) for _ in range(4))
    mask = (torch.rand(2, 4, 45, generator=g) > 0.5).to(torch.uint8)
    xh, x_in = lat.clone().cuda(), torch.empty_like(lat).cuda()
    _testing.guided_step(None, 0, 2, 4, 45, False, False, 1.0, 0.0, 0.0, (1.0, 0.0, 0.0, 2.5, 0.25), xh, x_in, z=z.cuda(), zb=zb.cuda(),
                         mask=mask.cuda(), ref=ref.cuda(), sigma_blend=1.5)
    torch.cuda.synchronize()
    want = torch.where(mask.bool(), lat.double() + 2.5 * z.double(), ref.double() + 1.5 * zb.double())
    assert rel_err(xh, want) < 1e-6 and rel_err(x_in, want * 0.25) < 1e-6
    xh = lat.clone().cuda()   # cx = 1 alone: the state passes through bit for bit
    _testing.guided_step(None, 0, 2, 4, 45, False, False, 1.0, 0.0, 0.0, (1.0, 0.0, 0.0, 0.0, 1.0), xh, x_in)
    torch.cuda.synchronize()
    assert torch.equal(xh.cpu(), lat) and torch.equal(x_in.cpu(), lat)


def test_float_timestep_embedding(ctx):
    dim = 320
    t = torch.tensor([0.0, 1.0, 499.0, 999.0, 0.25, 152.3857, 690.141, 998.5])
    got = _testing.timestep_embedding_f32(t.cuda(), dim).cpu()
    half = dim // 2
    freq = torch.exp(torch.arange(half, dtype=torch.float64) * (-np.log(10000.0) / half))
    arg = t.double()[:, None] * freq[None]
    want = torch.cat([arg.cos(), arg.sin()], 1)
    err = float((got.double() - want).abs().max())
    print(f"float timestep embedding: max abs err vs float64 {err:.2e}")
    assert err < 2e-4   # f32 arguments up to 999: the int kernel's own accuracy
    ints = [0, 1, 499, 999]
    assert torch.equal(got[:4], ctx.timestep_embedding(ints, dim).cpu())


def test_forward_at_integer_t_is_the_int_forward(S):
    x = arb(2, 4, 16, 16).cuda()
    S.d.set_conditioning(h16f(arb(2, 7, 24)), h16f(arb(2, 8)))
    a, b, c = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
    lib, ctx = S.ctx.lib, S.ctx
    ctx.call("forward_f32", lib.sdxl_unet_forward_f32, S.d.h, 2, 16, 16, x.data_ptr(), 500, a.data_ptr())
    ctx.call("forward_f32_at", lib.sdxl_unet_forward_f32_at, S.d.h, 2, 16, 16, x.data_ptr(), 500.0, b.data_ptr())
    ctx.call("forward_f32_at", lib.sdxl_unet_forward_f32_at, S.d.h, 2, 16, 16, x.data_ptr(), 500.5, c.data_ptr())
    ctx.synchronize()
    assert torch.equal(a, b) and not torch.equal(a, c)
    ts = torch.tensor([500.5])
    ref = O.unet_forward(TINY, S.wf, x.cpu(), ts, h16f(arb(2, 7, 24)), h16f(arb(2, 8)))
    assert rel_err(c, ref) < 2e-3


# ---- samples -----------------------------------------------------------------------------------------------------------------------
def test_euler_on_the_reference_spacing_is_sample_latent(S):
    """Ties the whole new path to the reference-derived one: same noise, n dividing 1000 so that both run n steps."""
    z = noises(1)[0]
    ddim = S.d.sample_latent(S.cond, 7.5, 10, noise=z)
    b0 = plan_builds(S.d)
    got = S.d.sample_latent(S.cond, 7.5, 10, noise=z, schedule=Schedule("euler", "reference", 10))
    ref = O.sample_latent(TINY, S.wf, S.alphas, z, S.oc, 7.5, 10)
    e, e_ddim, e_euler = rel_err(got, ddim), rel_err(ddim, ref), rel_err(got, ref)
    print(f"Euler / reference spacing vs sdxl_sample_latent (10 steps): rel L2 {e:.2e}; vs the DDIM oracle: DDIM {e_ddim:.2e}, Euler {e_euler:.2e}")
    # the two updates are the same function (tests/test_schedulers_cpu.py, 1e-12) evaluated with different f32 roundings of the state;
    # the f16 activations of ten guided forwards amplify those last bits to the order of either path's own distance to the oracle
    assert e <= 2e-3 and e_euler <= SAMPLE_TOL
    assert plan_builds(S.d) == b0  # the same plan serves both


@pytest.mark.parametrize("sampler", sorted(SAMPLERS))
@pytest.mark.parametrize("spacing", ["karras", "trailing", "leading"])
@pytest.mark.parametrize("n", [4, 10])
def test_samplers_vs_oracle_chain(S, sampler, spacing, n):
    sch = Schedule(sampler, spacing, n)
    z = noises(sch.n_noise(initial=True), seed=n)
    got = S.d.sample_latent(S.cond, 7.5, n, noise=z[0], step_noise=z[1:] if len(z) > 1 else None, schedule=sch)
    ref = S.oracle(sch, list(z))
    e = rel_err(got, ref)
    print(f"{sampler} / {spacing} / {n} steps: rel err vs oracle chain {e:.2e}")
    assert e <= SAMPLE_TOL


def test_no_cfg_runs_the_conditional_rows_alone(S):
    sch = Schedule("euler", "trailing", 4, no_cfg=True)
    z = noises(1)[0]
    S.d.sample_latent(S.cond, 7.5, 4, noise=z, schedule=Schedule("euler", "trailing", 4))
    b0, l0 = plan_builds(S.d), S.ctx.launch_count
    S.d.sample_latent(S.cond, 7.5, 4, noise=z, schedule=Schedule("dpmpp_2m", "karras", 4))   # sampler and schedule: the plan stays
    assert plan_builds(S.d) == b0
    cfg_launches = S.ctx.launch_count - l0
    got = S.d.sample_latent(S.cond, 7.5, 4, noise=z, schedule=sch)
    assert plan_builds(S.d) == b0 + 1  # the batch is the plan's key
    kw = tiny_conditioning(refiner=True)
    kw.update(unconditional_context_full=None, unconditional_channel_context=None, unconditional_context_open_clip=None,
              unconditional_channel_context_refiner=None)
    l1 = S.ctx.launch_count
    bare = S.d.sample_latent(Conditioning(**kw), 123.0, 4, noise=z, schedule=sch)   # no unconditional tensors, guidance ignored
    assert plan_builds(S.d) == b0 + 1 and torch.equal(got, bare)
    assert S.ctx.launch_count - l1 == cfg_launches   # the rows are one batched forward: the same launches on half the rows
    with pytest.raises(SdxlError, match="null"):
        S.d.sample_latent(Conditioning(**kw), 7.5, 4, noise=z, schedule=Schedule("euler", "trailing", 4))
    e = rel_err(got, S.oracle(sch, [z]))
    print(f"no_cfg Euler trailing 4 steps: rel err vs oracle chain {e:.2e}")
    assert e <= SAMPLE_TOL
    # one step's eps is the direct forward of the conditional rows, bit for bit: xh' = D = xh - sigma eps
    one = Schedule("euler", "trailing", 1, no_cfg=True)
    t, sig = schedulers.build(S.a64, one)
    D = S.d.sample_latent(S.cond, 1.0, 1, noise=z, schedule=one)
    xh = (torch.zeros_like(z) + np.float32((sig[0] ** 2 + 1) ** 0.5) * z).cuda()   # the entry kernel's arithmetic
    x_in = xh * np.float32(1.0 / (sig[0] ** 2 + 1) ** 0.5)
    eps = S.d.unet_forward(x_in, [t[0]], S.cond.context_full, S.cond.channel_context)
    assert rel_err(D, xh - np.float32(sig[0]) * eps) < 1e-6


def test_partial_schedules(S):
    sch = Schedule("euler_ancestral", "karras", 6)
    z = noises(sch.n_noise(initial=True), seed=3)
    whole = S.d.sample_latent(S.cond, 7.5, 6, noise=z[0], step_noise=z[1:], schedule=sch)
    from dataclasses import replace
    head = S.d.sample_latent(S.cond, 7.5, 6, noise=z[0], step_noise=z[1:4], schedule=replace(sch, last_step=3))
    tail = S.d.refine_latent(head, S.cond, 7.5, 0, 6, noise=z[4:], schedule=replace(sch, first_step=3))
    assert torch.equal(tail, whole)   # the hand-off at sigma_3 with renoise = 0
    # img2img: the latent re-noised to sigma_k0, against the oracle
    img = Schedule.from_strength(6, 0.5, sampler="dpmpp_2m", spacing="karras")
    lat = arb(*LAT) * 0.7
    zr = noises(1, seed=9)
    got = S.d.refine_latent(lat, S.cond, 7.5, 0, 6, noise=zr, schedule=img)
    e = rel_err(got, S.oracle(img, list(zr), init=lat))
    print(f"img2img DPM++ 2M from step 3 of 6: rel err vs oracle chain {e:.2e}")
    assert e <= SAMPLE_TOL
    with pytest.raises(SdxlError, match="init_latent"):
        S.d._sample(S.cond, 7.5, 6, 0, None, None, 0, None, None, schedule=replace(sch, first_step=3))
    with pytest.raises(SdxlError, match="last_step"):
        S.d.sample_latent(S.cond, 7.5, 6, schedule=replace(sch, last_step=7))


def test_inpainting_blend_vs_oracle(S):
    sch = Schedule("euler_ancestral", "trailing", 4)
    z = noises(sch.n_noise(initial=True, inpainting=True), seed=4)
    ref = arb(*LAT) * 0.5
    mask = (arb(*LAT) > 0.1)
    got = S.d.sample_latent_with_inpainting(S.cond, 7.5, 4, ref, mask, init_noise=z[0], step_noise=z[1:], schedule=sch)
    want = S.oracle(sch, list(z), blend=(ref, mask))
    e = rel_err(got, want)
    print(f"inpainting blend, Euler-a trailing 4 steps: rel err vs oracle chain {e:.2e}")
    assert e <= SAMPLE_TOL


def test_seeded_runs(S):
    sch = Schedule("lcm", "lcm", 4, no_cfg=True)
    a = S.d.sample_latent(S.cond, 1.0, 4, seed=7, schedule=sch)
    b = S.d.sample_latent(S.cond, 1.0, 4, seed=7, schedule=sch)
    c = S.d.sample_latent(S.cond, 1.0, 4, seed=8, schedule=sch)
    assert torch.equal(a, b) and rel_err(a, c) > 1e-2 and bool(torch.isfinite(a).all())
    # the seeded stream is sdxl_randn's: injecting its tensors in the documented order reproduces the run bit for bit
    z = torch.stack([S.ctx.randn(int(np.prod(LAT)), 7, i).reshape(LAT) for i in range(sch.n_noise(initial=True))])
    d = S.d.sample_latent(S.cond, 1.0, 4, noise=z[0], step_noise=z[1:], schedule=sch)
    assert torch.equal(a, d)


def test_pag_with_adaptive_scale_vs_oracle(S):
    """CFG + PAG through the new entry, p_t from the schedule's timesteps (integers here: the PAG oracle takes integer timesteps)."""
    sch = Schedule("euler", "trailing", 4)
    z = noises(1, seed=2)[0]
    S.d.set_pag("mid", 3.0, 0.004)
    try:
        got = S.d.sample_latent(S.cond, 7.5, 4, noise=z, schedule=sch)
    finally:
        S.d.set_pag(None)
    layers = PO.paths_of_mask(TINY, pag_layer_mask(TINY, "mid"))
    t, sig = SO.schedule("trailing", 4, S.a64)
    att = PO.attach(TINY, layers, 3.0, 0.004)
    f = lambda x_in, tk: O.forward_diffuser(TINY, S.wf, x_in.float(), torch.tensor([int(tk)], dtype=torch.int32), S.oc, 7.5, att)   # noqa: E731
    ref = SO.sample(f, "euler", t, sig, z * (sig[0] ** 2 + 1) ** 0.5)
    e, moved = rel_err(got, ref), rel_err(got, S.d.sample_latent(S.cond, 7.5, 4, noise=z, schedule=sch))
    print(f"CFG + PAG (adaptive) Euler trailing 4 steps: rel err vs oracle {e:.2e}; PAG moves the latent by {moved:.2e}")
    assert e <= SAMPLE_TOL and moved > 1e-3
