"""GPU tests of DPM++ 2M SDE, DPM++ 3M SDE, UniPC, Heun and DPM2 (DESIGN.md §20), tiny configs: the step kernel's two-row form
against float64, partial schedules, seeded noise, the latent blend before every evaluation, and the attachments per evaluation
(PAG with guidance rescale and the v prediction, DeepCache, ControlNet) and every sampler x {Karras, trailing} x {4, 10} steps
against the oracle chains of tests/scheduler2_oracle.py (oracle/unet_oracle.py forward + the sampler's recurrence)."""
from dataclasses import replace

import numpy as np
import pytest
import torch

from sdxl_b200 import TINY, TINY_CONTROLNET, ControlNet, _testing, pag_layer_mask, synth_weights
from sdxl_b200.schedulers import MORE_SAMPLERS, Schedule
from oracle import unet_oracle as O
import deepcache_oracle as DO
import pag_oracle as PO
import prediction_oracle as PR
import scheduler2_oracle as SO
import scheduler_oracle as SO1
from harness import arb, rel_err
from test_schedulers_gpu import LAT, Setup, noises

pytestmark = pytest.mark.gpu
SAMPLE_TOL = 5e-3


@pytest.fixture(scope="module")
def S(ctx):
    s = Setup(ctx)
    yield s
    s.d.close()


def chain(S, sch, z, guidance=7.5, init=None, blend=None):
    """Setup.oracle's chain (float32 tensors, float64 scalars; z: the call's noise tensors in its documented order) with a §20
    sampler, on the engine's noise table."""
    t, sig = SO1.schedule(sch.spacing, sch.n_steps, S.a64, sch.karras_rho or 7.0)
    it = iter(z)
    k0, k1 = sch.first_step, sch.last_step or sch.n_steps
    x = next(it) * (sig[0] ** 2 + 1) ** 0.5 if init is None else init + (sig[k0] * next(it) if sch.renoise else 0.0)
    return SO.sample2(S.eps_fn(guidance, sch.no_cfg), sch.sampler, t, sig, x, lambda: next(it), k0, k1, sch.eta or 1.0,
                      sch.s_noise or 1.0, blend, torch.where, SO1.log_sigmas(S.a64))


# ---- the kernel ------------------------------------------------------------------------------------------------------------------
# (coef = (cx, cs, cd, ch, ch2, cn, c_in), rows = (sx, ss, sd, sh, sh2), write_hist, write_xs, shift): each sampler's launch shapes
ROW_CASES = {
    "3m_three_history": ((0.3, 0.0, 0.8, -0.4, 0.1, 0.9, 0.7), (0.0,) * 5, True, False, True),
    "3m_two_history": ((0.3, 0.0, 0.8, -0.4, 0.0, 0.9, 0.7), (0.0,) * 5, True, False, True),
    "2m_sde_one_history": ((0.5, 0.0, 0.7, -0.3, 0.0, 1.2, 0.9), (0.0,) * 5, True, False, False),
    "unipc_corrected": ((0.0, 0.4, 0.6, 0.3, -0.2, 0.0, 0.5), (0.0, 0.9, 0.2, 0.5, -0.1), True, True, True),
    "unipc_first": ((0.6, 0.0, 0.4, 0.0, 0.0, 0.0, 0.8), (1.0, 0.0, 0.0, 0.0, 0.0), True, True, False),
    "heun_stage2": ((0.2, 1.1, -0.2, -0.1, 0.0, 0.0, 0.6), (0.0,) * 5, False, False, False),
    "dpm2_stage1": ((0.7, 0.0, 0.3, 0.0, 0.0, 0.0, 0.6), (1.0, 0.0, 0.0, 0.0, 0.0), False, True, False),
}


@pytest.mark.parametrize("use_cfg, use_pag", [(False, False), (True, False), (True, True)])
@pytest.mark.parametrize("case", sorted(ROW_CASES))
@pytest.mark.parametrize("HW", [37 * 5, 64])
def test_two_row_step_kernel(ctx, case, use_cfg, use_pag, HW):
    """Both rows from the values before the launch, the history shift, injected and in-kernel noise, a padded eps pitch holding NaN
    and an extent that is not a multiple of the 4-wide blocks."""
    coef, rows, write_hist, write_xs, shift = ROW_CASES[case]
    Bimg, Cc, ld = 3, 4, 8
    groups = 1 + use_cfg + use_pag
    g = torch.Generator().manual_seed(HW + groups)
    eps = torch.randn(groups * Bimg, HW, ld, generator=g)
    eps[:, :, Cc:] = float("nan")
    xh0, xs0, h10, h20, z = (torch.randn(Bimg, Cc, HW, generator=g) for _ in range(5))
    s, p_t, sigma = 7.5, 2.25, 3.7
    e = eps.double().permute(0, 2, 1)[:, :Cc]
    c = e[:Bimg]
    guided = e[Bimg:2 * Bimg] + (c - e[Bimg:2 * Bimg]) * s if use_cfg else c
    if use_pag:
        guided = guided + p_t * (c - e[(groups - 1) * Bimg:])
    D = xh0.double() - sigma * guided
    cx, cs, cd, ch, ch2, cn, c_in = coef
    sx, ss, sd, sh, sh2 = rows
    X, XS, H1, H2 = xh0.double(), xs0.double(), h10.double(), h20.double()
    worst = 0.0
    for injected in (True, False):
        zz = z if injected else ctx.randn(xh0.numel(), 11, 5).cpu().reshape(xh0.shape)
        xh, xs, h1, h2 = (v.clone().cuda() for v in (xh0, xs0, h10, h20))
        x_in = torch.empty_like(xh)
        _testing.guided_step_rows(eps.cuda(), ld, Bimg, Cc, HW, use_cfg, use_pag, s, p_t, sigma, coef, rows, xh, x_in, hist=h1, h2=h2, xs=xs,
                                  write_hist=write_hist, write_xs=write_xs, shift=shift, z=z.cuda() if injected else None, seed=11, z_subseq=5)
        torch.cuda.synchronize()
        want = cx * X + cs * XS + cd * D + ch * H1 + ch2 * H2 + cn * zz.double()
        want_xs = sx * X + ss * XS + sd * D + sh * H1 + sh2 * H2 if write_xs else XS
        worst = max(worst, rel_err(xh, want), rel_err(x_in, want * c_in), rel_err(xs, want_xs))
        assert rel_err(h1, D if write_hist else H1) < 1e-6
        assert torch.equal(h2.cpu(), h10 if shift else h20)
    print(f"two-row step {case} cfg={use_cfg} pag={use_pag} HW={HW}: rel err vs float64 {worst:.2e}")
    assert worst < 1e-6


# ---- samples -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sampler", sorted(MORE_SAMPLERS))
@pytest.mark.parametrize("spacing", ["karras", "trailing"])
@pytest.mark.parametrize("n", [4, 10])
def test_samplers_vs_oracle_chain(S, sampler, spacing, n):
    sch = Schedule(sampler, spacing, n)
    z = noises(sch.n_noise(initial=True), seed=n)
    got = S.d.sample_latent(S.cond, 7.5, n, noise=z[0], step_noise=z[1:] if len(z) > 1 else None, schedule=sch)
    e = rel_err(got, chain(S, sch, list(z)))
    print(f"{sampler} / {spacing} / {n} steps: rel err vs oracle chain {e:.2e}")
    assert e <= SAMPLE_TOL


@pytest.mark.parametrize("sampler", sorted(MORE_SAMPLERS))
def test_deepcache_interval_1_and_detach_are_bit_identical(S, sampler):
    sch = Schedule(sampler, "karras", 4)
    z = noises(1, seed=8)[0]
    plain = S.d.sample_latent(S.cond, 7.5, 4, noise=z, seed=5, schedule=sch)
    S.d.set_deepcache(1, 2)
    try:
        one = S.d.sample_latent(S.cond, 7.5, 4, noise=z, seed=5, schedule=sch)
        S.d.set_deepcache(3, 2)
        moved = S.d.sample_latent(S.cond, 7.5, 4, noise=z, seed=5, schedule=sch)
    finally:
        S.d.set_deepcache(None)
    assert torch.equal(one, plain) and torch.equal(S.d.sample_latent(S.cond, 7.5, 4, noise=z, seed=5, schedule=sch), plain)
    assert not torch.equal(moved, plain)


def test_heun_split_is_the_whole_run(S):
    sch = Schedule("heun_discrete", "karras", 6)
    z = noises(1, seed=3)[0]
    whole = S.d.sample_latent(S.cond, 7.5, 6, noise=z, schedule=sch)
    head = S.d.sample_latent(S.cond, 7.5, 6, noise=z, schedule=replace(sch, last_step=3))
    tail = S.d.refine_latent(head, S.cond, 7.5, 0, 6, schedule=replace(sch, first_step=3))
    assert torch.equal(tail, whole)   # the hand-off at sigma_3 with renoise = 0: Heun keeps nothing across steps


def test_seeded_sde_and_inpainting_runs_are_randn_in_the_documented_order(S):
    lat = int(np.prod(LAT))
    sch = Schedule("dpmpp_2m_sde", "karras", 5)
    a = S.d.sample_latent(S.cond, 7.5, 5, seed=7, schedule=sch)
    z = torch.stack([S.ctx.randn(lat, 7, i).reshape(LAT) for i in range(sch.n_noise(initial=True))])
    assert torch.equal(a, S.d.sample_latent(S.cond, 7.5, 5, noise=z[0], step_noise=z[1:], schedule=sch))
    assert rel_err(a, S.d.sample_latent(S.cond, 7.5, 5, seed=8, schedule=sch)) > 1e-2
    # inpainting with Heun: a blend before each of the two evaluations of a step, at its sigma
    ref, mask = arb(*LAT) * 0.5, arb(*LAT) > 0.1
    sch = Schedule("heun_discrete", "trailing", 4)
    init = noises(1, seed=2)[0]
    a = S.d.sample_latent_with_inpainting(S.cond, 7.5, 4, ref, mask, init_noise=init, seed=9, schedule=sch)
    n = sch.n_noise(initial=False, inpainting=True)
    assert n == 7
    z = torch.stack([S.ctx.randn(lat, 9, i).reshape(LAT) for i in range(n)]).cpu()
    assert torch.equal(a, S.d.sample_latent_with_inpainting(S.cond, 7.5, 4, ref, mask, init_noise=init, step_noise=z, schedule=sch))
    e = rel_err(a, chain(S, sch, [init] + list(z), blend=(ref, mask)))
    print(f"inpainting blend, Heun trailing 4 steps: rel err vs oracle chain {e:.2e}")
    assert e <= SAMPLE_TOL


@pytest.mark.parametrize("sampler", ["dpmpp_3m_sde", "dpm_2"])
def test_no_cfg_and_img2img(S, sampler):
    """The SDE noise on a call without CFG, and an img2img start (history restarts at first order)."""
    sch = Schedule(sampler, "karras", 6, no_cfg=True)
    z = noises(sch.n_noise(initial=True), seed=5)
    got = S.d.sample_latent(S.cond, 7.5, 6, noise=z[0], step_noise=z[1:] if len(z) > 1 else None, schedule=sch)
    e = rel_err(got, chain(S, sch, list(z)))
    img = Schedule.from_strength(6, 0.5, sampler=sampler, spacing="karras")
    lat = arb(*LAT) * 0.7
    zr = noises(img.n_noise(initial=False), seed=9)
    got = S.d.refine_latent(lat, S.cond, 7.5, 0, 6, noise=zr, schedule=img)
    e2 = rel_err(got, chain(S, img, list(zr), init=lat))
    print(f"{sampler}: no_cfg Karras 6 steps rel err {e:.2e}; img2img from step 3 of 6 rel err {e2:.2e}")
    assert e <= SAMPLE_TOL and e2 <= SAMPLE_TOL


def v_as_eps(g_fn, ls):
    """An eps-form model function whose D is the v model's, D = x / (s^2 + 1) - s / sqrt(s^2 + 1) g, at s = sigma(t)."""
    def f(x_in, t):
        s = SO1.sigma_of_t(ls, t)
        x = x_in.double() * (s * s + 1) ** 0.5
        D = x / (s * s + 1) - (s / (s * s + 1) ** 0.5) * g_fn(x_in, t).double()
        return (x - D) / s
    return f


def test_heun_with_pag_rescale_and_v_prediction(S):
    """PAG's adaptive scale, guidance rescale's statistics and v's d_scale at each evaluation's timestep, on the loaded noise table
    (trailing spacing). Not on the zero-terminal-SNR table: from sigma = 4096 Heun's second evaluation of the first step enters
    with (sigma' - sigma) / (2 sigma') ~ -890, which amplifies the f16 error of that forward (1.2e-2 from the chain, DESIGN.md §20)."""
    table = S.a64
    S.d.set_pag("mid", 3.0, 0.004)
    S.d.set_prediction("v_prediction", 0.7)
    sch = Schedule("heun_discrete", "trailing", 4)
    z = noises(1, seed=6)[0]
    try:
        got = S.d.sample_latent(S.cond, 7.5, 4, noise=z, schedule=sch)
    finally:
        S.d.set_prediction()
        S.d.set_pag(None)
    att = PO.attach(TINY, PO.paths_of_mask(TINY, pag_layer_mask(TINY, "mid")), 3.0, 0.004)
    t, sig = SO1.schedule("trailing", 4, table)
    ls = SO1.log_sigmas(table)
    ref = SO.sample2(v_as_eps(PR.model_fn(TINY, S.wf, S.oc, 7.5, 0.7, att), ls), "heun_discrete", t, sig, z.double() * (sig[0] ** 2 + 1) ** 0.5,
                     where=torch.where, ls=ls)
    e = rel_err(got, ref)
    print(f"Heun + PAG (adaptive) + guidance rescale 0.7 + v, trailing 4 steps: rel err vs oracle {e:.2e}")
    assert bool(torch.isfinite(got).all()) and e <= SAMPLE_TOL


def test_heun_with_deepcache_counts_evaluations(S):
    """Interval 2: each two-evaluation step runs one full and one cached forward (DeepCache counts evaluations, not steps)."""
    sch = Schedule("heun_discrete", "karras", 5)
    z = noises(1, seed=4)[0]
    S.d.set_deepcache(2, 2)
    try:
        got = S.d.sample_latent(S.cond, 7.5, 5, noise=z, schedule=sch)
    finally:
        S.d.set_deepcache(None)
    t, sig = SO1.schedule("karras", 5, S.a64)
    x = z * (sig[0] ** 2 + 1) ** 0.5
    evals = []   # the oracle's cache is full on evaluations 0, 2, 4, ...: the first stage of every step, the second cached
    ref = SO.sample2(DO.eps_fn(TINY, S.wf, S.oc, 7.5, 2, 2), "heun_discrete", t, sig, x, where=torch.where, on_eval=evals.append)
    plain = SO.sample2(DO.eps_fn(TINY, S.wf, S.oc, 7.5, 1, 2), "heun_discrete", t, sig, x, where=torch.where)
    assert len(evals) == sch.n_evaluations() == 9
    e, moved = rel_err(got, ref), rel_err(ref, plain)
    print(f"Heun + DeepCache interval 2 (full, cached per step), Karras 5 steps: rel err vs oracle {e:.2e}; DeepCache moves the "
          f"oracle by {moved:.2e}")
    assert e <= SAMPLE_TOL and moved > 3 * e


def test_unipc_with_controlnet(S, ctx):
    wc = synth_weights(TINY_CONTROLNET, seed=7)
    net = ControlNet(ctx, TINY_CONTROLNET, wc)
    hint = torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(4))
    sch = Schedule("unipc", "karras", 5)
    z = noises(1)[0]
    plain = S.d.sample_latent(S.cond, 7.5, 5, noise=z, schedule=sch)
    S.d.set_controls([(net, hint, 0.8)])
    try:
        got = S.d.sample_latent(S.cond, 7.5, 5, noise=z, schedule=sch)
    finally:
        S.d.set_controls([])
        net.close()
    att = O.Attach(controls=[(TINY_CONTROLNET, O.to_f32(wc), hint, 0.8)])
    t, sig = SO1.schedule("karras", 5, S.a64)
    f = lambda x_in, tk: O.forward_diffuser(TINY, S.wf, x_in.float(), torch.tensor([float(tk)]), S.oc, 7.5, att)   # noqa: E731
    ref = SO.sample2(f, "unipc", t, sig, z * (sig[0] ** 2 + 1) ** 0.5, where=torch.where)
    e, moved = rel_err(got, ref), rel_err(got, plain)
    print(f"UniPC + ControlNet, Karras 5 steps: rel err vs oracle chain {e:.2e}; the ControlNet moves the latent by {moved:.2e}")
    assert e <= SAMPLE_TOL and moved > 3 * e
