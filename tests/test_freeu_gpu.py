"""GPU tests of FreeU (sdxl_unet_set_freeu and the OP_FREEU kernel), tiny configs: the kernel against float64, forwards, a CFG sample
and a refiner refine against the f32 oracle (oracle/unet_oracle.py) with the bounds of tests/test_unet_gpu.py, its composition with
ControlNets, PAG, image prompts and the inpainting UNet, batch invariance, the bit-exact identities of detach and value 0, the plan
kept by value-only changes, and the refusals that leave the previous state in effect."""
import ctypes as C

import numpy as np
import pytest
import torch

import sdxl_b200
from sdxl_b200 import (TINY, TINY_CONTROLNET, TINY_INPAINT, TINY_REFINER, Conditioning, ControlNet, Diffuser, IPAdapter, SdxlError,
                       _lib, _testing, pag_layer_mask, synth_weights)
from sdxl_b200.ip_adapter import synth_ip_adapter
from oracle import unet_oracle as O
import freeu_oracle as FO
import ip_adapter_oracle as IPO
import pag_oracle as PO
from harness import h16f, plan_builds, rel_err, tiny_conditioning

pytestmark = pytest.mark.gpu
FWD_TOL = 2e-3
SAMPLE_TOL = 5e-3
T = 499
FV = FO.RECOMMENDED_SDXL
D = 32   # image_embed_dim of the tiny IP-Adapter


class Setup:
    def __init__(self, ctx):
        self.ctx = ctx
        self.w = synth_weights(TINY, seed=0)
        self.wf = O.to_f32(self.w)
        self.d = Diffuser(ctx, TINY, self.w)
        g = torch.Generator().manual_seed(1)
        self.x = torch.randn(3, 4, 16, 16, generator=g)
        self.c = h16f(torch.randn(3, 7, TINY.context_dim, generator=g))
        self.y = h16f(torch.randn(3, TINY.adm_in_channels, generator=g))
        self.noise = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(0))

    def fwd(self, B=2, x=None):
        x = self.x[:B] if x is None else x
        return self.d.unet_forward(x, [T], self.c[:B], self.y[:B]).cpu()

    def ref(self, B=2, x=None, **kw):
        x = self.x[:B] if x is None else x
        return O.unet_forward(TINY, self.wf, x, torch.tensor([T]), self.c[:B], self.y[:B], O.Attach(freeu=FV, **kw))

    def sample(self, B=2):
        return self.d.sample_latent(Conditioning(**tiny_conditioning(B, refiner=True)), 7.5, 4, noise=self.noise[:B]).cpu()


@pytest.fixture(scope="module")
def S(ctx):
    s = Setup(ctx)
    yield s
    s.d.set_freeu(None)
    s.d.close()


# ---- kernel ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C_", [320, 640, 1280])
@pytest.mark.parametrize("H, W", [(8, 8), (5, 7), (1, 2), (32, 32), (48, 48), (64, 64)])
@pytest.mark.parametrize("Cx_mult", [1, 2])
def test_kernel_vs_float64(ctx, C_, H, W, Cx_mult):
    """The skip against the float64 closed form (fourier_filter_closed, itself checked against torch.fft on the CPU), the backbone's
    first half against x * b (one f32 rounding: exact), its second half untouched. 32 x 32, 48 x 48 and 64 x 64 split the pixels
    over clusters of 2, 4 and 8 blocks."""
    B, Cx, s, b = 2, Cx_mult * C_, 0.2, 1.4
    g = torch.Generator().manual_seed(C_ + 10 * H + W + Cx)
    r0 = torch.randn(B, H, W, C_, generator=g) + 0.5   # a mean, so the (0, 0) bin is large
    x0 = torch.randn(B, H, W, Cx, generator=g)
    r, x = r0.cuda(), x0.cuda()
    tw = _testing.freeu_twiddles(H, W).cuda()
    sv, bv = torch.tensor([s], device="cuda"), torch.tensor([b], device="cuda")
    _testing.freeu(r, C_, x, Cx, B, H, W, tw, sv, bv)
    torch.cuda.synchronize()
    want = FO.fourier_filter_closed(r0.double().permute(0, 3, 1, 2), s).permute(0, 2, 3, 1)
    e = rel_err(r, want)
    print(f"freeu C={C_} {H}x{W} Cx={Cx}: skip rel err vs float64 {e:.2e}")
    assert e < 1e-5
    assert torch.equal(x[..., :Cx // 2].cpu(), (x0[..., :Cx // 2].double() * np.float32(b)).float())
    assert torch.equal(x[..., Cx // 2:].cpu(), x0[..., Cx // 2:])


# ---- forwards ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h, w", [(16, 16), (32, 32), (20, 28)])
def test_forward_vs_oracle(S, h, w):
    """20 x 28: the deepest level is 5 x 7, odd extents on both axes."""
    x = torch.randn(2, 4, h, w, generator=torch.Generator().manual_seed(h + w))
    S.d.set_freeu(*FV)
    got = S.fwd(2, x)
    prof = S.d.profile_plan()
    S.d.set_freeu(None)
    plain = S.fwd(2, x)
    ref = S.ref(2, x)
    e, moved = rel_err(got, ref), rel_err(got, plain)
    print(f"FreeU forward {h}x{w}: rel err vs oracle {e:.2e}; FreeU moves it by {moved:.2e}")
    assert e <= FWD_TOL and moved > 1e-3
    assert prof["freeu"]["launches"] == 6


def test_forward_with_controlnet_vs_oracle(S, ctx):
    """The ControlNet residuals are added to the skips before the filter; filtering first differs by more than the tolerance."""
    wc = synth_weights(TINY_CONTROLNET, seed=7)
    net = ControlNet(ctx, TINY_CONTROLNET, wc)
    hint = torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(4))
    S.d.set_controls([(net, hint, 0.8)])
    S.d.set_freeu(*FV)
    got = S.fwd(2)
    S.d.set_freeu(None)
    S.d.set_controls([])
    net.close()
    wcf = O.to_f32(wc)
    ref = S.ref(2, controls=[(TINY_CONTROLNET, wcf, hint, 0.8)])
    wrong = _wrong_order_forward(S, wcf, hint)
    e, e_wrong = rel_err(got, ref), rel_err(got, wrong)
    print(f"FreeU + ControlNet: rel err vs oracle {e:.2e}; vs the oracle that filters before the control add {e_wrong:.2e}")
    assert e <= FWD_TOL and e_wrong > 2 * FWD_TOL and rel_err(wrong, ref) > 2 * FWD_TOL   # the two orders differ by 9e-3


def _wrong_order_forward(S, wcf, hint):
    """The oracle with the filter applied to the skips before the ControlNet residuals are added (the order diffusers does not use)."""
    ts, x, c, y = torch.tensor([T]), S.x[:2], S.c[:2], S.y[:2]
    w = S.wf
    emb = O._emb(TINY, w, ts, y)
    h, saved = O.encoder(TINY, w, x, emb, c)
    res, r_mid = O.controlnet_forward(TINY_CONTROLNET, wcf, x, ts, c, y, O.hint_embedding(TINY_CONTROLNET, wcf, hint))
    h = h + 0.8 * r_mid
    for i, (kind, p, nh, d) in enumerate(O.unet_blocks(TINY)[2]):
        skip, r = saved.pop(), res[len(saved)]
        if i // 3 < 2:
            h, skip = O.apply_freeu(i // 3, h, skip, FV)
        h = torch.cat([h, skip + 0.8 * r], dim=1)
        h = O._run_block(kind, p, nh, d, h, emb, c, w)
    h = O.group_norm(h, w["norm_out/weight"], w["norm_out/bias"])
    return O.conv2d(O.silu(h), w, "conv_out")


def test_forward_with_pag_vs_oracle(S):
    """FreeU on every row, the perturbed one included."""
    S.d.set_pag("mid", 3.0)
    S.d.set_freeu(*FV)
    got = S.d.unet_forward(S.x, [T], S.c, S.y, perturbed_rows=1).cpu()
    S.d.set_freeu(None)
    S.d.set_pag(None)
    layers = PO.paths_of_mask(TINY, pag_layer_mask(TINY, "mid"))
    ref = torch.cat([S.ref(2), O.unet_forward(TINY, S.wf, S.x[2:], torch.tensor([T]), S.c[2:], S.y[2:], O.Attach(freeu=FV, pag_layers=layers))])
    e = rel_err(got, ref)
    print(f"FreeU + PAG (mid): rel err vs oracle {e:.2e}")
    assert e <= FWD_TOL


def test_forward_with_image_prompt_vs_oracle(S, ctx):
    wa = synth_ip_adapter(TINY, D, seed=3)
    ad = IPAdapter(ctx, TINY, D, wa)
    e = torch.randn(1, 1, D, generator=torch.Generator().manual_seed(2))   # n_batch 1: every row (of any batch) uses it
    S.d.set_image_prompt(ad, e, 0.8)
    S.d.set_freeu(*FV)
    got = S.fwd(2)
    S.d.set_freeu(None)
    S.d.set_image_prompt(None)
    ad.close()
    waf = O.to_f32(wa)
    ref = S.ref(2, prompts=[(waf, IPO.prompt_tokens(waf, e).expand(2, -1, -1), IPO.uniform_scales(TINY, 0.8), None)])
    err = rel_err(got, ref)
    print(f"FreeU + IP-Adapter: rel err vs oracle {err:.2e}")
    assert err <= FWD_TOL


def test_inpainting_unet_vs_oracle(ctx):
    w = synth_weights(TINY_INPAINT, seed=0)
    d = Diffuser(ctx, TINY_INPAINT, w)
    g = torch.Generator().manual_seed(6)
    x, cond = torch.randn(2, 4, 16, 16, generator=g), torch.rand(1, 5, 16, 16, generator=g)
    c, y = h16f(torch.randn(2, 7, TINY.context_dim, generator=g)), h16f(torch.randn(2, TINY.adm_in_channels, generator=g))
    d.set_inpaint_condition(cond)
    d.set_freeu(*FV)
    got = d.unet_forward(x, [T], c, y).cpu()
    d.close()
    ref = O.unet_forward(TINY_INPAINT, O.to_f32(w), x, torch.tensor([T]), c, y, O.Attach(concat=cond, freeu=FV))
    e = rel_err(got, ref)
    print(f"FreeU, inpainting UNet: rel err vs oracle {e:.2e}")
    assert e <= FWD_TOL


def test_refiner_forward_vs_oracle(ctx):
    w = synth_weights(TINY_REFINER, seed=1)
    d = Diffuser(ctx, TINY_REFINER, w)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 4, 8, 16, generator=g)
    c, y = h16f(torch.randn(2, 6, 40, generator=g)), h16f(torch.randn(2, 16, generator=g))
    d.set_freeu(*FV)
    got = d.unet_forward(x, [T], c, y).cpu()
    d.close()
    e = rel_err(got, O.unet_forward(TINY_REFINER, O.to_f32(w), x, torch.tensor([T]), c, y, O.Attach(freeu=FV)))
    print(f"FreeU, TINY_REFINER forward: rel err vs oracle {e:.2e}")
    assert e <= FWD_TOL


# ---- samples -----------------------------------------------------------------------------------------------------------------------
def test_sample_cfg_vs_oracle(S):
    S.d.set_freeu(*FV)
    got = S.sample()
    S.d.set_freeu(None)
    ref = O.sample_latent(TINY, S.wf, sdxl_b200.alphas_cumprod(TINY.n_steps), S.noise,
                          O.OracleConditioning(**tiny_conditioning(refiner=True)), 7.5, 4,
                          att=O.Attach(freeu=FV))
    e, moved = rel_err(got, ref), rel_err(got, S.sample())
    print(f"CFG sample with FreeU: rel err vs oracle {e:.2e}; FreeU moves the latent by {moved:.2e}")
    assert e <= SAMPLE_TOL and moved > 1e-3


def test_refiner_refine_vs_oracle(ctx):
    w = synth_weights(TINY_REFINER, seed=1)
    d = Diffuser(ctx, TINY_REFINER, w)
    g = torch.Generator().manual_seed(5)
    latent, noise = torch.randn(2, 4, 8, 16, generator=g), torch.randn(2, 4, 8, 16, generator=g)
    c = tiny_conditioning(2, 6, (64, 128), refiner=True)
    d.set_freeu(*FV)
    got = d.refine_latent(latent, Conditioning(**c), 7.5, 800, 50, noise=noise).cpu()
    d.set_freeu(None)
    plain = d.refine_latent(latent, Conditioning(**c), 7.5, 800, 50, noise=noise).cpu()
    d.close()
    ref = O.refine_latent(TINY_REFINER, O.to_f32(w), sdxl_b200.alphas_cumprod(), latent, O.OracleConditioning(**c), 7.5, 800, 50,
                          noise, att=O.Attach(freeu=FV))
    e = rel_err(got, ref)
    print(f"TINY_REFINER refine with FreeU: rel err vs oracle {e:.2e}; FreeU moves it by {rel_err(got, plain):.2e}")
    assert e <= SAMPLE_TOL and not torch.equal(got, plain)


# ---- identities --------------------------------------------------------------------------------------------------------------------
def test_batch_invariance(S):
    S.d.set_freeu(*FV)
    both = S.fwd(2)
    one = [S.d.unet_forward(S.x[i:i + 1], [T], S.c[i:i + 1], S.y[i:i + 1]).cpu() for i in range(2)]
    S.d.set_freeu(None)
    assert torch.equal(both[0], one[0][0]) and torch.equal(both[1], one[1][0])


def test_detach_and_value_zero_are_bit_identical(S, ctx):
    fresh = Diffuser(ctx, TINY, S.w)
    never = fresh.sample_latent(Conditioning(**tiny_conditioning(refiner=True)), 7.5, 4, noise=S.noise).cpu()
    fresh_fwd = fresh.unet_forward(S.x[:2], [T], S.c[:2], S.y[:2]).cpu()
    fresh_ops = fresh.plan_num_ops
    fresh.close()
    S.d.set_freeu(*FV)
    moved = S.sample()
    S.d.set_freeu(None)
    assert torch.equal(S.sample(), never) and not torch.equal(moved, never)
    assert torch.equal(S.fwd(2), fresh_fwd) and S.d.plan_num_ops == fresh_ops
    for zero in range(4):
        v = list(FV)
        v[zero] = 0.0
        S.d.set_freeu(*FV)
        S.d.set_freeu(*v)                                         # any value 0: detached
        assert torch.equal(S.fwd(2), fresh_fwd) and S.d.plan_num_ops == fresh_ops
    assert torch.equal(S.sample(), never)


def test_value_only_change_keeps_the_plan(S):
    S.d.set_freeu(*FV)
    S.sample()
    n = plan_builds(S.d)
    results = []
    for v in ((1.1, 0.5, 1.2, 1.1), (0.7, 0.3, 1.5, 1.3), FV):
        S.d.set_freeu(*v)
        results.append(S.sample())
        assert plan_builds(S.d) == n
    assert not torch.equal(results[0], results[2])
    S.d.set_freeu(None)
    S.d.set_freeu(1.1, 0.5, 1.2, 1.1)                         # a fresh attach with the same values computes the same latent
    assert torch.equal(S.sample(), results[0])
    S.d.set_freeu(None)


def test_refusals_leave_the_previous_state(S):
    S.d.set_freeu(*FV)
    want = S.fwd(2)
    n = plan_builds(S.d)
    for i, name in enumerate(("s1", "s2", "b1", "b2")):
        for bad in (float("nan"), float("inf"), -float("inf")):
            f = _lib.Freeu()
            v = list(FV)
            v[i] = bad
            if i == 0:
                v[1] = 0.0    # a refused value is refused even where another value would detach
            f.s1, f.s2, f.b1, f.b2 = v
            assert S.ctx.lib.sdxl_unet_set_freeu(S.d.h, C.byref(f)) != 0
            assert name in S.ctx.lib.sdxl_last_error(S.ctx.h).decode()
            assert torch.equal(S.fwd(2), want) and plan_builds(S.d) == n
    with pytest.raises(SdxlError, match="all four values"):
        S.d.set_freeu(0.9, 0.2)
    assert torch.equal(S.fwd(2), want) and plan_builds(S.d) == n
    S.d.set_freeu(None)


def test_sampler_needs_a_new_begin_after_attach(S):
    """Attaching drops the plan: a step without a new sampler_begin is refused, and a new begin runs with FreeU."""
    cond = Conditioning(**tiny_conditioning(refiner=True))
    s, keep = cond.to_struct(S.ctx.device)
    lib = S.ctx.lib
    assert lib.sdxl_sampler_begin(S.d.h, C.byref(s), C.c_double(7.5)) == 0
    S.d.set_freeu(*FV)
    assert lib.sdxl_sampler_step(S.d.h, 999, 749) != 0
    assert "sampler_begin" in lib.sdxl_last_error(S.ctx.h).decode()
    S.d.set_freeu(None)
    torch.cuda.synchronize()


def test_pipeline_freeu_attaches_for_the_call(ctx):
    import os
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
    kw = dict(guidance=5.0, n_steps=4, resolution=(64, 64), seed=0)
    plain = sample(emb, dif, vae, "a photo of a cat", **kw)
    with_freeu = sample(emb, dif, vae, "a photo of a cat", freeu=FV, **kw)
    dif.set_freeu(*FV)
    same = sample(emb, dif, vae, "a photo of a cat", **kw)
    dif.set_freeu(None)
    assert torch.equal(with_freeu, same) and not torch.equal(with_freeu, plain)
    assert torch.equal(sample(emb, dif, vae, "a photo of a cat", **kw), plain)   # detached after the call
    both = sample(emb, dif, vae, "a photo of a cat", freeu=FV, pag=(3.0, "mid"), **kw)
    assert not torch.equal(both, with_freeu)
    assert torch.equal(sample(emb, dif, vae, "a photo of a cat", **kw), plain)
    dif.close()
