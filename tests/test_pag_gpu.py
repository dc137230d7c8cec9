"""GPU tests of perturbed-attention guidance (sdxl_unet_set_pag, the identity self-attention op and the PAG-guided DDIM update), tiny
configs, against float64 (kernels) and the f32 oracle (oracle/unet_oracle.py) with the bounds of tests/test_unet_gpu.py, plus the
bit-exact identities of detach and scale 0, the plan kept by scale-only changes, the composition with image prompts and ControlNets,
and the refusals that leave the previous attachment in effect."""
import ctypes as C

import pytest
import torch

import sdxl_b200
from sdxl_b200 import (TINY, TINY_CONTROLNET, TINY_REFINER, Conditioning, ControlNet, Diffuser, IPAdapter, SdxlError, _lib, _testing,
                       pag_layer_mask, synth_weights)
from sdxl_b200.ip_adapter import synth_ip_adapter
from oracle import unet_oracle as O
import ip_adapter_oracle as IPO
import pag_oracle as PO
from harness import h16f, plan_builds, rel_err, tiny_conditioning

pytestmark = pytest.mark.gpu
FWD_TOL = 2e-3
SAMPLE_TOL = 5e-3
T = 499
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

    def fwd(self, rows=1):
        return self.d.unet_forward(self.x, [T], self.c, self.y, perturbed_rows=rows).cpu()

    def sample(self, B=2):
        return self.d.sample_latent(Conditioning(**tiny_conditioning(B, refiner=True)), 7.5, 4, noise=self.noise[:B]).cpu()


@pytest.fixture(scope="module")
def S(ctx):
    s = Setup(ctx)
    yield s
    s.d.set_pag(None)
    s.d.close()


# ---- kernels -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C_", [128, 256])
@pytest.mark.parametrize("Tq", [77, 200])
@pytest.mark.parametrize("Bp", [1, 2])
def test_identity_kernel(ctx, C_, Tq, Bp):
    """The perturbed rows get the V window of the fused QKV rows; the attended rows' output is not touched."""
    Bf = Bp + 2
    g = torch.Generator().manual_seed(C_ + Tq + Bp)
    qkv = torch.randn(Bf * Tq, 3 * C_, generator=g).half().cuda()
    out = torch.full((Bf * Tq, C_), 7.0, dtype=torch.float16, device="cuda")
    r0 = (Bf - Bp) * Tq
    _testing.pag_identity(qkv[r0:], C_, Bp * Tq, out[r0:])
    torch.cuda.synchronize()
    want = qkv[r0:, 2 * C_:].double()
    assert torch.equal(out[r0:].double(), want)
    assert bool((out[:r0] == 7.0).all())


@pytest.mark.parametrize("use_cfg, Bimg", [(True, 1), (True, 2), (False, 2)])
def test_cfg_ddim_kernel_pag(ctx, use_cfg, Bimg):
    """cfg_ddim_kernel's guided update with PAG against float64, for the base layout [cond | uncond | ptb] and the refiner's
    [cond | ptb]."""
    Cc, HW, ld = 4, 37 * 5, 4
    groups = 3 if use_cfg else 2
    g = torch.Generator().manual_seed(Bimg)
    eps = torch.randn(groups * Bimg, HW, ld, generator=g)
    x0 = torch.randn(Bimg, Cc, HW, generator=g)
    s, p_t, a, ap = 7.5, 2.25, 0.31, 0.55
    x = x0.clone().cuda()
    _testing.cfg_ddim(eps.cuda(), ld, Bimg, Cc, HW, use_cfg, s, a ** 0.5, (1 - a) ** 0.5, ap ** 0.5, (1 - ap) ** 0.5, x,
                      use_pag=True, p_t=p_t)
    torch.cuda.synchronize()
    e = eps.double().permute(0, 2, 1)[:, :Cc]
    c, ptb = e[:Bimg], e[(groups - 1) * Bimg:]
    guided = (e[Bimg:2 * Bimg] + (c - e[Bimg:2 * Bimg]) * s if use_cfg else c) + p_t * (c - ptb)
    want = (x0.double() - guided * (1 - a) ** 0.5) / a ** 0.5 * ap ** 0.5 + guided * (1 - ap) ** 0.5
    assert rel_err(x, want) < 1e-6


# ---- forwards ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layers", ["mid", ["down_blocks.1", "up_blocks.0.attentions.1"], [".*"]])
def test_forward_vs_oracle(S, layers):
    mask = pag_layer_mask(TINY, layers)
    S.d.set_pag(layers, 3.0)
    got = S.fwd(1)
    prof = S.d.profile_plan()
    S.d.set_pag(None)
    ref = PO.forward_rows(TINY, S.wf, S.x, torch.tensor([T]), S.c, S.y, PO.paths_of_mask(TINY, mask), 1)
    plain = S.d.unet_forward(S.x[:2], [T], S.c[:2], S.y[:2]).cpu()
    e, moved = rel_err(got, ref), rel_err(got[2], S.d.unet_forward(S.x, [T], S.c, S.y).cpu()[2])
    print(f"PAG {layers}: forward rel err vs oracle {e:.2e}; the perturbed row moves by {moved:.2e}")
    assert e <= FWD_TOL and moved > 1e-3   # TINY's "mid" is 2 self-attentions: the smallest move, ~5e-3
    assert prof["pag_identity"]["launches"] == sum(mask)
    assert torch.equal(got[:2], plain)   # the attended rows: the same work as without the perturbed row, bit for bit


def test_two_perturbed_rows(S):
    S.d.set_pag("mid", 3.0)
    got = S.fwd(2)
    S.d.set_pag(None)
    ref = PO.forward_rows(TINY, S.wf, S.x, torch.tensor([T]), S.c, S.y, PO.paths_of_mask(TINY, pag_layer_mask(TINY, "mid")), 2)
    assert rel_err(got, ref) <= FWD_TOL


def test_forward_with_controlnet_vs_oracle(S, ctx):
    wc = synth_weights(TINY_CONTROLNET, seed=7)
    net = ControlNet(ctx, TINY_CONTROLNET, wc)
    hint = torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(4))
    S.d.set_controls([(net, hint, 0.8)])
    S.d.set_pag("mid", 3.0)
    got = S.fwd(1)
    S.d.set_pag(None)
    S.d.set_controls([])
    net.close()
    layers = PO.paths_of_mask(TINY, pag_layer_mask(TINY, "mid"))
    ctl = [(TINY_CONTROLNET, O.to_f32(wc), hint, 0.8)]
    ts = torch.tensor([T])
    ref = torch.cat([O.unet_forward(TINY, S.wf, S.x[:2], ts, S.c[:2], S.y[:2], O.Attach(controls=ctl)),
                     O.unet_forward(TINY, S.wf, S.x[2:], ts, S.c[2:], S.y[2:], O.Attach(controls=ctl, pag_layers=layers))])
    assert rel_err(got, ref) <= FWD_TOL


# ---- samples -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("adaptive", [0.0, 0.004])
def test_sample_cfg_pag_vs_oracle(S, adaptive):
    """adaptive 0.004: p_t falls from 2.996 at t = 999 to 0 (clamped) at t = 249."""
    S.d.set_pag("mid", 3.0, adaptive)
    got = S.sample()
    S.d.set_pag(None)
    alphas = sdxl_b200.alphas_cumprod(TINY.n_steps)
    layers = PO.paths_of_mask(TINY, pag_layer_mask(TINY, "mid"))
    ref = O.sample_latent(TINY, S.wf, alphas, S.noise, O.OracleConditioning(**tiny_conditioning(refiner=True)), 7.5, 4,
                          att=PO.attach(TINY, layers, 3.0, adaptive))
    e, moved = rel_err(got, ref), rel_err(got, S.sample())
    print(f"CFG + PAG sample (adaptive {adaptive}): rel err vs oracle {e:.2e}; PAG moves the latent by {moved:.2e}")
    assert e <= SAMPLE_TOL and moved > 1e-3


def test_refiner_refine_with_pag_vs_oracle(ctx):
    w = synth_weights(TINY_REFINER, seed=1)
    d = Diffuser(ctx, TINY_REFINER, w)
    g = torch.Generator().manual_seed(5)
    latent, noise = torch.randn(2, 4, 8, 16, generator=g), torch.randn(2, 4, 8, 16, generator=g)
    c = tiny_conditioning(2, 6, (64, 128), refiner=True)
    d.set_pag(["mid", "up_blocks.1.attentions.2"], 2.0)
    got = d.refine_latent(latent, Conditioning(**c), 7.5, 800, 50, noise=noise).cpu()
    d.set_pag(None)
    plain = d.refine_latent(latent, Conditioning(**c), 7.5, 800, 50, noise=noise).cpu()
    d.close()
    layers = PO.paths_of_mask(TINY_REFINER, pag_layer_mask(TINY_REFINER, ["mid", "up_blocks.1.attentions.2"]))
    ref = O.refine_latent(TINY_REFINER, O.to_f32(w), sdxl_b200.alphas_cumprod(), latent, O.OracleConditioning(**c), 7.5, 800, 50, noise,
                          att=PO.attach(TINY_REFINER, layers, 2.0))
    e = rel_err(got, ref)
    print(f"TINY_REFINER refine with PAG: rel err vs oracle {e:.2e}; PAG moves it by {rel_err(got, plain):.2e}")
    assert e <= SAMPLE_TOL and not torch.equal(got, plain)


# ---- identities --------------------------------------------------------------------------------------------------------------------
def test_detach_and_scale_zero_are_bit_identical(S, ctx):
    fresh = Diffuser(ctx, TINY, S.w)
    never = fresh.sample_latent(Conditioning(**tiny_conditioning(refiner=True)), 7.5, 4, noise=S.noise).cpu()
    fresh_fwd = fresh.unet_forward(S.x, [T], S.c, S.y).cpu()
    fresh_ops = fresh.plan_num_ops
    fresh.close()
    S.d.set_pag("mid", 3.0)
    guided = S.sample()
    S.d.set_pag(None)
    assert torch.equal(S.sample(), never) and not torch.equal(guided, never)
    assert torch.equal(S.d.unet_forward(S.x, [T], S.c, S.y).cpu(), fresh_fwd) and S.d.plan_num_ops == fresh_ops
    S.d.set_pag("mid", 0.0)                                   # scale 0: no third row group at all
    assert torch.equal(S.sample(), never)
    assert S.d.unet_forward(S.x, [T], S.c, S.y).cpu().shape[0] == 3 and S.d.plan_num_ops == fresh_ops


def test_scale_only_change_keeps_the_plan(S):
    S.d.set_pag("mid", 3.0)
    S.sample()
    n = plan_builds(S.d)
    results = []
    for scale, adaptive in ((1.5, 0.0), (4.0, 0.002), (3.0, 0.0)):
        S.d.set_pag("mid", scale, adaptive)
        results.append(S.sample())
        assert plan_builds(S.d) == n
    assert not torch.equal(results[0], results[2])
    S.d.set_pag(None)
    S.d.set_pag("mid", 1.5)                                   # a fresh attach at the same scale computes the same latent
    assert torch.equal(S.sample(), results[0])
    n = plan_builds(S.d)
    S.d.set_pag(["down_blocks.1"], 1.5)                       # a new layer set rebuilds the plan
    S.sample()
    assert plan_builds(S.d) == n + 1
    S.d.set_pag(None)


# ---- composition -------------------------------------------------------------------------------------------------------------------
def test_sample_with_image_prompt_vs_oracle(S, ctx):
    """The perturbed rows see the positive image tokens, the unconditional rows the projection of zero embeddings."""
    wa = synth_ip_adapter(TINY, D, seed=3)
    ad = IPAdapter(ctx, TINY, D, wa)
    e = torch.randn(2, 1, D, generator=torch.Generator().manual_seed(2))
    S.d.set_image_prompt(ad, e, 0.8)
    S.d.set_pag("mid", 3.0)
    got = S.sample()
    S.d.set_pag(None)
    S.d.set_image_prompt(None)
    ad.close()
    waf = O.to_f32(wa)
    layers = PO.paths_of_mask(TINY, pag_layer_mask(TINY, "mid"))
    ip = IPO.attach(waf, e, None, IPO.uniform_scales(TINY, 0.8))
    ref = O.sample_latent(TINY, S.wf, sdxl_b200.alphas_cumprod(TINY.n_steps), S.noise,
                          O.OracleConditioning(**tiny_conditioning(refiner=True)), 7.5, 4,
                          att=PO.attach(TINY, layers, 3.0, prompts=ip.prompts, uncond_tokens=ip.uncond_tokens))
    err = rel_err(got, ref)
    print(f"CFG + PAG + IP-Adapter sample: rel err vs oracle {err:.2e}")
    assert err <= SAMPLE_TOL


# ---- refusals ----------------------------------------------------------------------------------------------------------------------
def test_refusals_leave_the_previous_attachment(S):
    S.d.set_pag("mid", 2.0)
    want = S.fwd(1)
    n = plan_builds(S.d)

    def unchanged():
        assert torch.equal(S.d.unet_forward(S.x, [T], S.c, S.y).cpu(), want) and plan_builds(S.d) == n

    n_sa = int(S.ctx.lib.sdxl_unet_num_self_attentions(S.d.h))
    assert n_sa == 17
    mask = pag_layer_mask(TINY, "down_blocks.1")
    keep = (C.c_uint8 * 18)(*(mask + [0]))
    zeros = (C.c_uint8 * 17)()
    for scale, adaptive, nl, layers, rows, what in ((float("nan"), 0.0, 17, keep, 1, "scale"), (-1.0, 0.0, 17, keep, 1, "scale"),
                                                    (0.0, 0.0, 17, keep, 1, "scale"), (2.0, -0.5, 17, keep, 1, "adaptive_scale"),
                                                    (2.0, float("inf"), 17, keep, 1, "adaptive_scale"), (2.0, 0.0, 18, keep, 1, "n_layers"),
                                                    (2.0, 0.0, 16, keep, 1, "n_layers"), (2.0, 0.0, 17, None, 1, "null layers_host"),
                                                    (2.0, 0.0, 17, zeros, 1, "no self-attention"), (2.0, 0.0, 17, keep, -1, "negative")):
        p = _lib.Pag()
        p.scale, p.adaptive_scale, p.n_layers, p.forward_perturbed_rows = scale, adaptive, nl, rows
        p.layers_host = None if layers is None else C.addressof(layers)
        assert S.ctx.lib.sdxl_unet_set_pag(S.d.h, C.byref(p)) != 0
        assert what in S.ctx.lib.sdxl_last_error(S.ctx.h).decode()
        unchanged()
    with pytest.raises(SdxlError, match="matches no self-attention"):
        S.d.set_pag("down_blocks.0", 2.0)
    unchanged()
    with pytest.raises(SdxlError, match="at least one row must be attended"):
        S.fwd(3)
    S.d.set_pag(None)
    with pytest.raises(SdxlError, match="needs PAG attached"):
        S.fwd(1)


def test_pipeline_pag_attaches_for_the_call(ctx):
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
    guided = sample(emb, dif, vae, "a photo of a cat", pag=(3.0, "mid"), **kw)
    dif.set_pag("mid", 3.0)
    same = sample(emb, dif, vae, "a photo of a cat", **kw)
    dif.set_pag(None)
    assert torch.equal(guided, same) and not torch.equal(guided, plain)
    assert torch.equal(sample(emb, dif, vae, "a photo of a cat", **kw), plain)   # detached after the call
    dif.close()
