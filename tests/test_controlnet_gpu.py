"""GPU tests of ControlNet conditioning (sdxl_unet_set_controls), tiny configs, against the f32 oracle
(oracle/unet_oracle.py) with the bounds of tests/test_unet_gpu.py, plus the bit-exact identities of attach / detach / rescale."""
import ctypes as C

import pytest
import torch

import sdxl_b200
from sdxl_b200 import TINY, TINY_CONTROLNET, Conditioning, ControlNet, ControlNetConfig, Diffuser, SdxlError, UNetConfig, synth_weights
from sdxl_b200 import _lib
from oracle import unet_oracle as O
from harness import arb, h16f, plan_builds, rel_err, tiny_conditioning

pytestmark = pytest.mark.gpu
FWD_TOL = 2e-3
SAMPLE_TOL = 5e-3
T = 499


def hint(n, seed):
    return torch.rand(n, 3, 128, 128, generator=torch.Generator().manual_seed(seed))


X = arb(2, 4, 16, 16)


class Setup:
    def __init__(self, ctx):
        self.ctx = ctx
        self.w = synth_weights(TINY, seed=0)
        self.wf = O.to_f32(self.w)
        self.d = Diffuser(ctx, TINY, self.w)
        self.wc = [synth_weights(TINY_CONTROLNET, seed=s) for s in (1, 2)]
        self.wcf = [O.to_f32(w) for w in self.wc]
        self.nets = [ControlNet(ctx, TINY_CONTROLNET, w) for w in self.wc]
        self.c = h16f(arb(2, 7, TINY.context_dim))
        self.y = h16f(arb(2, TINY.adm_in_channels))
        self.h = [hint(2, 10), hint(1, 11)]
        self.noise = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(0))

    def fwd(self):
        return self.d.unet_forward(X, [T], self.c, self.y)

    def oracle_fwd(self, controls):
        return O.unet_forward(TINY, self.wf, X, torch.tensor([T]), self.c, self.y,
                              O.Attach(controls=[(TINY_CONTROLNET, self.wcf[i], self.h[j], s) for i, j, s in controls]))


@pytest.fixture(scope="module")
def S(ctx):
    s = Setup(ctx)
    s.base = s.fwd()
    s.base_ops = s.d.plan_num_ops
    yield s
    s.d.set_controls([])
    for n in s.nets:
        n.close()
    s.d.close()


def test_embed_hint_vs_oracle(S):
    got = S.nets[0].embed_hint(S.h[0])
    ref = O.hint_embedding(TINY_CONTROLNET, S.wcf[0], S.h[0])
    assert got.shape == ref.shape
    assert rel_err(got, ref) <= FWD_TOL


def test_forward_vs_oracle_and_not_vacuous(S):
    S.d.set_controls([(S.nets[0], S.h[0], 1.0)])
    got = S.fwd()
    ref = S.oracle_fwd([(0, 0, 1.0)])
    e = rel_err(got, ref)
    moved = rel_err(got, S.base)
    print(f"one control: forward rel err vs oracle {e:.2e}; the control moves the output by {moved:.2e}")
    assert e <= FWD_TOL
    assert moved > 0.05
    S.d.set_controls([])


def test_two_controls_vs_oracle(S):
    S.d.set_controls([(S.nets[0], S.h[0], 0.7), (S.nets[1], S.h[1], 1.3)])
    got = S.fwd()
    ref = S.oracle_fwd([(0, 0, 0.7), (1, 1, 1.3)])
    assert rel_err(got, ref) <= FWD_TOL
    S.d.set_controls([])


def test_detach_is_bit_identical(S):
    S.fwd()
    n = plan_builds(S.d)
    S.d.set_controls([(S.nets[0], S.h[0], 1.0)])
    controlled = S.fwd()
    assert S.d.plan_num_ops > S.base_ops
    assert plan_builds(S.d) == n + 1          # attaching drops the plan: rebuilt once
    S.d.set_controls([])
    assert torch.equal(S.fwd(), S.base)
    assert S.d.plan_num_ops == S.base_ops
    assert plan_builds(S.d) == n + 2          # and so does detaching
    fresh = Diffuser(S.ctx, TINY, S.w)
    assert torch.equal(fresh.unet_forward(X, [T], S.c, S.y), S.base)
    assert fresh.plan_num_ops == S.base_ops
    fresh.close()
    assert not torch.equal(controlled, S.base)


def test_rescale_in_place_matches_fresh_attach(S):
    S.d.set_controls([(S.nets[0], S.h[0], 0.5)])
    S.fwd()
    S.fwd()                                   # plan built and graph captured
    n_ops = S.d.plan_num_ops
    n_builds = plan_builds(S.d)
    S.d.set_controls([(S.nets[0], S.h[0], 1.0)])   # same net, n_hint, size: buffers rewritten in place
    rescaled = S.fwd()
    assert S.d.plan_num_ops == n_ops
    assert plan_builds(S.d) == n_builds            # the plan and its graph were kept
    S.d.set_controls([])
    S.d.set_controls([(S.nets[0], S.h[0], 1.0)])
    assert torch.equal(S.fwd(), rescaled)
    # new hint values in place
    S.d.set_controls([(S.nets[0], S.h[0].flip(3), 1.0)])
    flipped = S.fwd()
    S.d.set_controls([])
    S.d.set_controls([(S.nets[0], S.h[0].flip(3), 1.0)])
    assert torch.equal(S.fwd(), flipped)
    S.d.set_controls([])


def test_batch_rows_use_their_own_hint(S):
    h0, h1 = S.h[0][:1], S.h[0][1:]
    S.d.set_controls([(S.nets[0], torch.cat([h0, h1]), 1.0)])
    mixed = S.fwd()
    S.d.set_controls([(S.nets[0], torch.cat([h0, h0]), 1.0)])
    only0 = S.fwd()
    S.d.set_controls([(S.nets[0], h1, 1.0)])    # n_hint = 1: every row uses h1
    only1 = S.fwd()
    S.d.set_controls([])
    assert torch.equal(mixed[0], only0[0]) and torch.equal(mixed[1], only1[1])
    assert not torch.equal(mixed[0], only1[0])


def test_sample_cfg_vs_oracle(S):
    S.d.set_controls([(S.nets[0], S.h[0], 1.0)])
    got = S.d.sample_latent(Conditioning(**tiny_conditioning()), 7.5, 4, noise=S.noise)
    S.d.set_controls([])
    alphas = sdxl_b200.alphas_cumprod(TINY.n_steps)
    c = O.OracleConditioning(**tiny_conditioning())
    ref = O.sample_latent(TINY, S.wf, alphas, S.noise, c, 7.5, 4, att=O.Attach(controls=[(TINY_CONTROLNET, S.wcf[0], S.h[0], 1.0)]))
    assert rel_err(got, ref) <= SAMPLE_TOL


def test_inpainting_with_control(S):
    g = torch.Generator().manual_seed(5)
    ref_lat = torch.randn(2, 4, 16, 16, generator=g)
    mask = torch.rand(2, 4, 16, 16, generator=g) > 0.5
    step_noise = torch.randn(4, 2, 4, 16, 16, generator=g)
    cond = Conditioning(**tiny_conditioning())
    plain = S.d.sample_latent_with_inpainting(cond, 7.5, 4, ref_lat, mask, init_noise=S.noise, step_noise=step_noise)
    S.d.set_controls([(S.nets[0], S.h[0], 0.0)])   # scale 0 adds exact zeros
    zero = S.d.sample_latent_with_inpainting(cond, 7.5, 4, ref_lat, mask, init_noise=S.noise, step_noise=step_noise)
    S.d.set_controls([(S.nets[0], S.h[0], 1.0)])
    got = S.d.sample_latent_with_inpainting(cond, 7.5, 4, ref_lat, mask, init_noise=S.noise, step_noise=step_noise)
    S.d.set_controls([])
    assert torch.equal(zero, plain)
    alphas = sdxl_b200.alphas_cumprod(TINY.n_steps)
    want = O.sample_latent_with_inpainting(TINY, S.wf, alphas, S.noise, O.OracleConditioning(**tiny_conditioning()), 7.5, 4, ref_lat, mask,
                                           list(step_noise), att=O.Attach(controls=[(TINY_CONTROLNET, S.wcf[0], S.h[0], 1.0)]))
    assert rel_err(got, want) <= SAMPLE_TOL and not torch.equal(got, plain)


def test_validation_leaves_outputs_unchanged(S, ctx):
    S.d.set_controls([(S.nets[0], S.h[0], 1.0)])
    want = S.fwd()

    def unchanged():
        assert torch.equal(S.fwd(), want)

    other_cfg = ControlNetConfig(UNetConfig(adm_in_channels=16, model_channels=64, channel_mults=(1, 2, 4), transformer_depths=(0, 1, 2),
                                            context_dim=24))
    other = ControlNet(ctx, other_cfg, synth_weights(other_cfg, seed=4))
    with pytest.raises(SdxlError, match="adm_in_channels"):
        S.d.set_controls([(other, S.h[0], 1.0)])
    unchanged()
    other.close()
    with pytest.raises(SdxlError, match="n_hint"):
        S.d.set_controls([(S.nets[0], S.h[0][:0], 1.0)])
    unchanged()
    ctx2 = sdxl_b200.Context(0)
    foreign = ControlNet(ctx2, TINY_CONTROLNET, S.wc[0])
    with pytest.raises(SdxlError, match="another sdxl_ctx"):
        S.d.set_controls([(foreign, S.h[0], 1.0)])
    unchanged()
    foreign.close()
    ctx2.close()
    arr = (_lib.Control * 5)()
    for i in range(5):
        arr[i].net, arr[i].hint, arr[i].n_hint, arr[i].height, arr[i].width, arr[i].scale = S.nets[0].h.value, 1, 1, 128, 128, 1.0
    assert S.d.ctx.lib.sdxl_unet_set_controls(S.d.h, 5, arr) != 0
    unchanged()
    # forwards the attached control cannot serve
    with pytest.raises(SdxlError, match="latent"):
        S.d.unet_forward(arb(2, 4, 8, 8), [T], S.c, S.y)
    with pytest.raises(SdxlError, match="multiple of n_hint"):
        S.d.unet_forward(X[:1], [T], S.c[:1], S.y[:1])
    unchanged()
    S.d.set_controls([])


def test_pipeline_controls_attach_for_the_call(ctx):
    import os
    from sdxl_b200 import TINY_CLIP, TINY_OPEN_CLIP, TINY_VAE, ClipTextEncoder, Embedder, LatentDecoder, OpenClipTokenizer
    from sdxl_b200.pipeline import sample
    mini = os.path.join(os.path.dirname(__file__), "golden", "mini_bpe")
    ca, cb = TINY_CLIP, TINY_OPEN_CLIP
    ucfg = UNetConfig(adm_in_channels=cb.embed_dim + 6 * 256, model_channels=64, channel_mults=(1, 2, 4), transformer_depths=(0, 1, 1),
                      context_dim=ca.n_state + cb.n_state)
    ncfg = ControlNetConfig(ucfg, hint_block_channels=(8, 16, 24, 32))
    tok = OpenClipTokenizer(os.path.join(mini, "mini_merges.txt"), os.path.join(mini, "mini_vocab.txt"))
    emb = Embedder(ctx, ClipTextEncoder(ctx, ca, synth_weights(ca, seed=1)), ClipTextEncoder(ctx, cb, synth_weights(cb, seed=2)), tok, tok)
    dif = Diffuser(ctx, ucfg, synth_weights(ucfg, seed=3))
    vae = LatentDecoder(ctx, TINY_VAE, synth_weights(TINY_VAE, seed=0))
    net = ControlNet(ctx, ncfg, synth_weights(ncfg, seed=4))
    image = (torch.rand(1, 64, 64, 3, generator=torch.Generator().manual_seed(3)) * 255).to(torch.uint8)
    kw = dict(guidance=5.0, n_steps=4, resolution=(64, 64), seed=0)
    plain = sample(emb, dif, vae, "a photo of a cat", **kw)
    controlled = sample(emb, dif, vae, "a photo of a cat", controls=[(net, image, 1.0)], **kw)
    dif.set_controls([(net, image, 1.0)])          # u8 [n, H, W, 3] and f32 [n, 3, H, W] / 255 are the same hint
    same = sample(emb, dif, vae, "a photo of a cat", **kw)
    dif.set_controls([(net, image.permute(0, 3, 1, 2).float() / 255.0, 1.0)])
    assert torch.equal(sample(emb, dif, vae, "a photo of a cat", **kw), same)
    dif.set_controls([])
    assert torch.equal(controlled, same) and not torch.equal(controlled, plain)
    assert torch.equal(sample(emb, dif, vae, "a photo of a cat", **kw), plain)   # detached after the call
    net.close()
    dif.close()
