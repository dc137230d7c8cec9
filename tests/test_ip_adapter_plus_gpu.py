"""GPU tests of IP-Adapter Plus image prompts: the perceiver LayerNorm kernel against float64, the Resampler
(sdxl_ip_adapter_resample) against the f32 oracle of tests/ip_adapter_plus_oracle.py, tiny UNet forwards and CFG samples with a Plus prompt
against the oracle with the bounds of tests/test_ip_adapter_gpu.py, and the bit-exact identities of attach / detach / rewrite."""
import ctypes as C

import pytest
import torch

from sdxl_b200 import TINY, Conditioning, Diffuser, IPAdapter, SdxlError, UNetConfig, alphas_cumprod, synth_weights
from sdxl_b200 import _lib
from sdxl_b200.ip_adapter import ResamplerConfig, synth_ip_adapter
from oracle import unet_oracle as O
import ip_adapter_oracle as IPO
import ip_adapter_plus_oracle as PO
from harness import arb, h16f, plan_builds, rel_err, tiny_conditioning

pytestmark = pytest.mark.gpu
FWD_TOL = 2e-3      # the UNet forward bound of test_unet_gpu / test_ip_adapter_gpu
SAMPLE_TOL = 5e-3   # the 4-step CFG sample bound of the same files
# Resampler tokens: the final LayerNorm's output is f16 (2^-12 relative RMS rounding), and the chain before it rounds a GEMM operand
# to f16 about 8 times per layer plus twice outside the layers (each 2^-12 RMS relative, independent): sqrt(2 * 8 + 3) * 2^-12
# ~ 1.1e-3 normwise for depth 2, doubled for the softmax / LayerNorm amplification of input errors.
RESAMPLE_TOL = 2.5e-3
T = 499
D = 40                                      # width of the tiny image features (a multiple of 8, not of 64)
L = 19                                      # hidden-state rows per image
R = ResamplerConfig(depth=2, heads=2, tokens=16)


def feats(nb, ni, seed):
    return torch.randn(nb, ni, L, D, generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("n,Lr,Q,Cw", [(2, 257, 16, 1280), (3, 17, 4, 128), (1, 1, 1, 64)])
def test_perceiver_ln_kernel(n, Lr, Q, Cw):
    """Against float64 on the same f32 inputs. Elementwise bound: the f16 output rounding (half an ulp, 2^-11 relative) plus the f32
    two-pass statistics (mean and centred sum over Cw <= 1280 terms: relative error of rstd and mean below Cw * 2^-24 < 8e-5 of the
    row scale, times |gamma| * |x - mean| * rstd <= 5 on these rows: 4e-4 absolute)."""
    from sdxl_b200 import _testing as TL
    g = torch.Generator().manual_seed(n * 1000 + Lr)
    x = (torch.randn(n * Lr, Cw, generator=g) * 3 + 1).cuda()
    lat = (torch.randn(n * Q, Cw, generator=g) * 0.2 - 0.5).cuda()
    g1, b1, g2, b2 = (1 + 0.1 * torch.randn(Cw, generator=g)).cuda(), (0.1 * torch.randn(Cw, generator=g)).cuda(), \
        (1 + 0.1 * torch.randn(Cw, generator=g)).cuda(), (0.1 * torch.randn(Cw, generator=g)).cuda()
    kv = torch.full((n, Lr + Q, Cw), float("nan"), dtype=torch.float16, device="cuda")
    q = torch.full((n * Q, Cw), float("nan"), dtype=torch.float16, device="cuda")
    TL.perceiver_ln(x, lat, n, Lr, Q, Cw, g1, b1, g2, b2, 1e-5, kv, q)
    torch.cuda.synchronize()
    ln = lambda t, ga, be: torch.nn.functional.layer_norm(t.double(), (Cw,), ga.double(), be.double(), 1e-5)  # noqa: E731
    want = torch.cat([ln(x, g1, b1).reshape(n, Lr, Cw), ln(lat, g2, b2).reshape(n, Q, Cw)], 1)
    d = (kv.double() - want).abs()
    assert bool((d <= want.abs() * 2.0 ** -11 + 4e-4).all()), float(d.max())
    assert torch.equal(q.reshape(n, Q, Cw), kv[:, Lr:])      # the to_q operand is the LN2 rows, bit for bit


class Setup:
    def __init__(self, ctx):
        self.ctx = ctx
        self.w = synth_weights(TINY, seed=0)
        self.wf = O.to_f32(self.w)
        self.d = Diffuser(ctx, TINY, self.w)
        self.wa = synth_ip_adapter(TINY, D, seed=5, resampler=R)
        self.waf = O.to_f32(self.wa)
        self.ad = IPAdapter(ctx, TINY, D, self.wa)
        self.base = IPAdapter(ctx, TINY, 32, synth_ip_adapter(TINY, 32, seed=3))
        self.x = arb(2, 4, 16, 16)
        self.c = h16f(arb(2, 7, TINY.context_dim))
        self.y = h16f(arb(2, TINY.adm_in_channels))

    def fwd(self):
        return self.d.unet_forward(self.x, [T], self.c, self.y).cpu()

    def attach(self, h, scale, neg=None):
        self.d.set_image_prompt(self.ad, h, scale, negative=torch.zeros_like(h) if neg is None else neg)

@pytest.fixture(scope="module")
def S(ctx):
    s = Setup(ctx)
    yield s
    s.d.set_image_prompt(None)
    s.ad.close()
    s.base.close()
    s.d.close()


def test_resample_against_oracle(S):
    assert S.ad.resampler == R
    h = feats(3, 1, 1)[:, 0]
    got = S.ad.resample(h).float().cpu()
    ref = PO.resample(S.waf, h).reshape(-1, TINY.context_dim)
    err = rel_err(got, ref)
    print(f"Resampler tokens: rel err {err:.3e}")
    assert err < RESAMPLE_TOL
    with pytest.raises(SdxlError, match="Plus"):
        S.ad.project(torch.zeros(1, D))                       # the base projection refuses a Plus adapter


@pytest.mark.parametrize("nb,ni", [(2, 1), (1, 2), (1, 9)])
def test_forward_against_oracle(S, nb, ni):
    """9 images give 144 image tokens: two 128-key blocks of the two-source attention."""
    h = feats(nb, ni, 7 + ni)
    S.attach(h, 0.8)
    out = S.fwd()
    S.d.set_image_prompt(None)
    tok = PO.plus_prompt_tokens(S.waf, h)[torch.arange(2) % nb]
    ref = O.unet_forward(TINY, S.wf, S.x, torch.tensor([T]), S.c, S.y, O.Attach(prompts=[(S.waf, tok, IPO.uniform_scales(TINY, 0.8), None)]))
    err = rel_err(out, ref)
    print(f"Plus forward n_batch={nb} n_images={ni}: rel err {err:.3e}")
    assert err < FWD_TOL


def test_cfg_sample_against_oracle(S):
    kw = tiny_conditioning()
    noise = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(0))
    h, neg = feats(1, 2, 20), feats(1, 2, 21) * 0.5
    S.attach(h, 0.9, neg)
    try:
        out = S.d.sample_latent(Conditioning(**kw), 7.5, 4, noise=noise).cpu()
    finally:
        S.d.set_image_prompt(None)
    c = O.OracleConditioning(**kw)
    ref = O.sample_latent(TINY, S.wf, alphas_cumprod(TINY.n_steps), noise, c, 7.5, 4, att=PO.attach(S.waf, h, neg, IPO.uniform_scales(TINY, 0.9)))
    err = rel_err(out, ref)
    print(f"Plus 4-step CFG sample: rel err {err:.3e}")
    assert err < SAMPLE_TOL


def test_detach_and_scale_zero_equal_no_prompt(S):
    base = S.fwd()
    S.attach(feats(2, 1, 1), 1.0)
    assert not torch.equal(S.fwd(), base)
    S.d.set_image_prompt(None)
    assert torch.equal(S.fwd(), base)
    S.attach(feats(2, 1, 2), 0.0)
    out = S.fwd()
    S.d.set_image_prompt(None)
    assert torch.equal(out, base)


def test_in_place_rewrite_equals_fresh_attach(S):
    h1, h2 = feats(2, 2, 3), feats(2, 2, 4)
    S.attach(h1, 0.5)
    S.fwd()
    S.fwd()                                 # the second run captures the CUDA graph
    n_builds = plan_builds(S.d)
    S.attach(h2, 1.3, h1)                   # same adapter, n_batch, n_images: buffers rewritten in place
    rewritten = S.fwd()
    assert plan_builds(S.d) == n_builds     # the plan (and its graph) was kept
    S.d.set_image_prompt(None)
    S.attach(h2, 1.3, h1)
    fresh = S.fwd()
    assert plan_builds(S.d) == n_builds + 1
    S.d.set_image_prompt(None)
    assert torch.equal(rewritten, fresh)


def test_switching_between_base_and_plus_rebuilds_the_plan(S):
    e = torch.randn(2, 1, 32, generator=torch.Generator().manual_seed(8))
    h = feats(2, 1, 9)
    S.d.set_image_prompt(S.base, e, 1.0)
    base_out = S.fwd()
    n_builds = plan_builds(S.d)
    S.attach(h, 1.0)
    plus_out = S.fwd()
    assert plan_builds(S.d) == n_builds + 1 and not torch.equal(plus_out, base_out)
    S.d.set_image_prompt(S.base, e, 1.0)
    assert torch.equal(S.fwd(), base_out) and plan_builds(S.d) == n_builds + 2
    S.d.set_image_prompt(None)
    S.attach(h, 1.0)
    assert torch.equal(S.fwd(), plus_out)
    S.d.set_image_prompt(None)


def _raw_prompt(S, h, neg, seq_len):
    """sdxl_unet_set_image_prompt through ctypes, so that a NULL negative or a wrong seq_len reaches the library."""
    ctx = S.ctx
    p = _lib.ImagePrompt()
    p.adapter, p.embeds, p.negative_embeds, p.on_host = S.ad.handle(), h.data_ptr(), None if neg is None else neg.data_ptr(), 1
    p.n_batch, p.n_images, p.scale, p.block_scales_host, p.seq_len = h.shape[0], h.shape[1], 1.0, None, seq_len
    ctx.enter()
    rc = ctx.lib.sdxl_unet_set_image_prompt(S.d.h, C.byref(p))
    ctx.leave()
    return rc, ctx.lib.sdxl_last_error(ctx.h).decode()


def test_null_negative_or_bad_seq_len_leaves_state(S):
    h = feats(2, 1, 30)
    S.attach(h, 1.0)
    ref = S.fwd()
    n_builds = plan_builds(S.d)
    other = feats(2, 1, 31).contiguous()
    rc, msg = _raw_prompt(S, other, None, L)
    assert rc != 0 and "negative" in msg
    for bad in (0, -3, 5000):
        rc, msg = _raw_prompt(S, other, torch.zeros_like(other), bad)
        assert rc != 0 and "seq_len" in msg
    assert torch.equal(S.fwd(), ref) and plan_builds(S.d) == n_builds
    with pytest.raises(SdxlError, match="negative"):
        S.d.set_image_prompt(S.ad, other, 1.0)
    assert torch.equal(S.fwd(), ref)
    S.d.set_image_prompt(None)


def test_pipeline_sample_with_plus_equals_manual_path(ctx):
    import os
    from sdxl_b200 import TINY_CLIP, TINY_OPEN_CLIP, TINY_VAE, ClipTextEncoder, Embedder, LatentDecoder, OpenClipTokenizer
    from sdxl_b200.clip_vision import TINY_VIT_80, ClipVisionEncoder, synth_vision_weights
    from sdxl_b200.pipeline import sample
    mini = os.path.join(os.path.dirname(__file__), "golden", "mini_bpe")
    ca, cb = TINY_CLIP, TINY_OPEN_CLIP
    ucfg = UNetConfig(adm_in_channels=cb.embed_dim + 6 * 256, model_channels=64, channel_mults=(1, 2, 4), transformer_depths=(0, 1, 1),
                      context_dim=ca.n_state + cb.n_state)
    tok = OpenClipTokenizer(os.path.join(mini, "mini_merges.txt"), os.path.join(mini, "mini_vocab.txt"))
    emb = Embedder(ctx, ClipTextEncoder(ctx, ca, synth_weights(ca, seed=1)), ClipTextEncoder(ctx, cb, synth_weights(cb, seed=2)), tok, tok)
    dif = Diffuser(ctx, ucfg, synth_weights(ucfg, seed=3))
    vae = LatentDecoder(ctx, TINY_VAE, synth_weights(TINY_VAE, seed=0))
    enc = ClipVisionEncoder(ctx, TINY_VIT_80, synth_vision_weights(TINY_VIT_80, seed=1))
    ad = IPAdapter(ctx, ucfg, TINY_VIT_80.n_state, synth_ip_adapter(ucfg, TINY_VIT_80.n_state, seed=6, resampler=R))
    images = (torch.rand(2, 70, 90, 3, generator=torch.Generator().manual_seed(3)) * 255).to(torch.uint8)
    kw = dict(guidance=5.0, n_steps=4, resolution=(64, 64), seed=0)
    plain = sample(emb, dif, vae, "a photo of a cat", **kw)
    prompted = sample(emb, dif, vae, "a photo of a cat", image_prompt=(ad, enc, images, 0.7), **kw)
    e, neg = ad.image_embeds(enc, images)
    assert e.shape == neg.shape == (2, TINY_VIT_80.n_tokens, TINY_VIT_80.n_state)
    dif.set_image_prompt(ad, e.unsqueeze(0), 0.7, negative=neg.unsqueeze(0))
    manual = sample(emb, dif, vae, "a photo of a cat", **kw)
    dif.set_image_prompt(None)
    assert torch.equal(prompted, manual) and not torch.equal(prompted, plain)
    assert torch.equal(sample(emb, dif, vae, "a photo of a cat", **kw), plain)   # detached after the call
    ad.close()
    enc.close()
    dif.close()
