"""GPU tests of the inpainting UNet (sdxl_unet_set_inpaint_condition and the two-source first conv), tiny configs: the kernel against
float64, forwards and CFG samples against the f32 oracle (oracle/unet_oracle.py) with the bounds of tests/test_unet_gpu.py, the
in-place rewrite, every refusal, the diffusers loader and the `sample` flow."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

import sdxl_b200
from sdxl_b200 import (TINY, TINY_CLIP, TINY_INPAINT, TINY_OPEN_CLIP, TINY_VAE, ClipTextEncoder, Conditioning, Diffuser, Embedder,
                       LatentDecoder, OpenClipTokenizer, SdxlError, UNetConfig, synth_weights)
from sdxl_b200 import _lib
from sdxl_b200 import _testing as KT
from sdxl_b200.diffusers_unet import from_diffusers, name_map
from oracle import clip_oracle as CO
from oracle import tokenizer_oracle as TO
from oracle import unet_oracle as O
from oracle import vae_oracle as VO
import inpaint_oracle as IO
from harness import arb, h16f, plan_builds, rel_err, tiny_conditioning

pytestmark = pytest.mark.gpu
FWD_TOL = 2e-3
SAMPLE_TOL = 5e-3
T = 499
U24 = 2.0 ** -24
MINI = os.path.join(os.path.dirname(__file__), "golden", "mini_bpe")


def condition(n, seed, h=16, w=16):
    g = torch.Generator().manual_seed(seed)
    mask = (torch.rand(n, 1, h, w, generator=g) < 0.4).float()
    return torch.cat([mask, torch.randn(n, 4, h, w, generator=g) * (1 - mask)], dim=1)


X = arb(2, 4, 16, 16)


@pytest.mark.parametrize("x_f32", [0, 1])
@pytest.mark.parametrize("W", [8, 13])
@pytest.mark.parametrize("n2", [1, 4])
def test_conv_in_cat(ctx, x_f32, W, n2):
    """The two-source first conv against float64, with test_conv_in's bound: channels [0, 4) from the latent x (Bx = 1 broadcast to
    B = 4), [4, 9) from the f32 condition x2 (image b % n2)."""
    g = torch.Generator().manual_seed(x_f32 + W + n2)
    Bx, B, H, C1, C2, Cout = 1, 4, 6, 4, 5, 320
    Cin = C1 + C2
    x = torch.randn(Bx, C1, H, W, generator=g)
    x = x.cuda() if x_f32 else x.cuda().half()
    x2 = torch.randn(n2, C2, H, W, generator=g).cuda()
    w = (torch.randn(Cout, Cin, 3, 3, generator=g) / math.sqrt(9 * Cin)).cuda()
    wk = w.permute(0, 2, 3, 1).contiguous()                             # [Cout][kh][kw][Cin]
    bias = (torch.randn(Cout, generator=g) * 0.1).cuda()
    y = torch.full((B, H, W, Cout), float("nan"), device="cuda")
    KT.conv_in_cat(x, Bx, B, C1, x2, n2, C2, H, W, wk, bias, Cout, y)
    xin = torch.cat([x.double()[[b % Bx for b in range(B)]], x2.double()[[b % n2 for b in range(B)]]], dim=1)
    ref = F.conv2d(xin, w.double(), bias.double(), padding=1).permute(0, 2, 3, 1)
    mag = F.conv2d(xin.abs(), w.double().abs(), bias.double().abs(), padding=1).permute(0, 2, 3, 1)
    err, tol = (y.double() - ref).abs(), (9 * Cin + 2) * U24 * mag
    print(f"conv_in_cat x_f32={x_f32} W={W} n2={n2}: max err {float(err.max()):.3e}, worst err / bound {float((err / tol).max()):.3f}")
    assert not bool((err > tol).any())


class Setup:
    def __init__(self, ctx):
        self.ctx = ctx
        self.w = synth_weights(TINY_INPAINT, seed=0)
        self.wf = O.to_f32(self.w)
        self.d = Diffuser(ctx, TINY_INPAINT, self.w)
        self.c = h16f(arb(2, 7, TINY.context_dim))
        self.y = h16f(arb(2, TINY.adm_in_channels))
        self.cond = [condition(1, 10), condition(2, 11)]
        self.noise = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(0))

    def fwd(self, x=X, t=T):
        return self.d.unet_forward(x, [t], self.c[:x.shape[0]], self.y[:x.shape[0]])

    def oracle_fwd(self, cond, t=T):
        return O.unet_forward(TINY_INPAINT, self.wf, X, torch.tensor([t]), self.c, self.y, O.Attach(concat=cond))


@pytest.fixture(scope="module")
def S(ctx):
    s = Setup(ctx)
    yield s
    s.d.set_inpaint_condition(None)
    s.d.close()


@pytest.mark.parametrize("k", [0, 1], ids=["n1", "nB"])
def test_forward_vs_oracle(S, k):
    S.d.set_inpaint_condition(S.cond[k])
    got = S.fwd()
    ref = S.oracle_fwd(S.cond[k])
    e = rel_err(got, ref)
    print(f"n = {S.cond[k].shape[0]}: forward rel err vs oracle {e:.2e}")
    assert got.shape == X.shape and e <= FWD_TOL


def test_sample_cfg_vs_oracle(S):
    S.d.set_inpaint_condition(S.cond[1])
    got = S.d.sample_latent(Conditioning(**tiny_conditioning()), 7.5, 4, noise=S.noise)
    ref = O.sample_latent(TINY_INPAINT, S.wf, sdxl_b200.alphas_cumprod(TINY.n_steps), S.noise,
                          O.OracleConditioning(**tiny_conditioning()), 7.5, 4, att=O.Attach(concat=S.cond[1]))
    e = rel_err(got, ref)
    print(f"CFG sample (batch 2, 4 steps) rel err vs oracle {e:.2e}")
    assert got.shape == S.noise.shape and e <= SAMPLE_TOL


def test_rewrite_in_place_matches_fresh_attach(S):
    S.d.set_inpaint_condition(S.cond[1])
    S.fwd()
    S.fwd()                                                 # plan built and graph captured
    n = plan_builds(S.d)
    others = [condition(2, 20), condition(2, 21)]
    results = []
    for c in others:
        S.d.set_inpaint_condition(c)                        # same n and size: rewritten in place
        results.append(S.fwd())
        assert plan_builds(S.d) == n
    assert not torch.equal(results[0], results[1])
    for c, want in zip(others, results):
        S.d.set_inpaint_condition(None)
        S.d.set_inpaint_condition(c)
        assert torch.equal(S.fwd(), want)
    S.d.set_inpaint_condition(S.cond[0])                    # a new n: a new plan
    S.fwd()
    assert plan_builds(S.d) > n


def test_batch_rows_use_their_own_condition(S):
    S.d.set_inpaint_condition(S.cond[1])
    mixed = S.fwd()
    S.d.set_inpaint_condition(S.cond[1][:1])
    only0 = S.fwd()
    S.d.set_inpaint_condition(S.cond[1][1:])
    only1 = S.fwd()
    assert torch.equal(mixed[0], only0[0]) and torch.equal(mixed[1], only1[1]) and not torch.equal(mixed[0], only1[0])


def test_refusals_leave_the_previous_state(S):
    S.d.set_inpaint_condition(S.cond[1])
    want = S.fwd()
    n = plan_builds(S.d)

    def unchanged():
        assert torch.equal(S.fwd(), want) and plan_builds(S.d) == n

    with pytest.raises(SdxlError, match="5 channels"):
        S.d.set_inpaint_condition(condition(2, 3)[:, :4])
    unchanged()
    s = _lib.InpaintCondition()
    s.cond, s.on_host, s.n, s.height, s.width = None, 0, 2, 128, 128
    with pytest.raises(SdxlError, match="null cond"):
        S.ctx.check(S.ctx.lib.sdxl_unet_set_inpaint_condition(S.d.h, s), "set")
    unchanged()
    keep = condition(2, 4).cuda()
    s.cond = keep.data_ptr()
    for field, value, msg in (("n", 0, "n = 0"), ("height", 100, "multiple of 8"), ("width", 0, "multiple of 8")):
        bad = _lib.InpaintCondition(s.cond, 0, s.n, s.height, s.width)
        setattr(bad, field, value)
        with pytest.raises(SdxlError, match=msg):
            S.ctx.check(S.ctx.lib.sdxl_unet_set_inpaint_condition(S.d.h, bad), "set")
        unchanged()
    # forwards and samples the attached condition cannot serve
    with pytest.raises(SdxlError, match="latent"):
        S.d.unet_forward(arb(2, 4, 8, 8), [T], S.c, S.y)
    with pytest.raises(SdxlError, match="latent"):
        S.d.sample_latent(Conditioning(**tiny_conditioning(res=(64, 64))), 7.5, 2, noise=S.noise[:, :, :8, :8])
    with pytest.raises(SdxlError, match="multiple of its n"):
        S.d.sample_latent(Conditioning(**tiny_conditioning(B=1)), 7.5, 2, noise=S.noise[:1])
    unchanged()
    with pytest.raises(SdxlError, match="multiple of its n"):
        S.fwd(X[:1])                                        # (its conditioning, set for batch 1 first, drops the plan)
    assert torch.equal(S.fwd(), want)
    # nothing attached
    S.d.set_inpaint_condition(None)
    with pytest.raises(SdxlError, match="no inpainting condition"):
        S.fwd()
    with pytest.raises(SdxlError, match="no inpainting condition"):
        S.d.sample_latent(Conditioning(**tiny_conditioning()), 7.5, 2, noise=S.noise)
    S.d.set_inpaint_condition(S.cond[1])
    assert torch.equal(S.fwd(), want)


def test_four_channel_unet_refuses_and_is_unchanged(ctx):
    w = synth_weights(TINY, seed=0)
    d = Diffuser(ctx, TINY, w)
    c, y = h16f(arb(2, 7, TINY.context_dim)), h16f(arb(2, TINY.adm_in_channels))
    before = d.unet_forward(X, [T], c, y)
    with pytest.raises(SdxlError, match="inpainting layout"):
        d.set_inpaint_condition(condition(1, 0))
    d.set_inpaint_condition(None)                           # nothing attached: detaching is a no-op
    assert torch.equal(d.unet_forward(X, [T], c, y), before)
    d.close()


def test_diffusers_named_weights_forward_bit_identically(ctx):
    w = synth_weights(TINY, seed=2)
    sd = {src: (w[dst].t().contiguous() if lin else w[dst]) for src, (dst, lin) in name_map(TINY).items()}
    js = {"down_block_types": ["DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"],
          "up_block_types": ["CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"], "block_out_channels": [64, 128, 256],
          "attention_head_dim": [1, 2, 4], "transformer_layers_per_block": [1, 1, 2], "cross_attention_dim": 24,
          "projection_class_embeddings_input_dim": 8, "addition_embed_type": "text_time", "use_linear_projection": True,
          "in_channels": 4, "out_channels": 4}
    cfg, wd = from_diffusers(sd, js)
    assert cfg == TINY
    c, y = h16f(arb(2, 7, TINY.context_dim)), h16f(arb(2, TINY.adm_in_channels))
    outs = []
    for weights in (w, wd):
        d = Diffuser(ctx, cfg, weights)
        outs.append(d.unet_forward(X, [T], c, y))
        d.close()
    assert torch.equal(outs[0], outs[1])


def test_pipeline_sample_vs_oracle_chain(ctx):
    ca, cb = TINY_CLIP, TINY_OPEN_CLIP
    ucfg = UNetConfig(adm_in_channels=cb.embed_dim + 6 * 256, model_channels=64, channel_mults=(1, 2, 4), transformer_depths=(0, 1, 1),
                      context_dim=ca.n_state + cb.n_state, in_channels=9)
    wa, wb, wu, wv = (synth_weights(cfg, seed=s) for cfg, s in ((ca, 1), (cb, 2), (ucfg, 3), (TINY_VAE, 0)))
    tok = OpenClipTokenizer(os.path.join(MINI, "mini_merges.txt"), os.path.join(MINI, "mini_vocab.txt"))
    emb = Embedder(ctx, ClipTextEncoder(ctx, ca, wa), ClipTextEncoder(ctx, cb, wb), tok, tok)
    dif = Diffuser(ctx, ucfg, wu)
    vae = LatentDecoder(ctx, TINY_VAE, wv)
    text, res = "a photo of a cat", (32, 32)
    rgb = torch.randint(0, 256, (1, 32, 32, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(1))
    noise = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(0))
    crop = (5, 27, 3, 19)
    img = sdxl_b200.sample(emb, dif, vae, text, guidance=5.0, n_steps=4, reference_rgb=rgb, crop=crop, crop_out=True, noise=noise)
    with pytest.raises(SdxlError, match="reference_rgb"):
        sdxl_b200.sample(emb, dif, vae, text, guidance=5.0, n_steps=4, resolution=res, noise=noise)
    with pytest.raises(SdxlError, match="no inpainting condition"):   # detached after the call
        dif.unet_forward(torch.zeros(1, 4, 8, 8), [T], torch.zeros(1, 7, ucfg.context_dim), torch.zeros(1, ucfg.adm_in_channels))
    # oracle chain: text -> conditioning; image + crop window -> condition; DDIM / CFG with the condition; decode
    otok = TO.OpenClipTokenizer(os.path.join(MINI, "mini_merges.txt"), os.path.join(MINI, "mini_vocab.txt"))
    oc = CO.text_to_conditioning(ca, O.to_f32(wa), cb, O.to_f32(wb), otok, otok, TO.tokenize_text, text, res, (0, 0), res)
    ocond = O.OracleConditioning(context_full=h16f(oc["context_full"]), unconditional_context_full=h16f(oc["unconditional_context_full"]),
                                 channel_context=h16f(oc["channel_context"]),
                                 unconditional_channel_context=h16f(oc["unconditional_channel_context"]), resolution=(64, 64))
    wvf = O.to_f32(wv)
    mask = IO.pixel_mask(32, 32, *crop, True)
    cond = IO.condition(rgb, mask, lambda im: VO.encode_image(TINY_VAE, wvf, im), 4)
    olat = O.sample_latent(ucfg, O.to_f32(wu), sdxl_b200.alphas_cumprod(), noise, ocond, 5.0, 4, att=O.Attach(concat=cond))
    oimg = VO.latent_to_image(TINY_VAE, wvf, olat).numpy().astype("int32")
    # the library's own condition and latent on the same path
    dcond = sdxl_b200.prepare_inpaint_condition(vae, rgb, sdxl_b200.make_inpaint_mask((32, 32), (32, 32), *crop, crop_out=True, n_channels=1))
    ec = rel_err(dcond, cond)
    diff = (img.cpu().numpy().astype("int32") - oimg)
    diff = abs(diff)
    print(f"sample(): condition rel err {ec:.2e}; image max diff {diff.max()}, within 1: {(diff <= 1).mean():.4f}")
    assert ec <= FWD_TOL and diff.max() <= 3 and (diff <= 1).mean() >= 0.99
    for o in (emb.clip, emb.open_clip, dif, vae):
        o.close()
