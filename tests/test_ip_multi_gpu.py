"""GPU tests of image-prompt sets (sdxl_unet_set_image_prompts, DESIGN.md §13): the N-source attention kernel and the mask resize
kernel against float64 / torch, tiny UNet forwards and a CFG sample against oracle/unet_oracle.py with the bounds of
tests/test_ip_adapter_gpu.py, and the bit-exact identities of the one-prompt path, detach, zero scales and in-place rewrites."""
import pytest
import torch
import torch.nn.functional as F

from sdxl_b200 import TINY, Conditioning, Diffuser, IPAdapter, SdxlError, alphas_cumprod, synth_weights
from sdxl_b200.ip_adapter import ResamplerConfig, synth_ip_adapter
from oracle import unet_oracle as O
import ip_adapter_oracle as IPO
import ip_adapter_plus_oracle as PO
import ip_multi_oracle as MO
from harness import arb, h16f, plan_builds, rel_err

pytestmark = pytest.mark.gpu
FWD_TOL = 2e-3
SAMPLE_TOL = 5e-3
T = 499
D = 32                                  # image_embed_dim of the tiny base adapter
DP, LP = 40, 19                         # the tiny Plus adapter's feature width and rows
R = ResamplerConfig(depth=2, heads=2, tokens=16)


def embeds(nb, ni, seed):
    return torch.randn(nb, ni, D, generator=torch.Generator().manual_seed(seed))


def feats(nb, ni, seed):
    return torch.randn(nb, ni, LP, DP, generator=torch.Generator().manual_seed(seed))


def halves(ni, H=128, W=128):
    """Image i of ni covers the i-th vertical strip of the H x W pixels."""
    m = torch.zeros(ni, H, W)
    for i in range(ni):
        m[i, :, i * W // ni:(i + 1) * W // ni] = 1
    return m


# ---------------------------------------------------------------------------------------------------------------------- kernels
def _ref_attention(q, k, v, sources, n_head):
    B, Tq, C = q.shape
    split = lambda t: t.double().reshape(B, t.shape[1], n_head, 64).transpose(1, 2)  # noqa: E731

    def att(k, v):
        s = split(q) @ split(k).transpose(-1, -2) / 8
        return (torch.softmax(s, -1) @ split(v)).transpose(1, 2).reshape(B, Tq, C)
    h = att(k, v)
    for kv, S, s, m in sources:
        a = s * att(kv[:, :, :C].reshape(B, S, C), kv[:, :, C:].reshape(B, S, C))
        h = h + (a if m is None else a * m.double()[None, :, None])
    return h


@pytest.mark.parametrize("n_src,Ss,Tq", [(1, [4], 200), (2, [16, 144], 256), (3, [4, 16, 144], 333), (8, [4, 16, 144, 4, 16, 4, 16, 4], 130)])
def test_attention_multi_kernel(n_src, Ss, Tq):
    """Against float64 softmaxes of the same f16 inputs. Masks hold 0, 1 and the bicubic overshoot range (-0.1, 1.1); source 1 of
    the 3- and 8-source cases has scale 0. Bound: P and O round to f16 (2^-11 relative) in each of the n_src + 1 softmaxes."""
    from sdxl_b200 import _testing as TL
    g = torch.Generator().manual_seed(n_src * 1000 + Tq)
    B, S, n_head = 2, 77, 3
    C = 64 * n_head
    q = torch.randn(B, Tq, C, generator=g).half().cuda()
    kv = torch.randn(B, S, 2 * C, generator=g).half().cuda()
    sources, ref_src = [], []
    for i, Sk in enumerate(Ss):
        skv = torch.randn(B, Sk, 2 * C, generator=g).half().cuda()
        s = 0.0 if (i == 1 and n_src >= 3) else 0.5 + 0.25 * i
        m = None
        if i % 2 == 1 or n_src == 1:
            m = torch.cat([torch.zeros(Tq // 3), torch.ones(Tq // 3), torch.linspace(-0.1, 1.1, Tq - 2 * (Tq // 3))])
            m = m[torch.randperm(Tq, generator=g)]
        sources.append((skv, 2 * C, 0, C, Sk, torch.tensor([s], device="cuda"), None if m is None else m.cuda()))
        ref_src.append((skv.cpu(), Sk, s, m))
    out = torch.full((B, Tq, C), float("nan"), dtype=torch.float16, device="cuda")
    TL.attention_multi(q, C, 0, kv, 2 * C, 0, C, B, Tq, S, n_head, out, C, sources)
    torch.cuda.synchronize()
    ref = _ref_attention(q.cpu(), kv[:, :, :C].cpu(), kv[:, :, C:].cpu(), ref_src, n_head)
    err = rel_err(out, ref)
    print(f"{n_src} sources: rel err {err:.3e}")
    assert err < 2e-3 and bool(torch.isfinite(out).all())
    if n_src == 1:   # the single-source form of the test launcher is the same kernel launch
        src = sources[0]
        out1 = torch.empty_like(out)
        TL.attention(q, C, 0, kv, 2 * C, 0, C, B, Tq, S, n_head, out1, C, src[0], 2 * C, 0, C, src[4], src[5])
        one = torch.empty_like(out)
        TL.attention_multi(q, C, 0, kv, 2 * C, 0, C, B, Tq, S, n_head, one, C, [src[:6] + (None,)])
        assert torch.equal(out1, one)


@pytest.mark.parametrize("H,W,mh,mw,Tq", [(128, 128, 16, 16, 256), (832, 1216, 26, 38, 988), (1216, 832, 78, 52, 4096), (64, 8, 5, 1, 2)])
def test_mask_resize_kernel(H, W, mh, mw, Tq):
    """Against torch's F.interpolate(mode="bicubic") on the GPU, padded or cut to Tq, within f32 rounding of the 16-tap sum."""
    from sdxl_b200 import _testing as TL
    m = (torch.rand(H, W, generator=torch.Generator().manual_seed(H * W)) > 0.5).float().cuda()
    got = TL.ip_mask_resize(m, mh, mw, Tq)
    full = F.interpolate(m[None, None], size=(mh, mw), mode="bicubic", align_corners=False).reshape(-1)
    want = torch.zeros(Tq, device="cuda")
    n = min(Tq, mh * mw)
    want[:n] = full[:n]
    assert float((got - want).abs().max()) < 1e-5


# ---------------------------------------------------------------------------------------------------------------------- UNet
class Setup:
    def __init__(self, ctx):
        self.ctx = ctx
        self.w = synth_weights(TINY, seed=0)
        self.wf = O.to_f32(self.w)
        self.d = Diffuser(ctx, TINY, self.w)
        self.wa = synth_ip_adapter(TINY, D, seed=3)
        self.waf = O.to_f32(self.wa)
        self.ad = IPAdapter(ctx, TINY, D, self.wa)
        self.wp = synth_ip_adapter(TINY, DP, seed=5, resampler=R)
        self.wpf = O.to_f32(self.wp)
        self.plus = IPAdapter(ctx, TINY, DP, self.wp)
        self.x = arb(2, 4, 16, 16)
        self.c = h16f(arb(2, 7, TINY.context_dim))
        self.y = h16f(arb(2, TINY.adm_in_channels))

    def fwd(self, x=None):
        return self.d.unet_forward(self.x if x is None else x, [T], self.c, self.y).cpu()

    def base_item(self, e, s, mask=None):
        return (self.ad, e, s, None, mask), (self.waf, IPO.prompt_tokens(self.waf, e), s, mask)

    def plus_item(self, h, s, mask=None):
        return (self.plus, h, s, torch.zeros_like(h), mask), (self.wpf, PO.plus_prompt_tokens(self.wpf, h), s, mask)

    def ref(self, items):
        prompts = [(wa, tok[torch.arange(2) % tok.shape[0]], IPO.uniform_scales(TINY, s), MO.binarize(m)) for wa, tok, s, m in items]
        return O.unet_forward(TINY, self.wf, self.x, torch.tensor([T]), self.c, self.y, O.Attach(prompts=prompts))


@pytest.fixture(scope="module")
def S(ctx):
    s = Setup(ctx)
    yield s
    s.d.set_image_prompts([])
    s.ad.close()
    s.plus.close()
    s.d.close()


@pytest.mark.parametrize("case", ["base_plus", "masked_2", "mixed_nb1", "mixed_nb2"])
def test_forward_against_oracle(S, case):
    if case == "base_plus":
        items = [S.base_item(embeds(2, 1, 1), 0.8), S.plus_item(feats(1, 2, 2), 0.6)]
    elif case == "masked_2":
        items = [S.base_item(embeds(1, 2, 3), 1.0, halves(2))]
    elif case == "mixed_nb1":
        items = [S.plus_item(feats(1, 1, 4), 0.7), S.base_item(embeds(1, 2, 5), 0.9, halves(2)), S.base_item(embeds(1, 1, 6), 0.5)]
    else:
        items = [S.base_item(embeds(2, 2, 7), 0.9, halves(2)), S.plus_item(feats(2, 3, 8), 0.8, halves(3))]
    S.d.set_image_prompts([a for a, _ in items])
    out = S.fwd()
    S.d.set_image_prompts([])
    err = rel_err(out, S.ref([b for _, b in items]))
    print(f"{case}: rel err {err:.3e}")
    assert err < FWD_TOL


def test_cfg_sample_against_oracle(S):
    kw = dict(context_full=h16f(arb(2, 7, TINY.context_dim) * 0.9), unconditional_context_full=h16f(arb(7, TINY.context_dim).cos()),
              channel_context=h16f(arb(2, TINY.adm_in_channels)), unconditional_channel_context=h16f(arb(TINY.adm_in_channels).cos()),
              resolution=(128, 128))
    noise = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(0))
    e, h = embeds(1, 2, 20), feats(1, 1, 21)
    neg = embeds(1, 2, 22)
    hn = feats(1, 1, 23)
    S.d.set_image_prompts([(S.ad, e, 0.9, neg, halves(2)), (S.plus, h, 0.7, hn, None)])
    try:
        out = S.d.sample_latent(Conditioning(**kw), 7.5, 4, noise=noise).cpu()
    finally:
        S.d.set_image_prompts([])
    att = O.Attach(prompts=[(S.waf, IPO.prompt_tokens(S.waf, e), IPO.uniform_scales(TINY, 0.9), halves(2)),
                            (S.wpf, PO.plus_prompt_tokens(S.wpf, h), IPO.uniform_scales(TINY, 0.7), None)],
                   uncond_tokens=[IPO.prompt_tokens(S.waf, neg), PO.plus_prompt_tokens(S.wpf, hn)])
    ref = O.sample_latent(TINY, S.wf, alphas_cumprod(TINY.n_steps), noise, O.OracleConditioning(**kw), 7.5, 4, att=att)
    err = rel_err(out, ref)
    print(f"4-step CFG sample: rel err {err:.3e}")
    assert err < SAMPLE_TOL


def test_bit_identities(S):
    none = S.fwd()
    e, h = embeds(2, 1, 30), feats(1, 1, 31)
    S.d.set_image_prompt(S.ad, e, 0.8)
    one = S.fwd()
    S.d.set_image_prompts([(S.ad, e, 0.8, None, None)])
    assert torch.equal(S.fwd(), one)                             # one host path
    S.d.set_image_prompts([(S.ad, e, 0.8, None, None), (S.plus, h, 0.0, torch.zeros_like(h), halves(1))])
    assert torch.equal(S.fwd(), one)                             # an all-zero-scale prompt is its absence
    S.d.set_image_prompts([(S.ad, e, 0.8, None, None), (S.plus, h, 0.0, torch.zeros_like(h), None)])
    assert torch.equal(S.fwd(), one)
    S.d.set_image_prompts([])
    assert torch.equal(S.fwd(), none)                            # detaching is never attaching
    S.d.set_image_prompt(None)


def test_rewrite_keeps_plan(S):
    e1, e2 = embeds(1, 2, 40), embeds(1, 2, 41)
    h = feats(1, 1, 42)
    S.d.set_image_prompts([(S.ad, e1, 0.5, None, halves(2)), (S.plus, h, 0.6, torch.zeros_like(h), None)])
    S.fwd()
    b = plan_builds(S.d)
    flipped = halves(2).flip(0)
    S.d.set_image_prompts([(S.ad, e2, 1.3, None, flipped), (S.plus, h, 0.2, torch.zeros_like(h), None)])
    out = S.fwd()
    assert plan_builds(S.d) == b                                  # same adapters, shapes and mask sizes: rewritten in place
    S.d.set_image_prompts([])
    S.d.set_image_prompts([(S.ad, e2, 1.3, None, flipped), (S.plus, h, 0.2, torch.zeros_like(h), None)])
    assert torch.equal(S.fwd(), out)                              # the rewrite equals a fresh attach
    assert plan_builds(S.d) == b + 1
    S.d.set_image_prompts([])


def test_refused_calls_leave_set(S, ctx):
    e = embeds(2, 1, 50)
    S.d.set_image_prompts([(S.ad, e, 0.7, None, None), (S.ad, embeds(1, 2, 51), 0.5, None, halves(2))])
    ref = S.fwd()
    with pytest.raises(SdxlError, match="n_batch"):
        S.d.set_image_prompts([(S.ad, e, 0.1, None, None), (S.ad, embeds(3, 1, 52), 1.0, None, None)])   # 3 does not divide 2
    with pytest.raises(SdxlError, match="not finite"):
        S.d.set_image_prompts([(S.ad, e, 0.1, None, None), (S.ad, e, float("nan"), None, None)])
    assert torch.equal(S.fwd(), ref)
    with pytest.raises(SdxlError, match="latent"):
        S.fwd(arb(2, 4, 8, 8))                                    # the masks cover a 16 x 16 latent
    assert torch.equal(S.fwd(), ref)
    S.d.set_image_prompts([])
