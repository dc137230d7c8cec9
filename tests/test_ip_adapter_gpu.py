"""GPU tests of IP-Adapter image prompts (sdxl_unet_set_image_prompt, the two-source attention kernel), tiny configs, against the
f32 oracle (oracle/unet_oracle.py) with the bounds of tests/test_unet_gpu.py, plus the bit-exact identities of attach /
detach / rescale."""
import dataclasses

import pytest
import torch

from sdxl_b200 import (TINY, TINY_CONTROLNET, TINY_REFINER, Conditioning, ControlNet, Diffuser, IPAdapter, SdxlError, alphas_cumprod,
                       synth_weights)
from sdxl_b200.ip_adapter import synth_ip_adapter, transformer_block_paths
from oracle import unet_oracle as O
import ip_adapter_oracle as IPO
from harness import arb, h16f, plan_builds, rel_err, tiny_conditioning

pytestmark = pytest.mark.gpu
FWD_TOL = 2e-3
SAMPLE_TOL = 5e-3
ATTN_TOL = 2e-3
T = 499
D = 32   # image_embed_dim of the tiny adapter


def embeds(nb, ni, seed):
    return torch.randn(nb, ni, D, generator=torch.Generator().manual_seed(seed))


class Setup:
    def __init__(self, ctx):
        self.ctx = ctx
        self.w = synth_weights(TINY, seed=0)
        self.wf = O.to_f32(self.w)
        self.d = Diffuser(ctx, TINY, self.w)
        self.wa = synth_ip_adapter(TINY, D, seed=3)
        self.waf = O.to_f32(self.wa)
        self.ad = IPAdapter(ctx, TINY, D, self.wa)
        self.x = arb(2, 4, 16, 16)
        self.c = h16f(arb(2, 7, TINY.context_dim))
        self.y = h16f(arb(2, TINY.adm_in_channels))

    def fwd(self):
        return self.d.unet_forward(self.x, [T], self.c, self.y).cpu()

    def ref(self, e, scales):
        tok = IPO.prompt_tokens(self.waf, e)[torch.arange(2) % e.shape[0]]
        return O.unet_forward(TINY, self.wf, self.x, torch.tensor([T]), self.c, self.y, O.Attach(prompts=[(self.waf, tok, scales, None)]))


@pytest.fixture(scope="module")
def S(ctx):
    s = Setup(ctx)
    yield s
    s.d.set_image_prompt(None)
    s.ad.close()
    s.d.close()


def ip_attention(ctx, q, k, v, kip, vip, n_head, scale):
    q, k, v, kip, vip = (t.to(ctx.device, torch.float16).contiguous() for t in (q, k, v, kip, vip))
    B, Tq, Cc = q.shape
    out = torch.empty_like(q)
    ctx.enter()
    ctx.check(ctx.lib.sdxl_op_ip_attention(ctx.h, q.data_ptr(), k.data_ptr(), v.data_ptr(), kip.data_ptr(), vip.data_ptr(), B, Tq,
                                           k.shape[1], kip.shape[1], Cc, n_head, float(scale), out.data_ptr()), "sdxl_op_ip_attention")
    ctx.leave()
    return out


@pytest.mark.parametrize("Tq", [1024, 4096, 300])
@pytest.mark.parametrize("S_ip", [4, 16, 129])
def test_ip_attention_kernel(ctx, Tq, S_ip):
    """Two-source attention against two separate softmax attentions (f32, on the same f16 inputs)."""
    g = torch.Generator().manual_seed(Tq + S_ip)
    B, S, n_head = 2, 77, 5
    q, k, v = (torch.randn(B, n, 64 * n_head, generator=g).half() for n in (Tq, S, S))
    kip, vip = (torch.randn(B, S_ip, 64 * n_head, generator=g).half() for _ in range(2))
    out = ip_attention(ctx, q, k, v, kip, vip, n_head, 0.7).float().cpu()
    ref = IPO.ip_attention(q.float(), k.float(), v.float(), kip.float(), vip.float(), n_head, 0.7)
    sdpa = (torch.nn.functional.scaled_dot_product_attention(*(t.float().reshape(B, -1, n_head, 64).transpose(1, 2) for t in (q, k, v)))
            + 0.7 * torch.nn.functional.scaled_dot_product_attention(*(t.float().reshape(B, -1, n_head, 64).transpose(1, 2) for t in (q, kip, vip))))
    assert rel_err(ref, sdpa.transpose(1, 2).reshape(B, Tq, -1)) < 1e-5
    assert rel_err(out, ref) < ATTN_TOL
    # scale 0: exactly the one-source kernel
    zero = ip_attention(ctx, q, k, v, kip, vip, n_head, 0.0)
    assert torch.equal(zero, ctx.qkv_attention(q, k, v, None, n_head))


def test_project(S):
    e = embeds(3, 1, 5)[:, 0]
    out = S.ad.project(e).float().cpu()
    ref = IPO.project(S.waf, e).reshape(-1, TINY.context_dim)
    assert rel_err(out, ref) < FWD_TOL


@pytest.mark.parametrize("nb,ni", [(2, 1), (1, 2), (2, 3)])
def test_forward_against_oracle(S, nb, ni):
    e = embeds(nb, ni, 7)
    S.d.set_image_prompt(S.ad, e, 0.8)
    out = S.fwd()
    S.d.set_image_prompt(None)
    assert rel_err(out, S.ref(e, IPO.uniform_scales(TINY, 0.8))) < FWD_TOL


def test_detach_restores_bit_identical(S):
    base = S.fwd()
    n_ops = S.d.plan_num_ops
    n_builds = plan_builds(S.d)
    S.d.set_image_prompt(S.ad, embeds(2, 1, 1), 1.0)
    with_ip = S.fwd()
    assert not torch.equal(with_ip, base) and S.d.plan_num_ops == n_ops
    assert plan_builds(S.d) == n_builds + 1  # attaching drops the plan: rebuilt once
    S.d.set_image_prompt(None)
    assert torch.equal(S.fwd(), base) and S.d.plan_num_ops == n_ops
    assert plan_builds(S.d) == n_builds + 2  # and so does detaching


def test_scale_zero_equals_no_prompt(S):
    base = S.fwd()
    S.d.set_image_prompt(S.ad, embeds(2, 1, 2), 0.0)
    out = S.fwd()
    S.d.set_image_prompt(None)
    assert torch.equal(out, base)


def test_in_place_rescale_equals_fresh_attach(S):
    e1, e2 = embeds(2, 2, 3), embeds(2, 2, 4)
    S.d.set_image_prompt(S.ad, e1, 0.5)
    S.fwd()
    S.fwd()                                 # the second run captures the CUDA graph
    n_builds = plan_builds(S.d)
    S.d.set_image_prompt(S.ad, e2, 1.3)    # same adapter, n_batch, n_images: buffers rewritten in place
    rewritten = S.fwd()
    assert plan_builds(S.d) == n_builds     # the plan (and its graph) was kept
    S.d.set_image_prompt(None)
    S.d.set_image_prompt(S.ad, e2, 1.3)
    fresh = S.fwd()
    assert plan_builds(S.d) == n_builds + 1  # a new attachment drops the plan: rebuilt at this forward
    S.d.set_image_prompt(None)
    assert torch.equal(rewritten, fresh)


def test_per_block_scales(S):
    paths = transformer_block_paths(TINY)
    for k in (0, len(paths) // 2, len(paths) - 1):
        scales = [0.0] * len(paths)
        scales[k] = 1.5
        e = embeds(2, 1, 10 + k)
        S.d.set_image_prompt(S.ad, e, scales)
        out = S.fwd()
        S.d.set_image_prompt(None)
        ref = S.ref(e, {p: s for p, s in zip(paths, scales)})
        assert rel_err(out, ref) < FWD_TOL


@pytest.mark.parametrize("negative", [False, True])
def test_cfg_sample_against_oracle(S, negative):
    kw = tiny_conditioning()
    noise = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(0))
    e = embeds(1, 2, 20)
    neg = embeds(1, 2, 21) if negative else None
    S.d.set_image_prompt(S.ad, e, 0.9, negative=neg)
    try:
        out = S.d.sample_latent(Conditioning(**kw), 7.5, 4, noise=noise).cpu()
    finally:
        S.d.set_image_prompt(None)
    c = O.OracleConditioning(**kw)
    ref = O.sample_latent(TINY, S.wf, alphas_cumprod(TINY.n_steps), noise, c, 7.5, 4, att=IPO.attach(S.waf, e, neg, IPO.uniform_scales(TINY, 0.9)))
    assert rel_err(out, ref) < SAMPLE_TOL


def test_with_lora_and_controlnet(S):
    """LoRA apply / restore and a scale-0 ControlNet leave the image-prompted forward bit-identical; the ControlNet branch sees
    text only (its plan builds and runs beside the two-source attentions)."""
    e = embeds(2, 1, 30)
    S.d.set_image_prompt(S.ad, e, 1.0)
    ref = S.fwd()
    net = ControlNet(S.ctx, TINY_CONTROLNET, synth_weights(TINY_CONTROLNET, seed=1))
    S.d.set_controls([(net, torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(1)), 0.0)])
    assert torch.equal(S.fwd(), ref)
    S.d.set_controls([(net, torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(1)), 1.0)])
    assert not torch.equal(S.fwd(), ref)
    S.d.set_controls([])
    net.close()
    path = "input_blocks/4/transformer/transformer_0/attn2/query"   # C = 128
    g = torch.Generator().manual_seed(2)
    lora = {f"{path}/lora_down": (torch.randn(4, 128, generator=g) * 0.1).half(), f"{path}/lora_up": (torch.randn(128, 4, generator=g) * 0.1).half()}
    S.d.set_adapters([(lora, 1.0)])
    assert not torch.equal(S.fwd(), ref)
    S.d.set_adapters([])
    assert torch.equal(S.fwd(), ref)
    S.d.set_image_prompt(None)


def test_invalid_calls_leave_state(S, ctx):
    e = embeds(2, 1, 40)
    S.d.set_image_prompt(S.ad, e, 1.0)
    ref = S.fwd()
    with pytest.raises(SdxlError, match="n_batch"):
        S.d.set_image_prompt(S.ad, embeds(3, 1, 41), 1.0)       # 3 does not divide the batch of 2
    with pytest.raises(SdxlError, match="image embeddings"):
        S.d.set_image_prompt(S.ad, torch.randn(2, 1, D + 8), 1.0)   # wrong image_embed_dim
    with pytest.raises(SdxlError, match="not finite"):
        S.d.set_image_prompt(S.ad, e, float("nan"))
    other = IPAdapter(ctx, dataclasses.replace(TINY, adm_in_channels=16), D, synth_ip_adapter(TINY, D, seed=3))
    with pytest.raises(SdxlError, match="adm_in_channels"):
        S.d.set_image_prompt(other, e, 1.0)
    other.close()
    assert torch.equal(S.fwd(), ref)
    S.d.set_image_prompt(None)
    with pytest.raises(SdxlError, match="refiner"):
        IPAdapter(ctx, TINY_REFINER, D, synth_ip_adapter(TINY, D))
    r = Diffuser(ctx, TINY_REFINER, synth_weights(TINY_REFINER, seed=0))
    with pytest.raises(SdxlError, match="refiner"):
        r.set_image_prompt(S.ad, e, 1.0)
    r.close()
