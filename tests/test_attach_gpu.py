"""GPU tests of the UNet's shared attach protocol (csrc/engine.cu: attach_install, attach_detach, attachments_fit) across the five
kinds of attachment: a detach with nothing attached keeps the plan, and a sampler_begin on a latent an attachment does not fit is
refused before it touches the conditioning or the plan. The per-kind in-place rewrite and detach identities are in each kind's tests."""
import pytest
import torch

from sdxl_b200 import (TINY, TINY_CONTROLNET, TINY_INPAINT, TINY_T2I_ADAPTER, Conditioning, ControlNet, Diffuser, IPAdapter, SdxlError,
                       T2IAdapter, synth_weights)
from sdxl_b200.ip_adapter import synth_ip_adapter
from harness import arb, h16f, plan_builds

pytestmark = pytest.mark.gpu
T = 499
D = 32   # image_embed_dim of the tiny adapter


X = arb(2, 4, 16, 16)   # a 128 x 128 pixel latent
C_CTX = h16f(arb(2, 7, TINY.context_dim))
Y = h16f(arb(2, TINY.adm_in_channels))


def conditioning(res):
    return Conditioning(context_full=C_CTX, unconditional_context_full=C_CTX[0].cos(), channel_context=Y,
                        unconditional_channel_context=Y[0].cos(), resolution=res)


DETACHES = {
    "controls": lambda d: d.set_controls([]),
    "image_prompts": lambda d: d.set_image_prompts([]),
    "t2i_adapters": lambda d: d.set_t2i_adapters([]),
    "inpaint_condition": lambda d: d.set_inpaint_condition(None),
    "pag": lambda d: d.set_pag(None),
}


@pytest.mark.parametrize("kind", list(DETACHES))
def test_detach_of_nothing_keeps_the_plan(ctx, kind):
    d = Diffuser(ctx, TINY, synth_weights(TINY, seed=0))
    before = d.unet_forward(X, [T], C_CTX, Y).cpu()
    n = plan_builds(d)
    DETACHES[kind](d)
    after = d.unet_forward(X, [T]).cpu()
    assert plan_builds(d) == n
    assert torch.equal(after, before)
    d.close()


def _control(ctx, d):
    net = ControlNet(ctx, TINY_CONTROLNET, synth_weights(TINY_CONTROLNET, seed=1))
    d.set_controls([(net, torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(2)), 1.0)])
    return [net]


def _t2i(ctx, d):
    ad = T2IAdapter(ctx, TINY_T2I_ADAPTER, synth_weights(TINY_T2I_ADAPTER, seed=1))
    d.set_t2i_adapters([(ad, torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(2)), 1.0)])
    return [ad]


def _masked_prompt(ctx, d):
    ad = IPAdapter(ctx, TINY, D, synth_ip_adapter(TINY, D, seed=3))
    mask = torch.zeros(2, 128, 128)
    mask[0, :, :64], mask[1, :, 64:] = 1, 1
    d.set_image_prompts([(ad, torch.randn(1, 2, D, generator=torch.Generator().manual_seed(4)), 0.8, None, mask)])
    return [ad]


def _inpaint(ctx, d):
    g = torch.Generator().manual_seed(5)
    mask = (torch.rand(1, 1, 16, 16, generator=g) > 0.5).float()
    d.set_inpaint_condition(torch.cat([mask, torch.randn(1, 4, 16, 16, generator=g)], dim=1))
    return []


@pytest.mark.parametrize("cfg,attach", [(TINY, _control), (TINY, _t2i), (TINY, _masked_prompt), (TINY_INPAINT, _inpaint)],
                         ids=["control", "t2i", "masked_prompt", "inpaint"])
def test_sampler_begin_on_another_latent_is_refused_and_changes_nothing(ctx, cfg, attach):
    d = Diffuser(ctx, cfg, synth_weights(cfg, seed=0))
    models = attach(ctx, d)
    before = d.unet_forward(X, [T], C_CTX, Y).cpu()
    n = plan_builds(d)
    with pytest.raises(SdxlError, match="latent"):
        d.sampler_begin(conditioning((256, 256)), 7.5)
    after = d.unet_forward(X, [T]).cpu()   # the retained conditioning: the refusal must not have replaced it
    assert plan_builds(d) == n
    assert torch.equal(after, before)
    d.close()
    for m in models:
        m.close()
