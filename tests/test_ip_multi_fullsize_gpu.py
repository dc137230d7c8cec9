"""SDXL base (synthetic weights) with a ViT-H-sized base IP-Adapter and a ViT-H-sized IP-Adapter Plus (synthetic weights), masked to
the left and right halves of the image: one CFG-batched forward with the prompt set against the f32 oracle
(oracle/unet_oracle.py), with the bound of the 1024^2 forward (test_fullsize_gpu, test_ip_adapter_fullsize_gpu), at 1024 x 1024
and at 832 x 1216."""
import pytest
import torch

import sdxl_b200
from sdxl_b200 import SDXL_BASE, Diffuser, IPAdapter
from sdxl_b200.ip_adapter import SDXL_PLUS, synth_ip_adapter
from oracle import unet_oracle as O
import ip_adapter_oracle as IPO
import ip_adapter_plus_oracle as PO

pytestmark = pytest.mark.gpu
TOL = 1e-3


def rel_err(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.mark.parametrize("H,W", [(1024, 1024), (832, 1216)])
def test_base_and_plus_masked_halves(ctx, H, W):
    w = sdxl_b200.synth_weights(SDXL_BASE, seed=0)
    wa = synth_ip_adapter(SDXL_BASE, 1024, seed=1)
    wp = synth_ip_adapter(SDXL_BASE, 1280, seed=2, resampler=SDXL_PLUS)
    d = Diffuser(ctx, SDXL_BASE, w)
    ad = IPAdapter(ctx, SDXL_BASE, 1024, wa)
    plus = IPAdapter(ctx, SDXL_BASE, 1280, wp)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, H // 8, W // 8, generator=g)
    c = torch.randn(2, 77, 2048, generator=g).half().float()
    y = torch.randn(2, 2816, generator=g).half().float()
    e = torch.randn(1, 1, 1024, generator=g)
    h = torch.randn(1, 1, 257, 1280, generator=g)
    left = torch.zeros(1, H, W)
    left[:, :, :W // 2] = 1
    right = 1 - left
    d.set_image_prompts([(ad, e, 0.8, None, left), (plus, h, 0.7, torch.zeros_like(h), right)])   # n_batch = 1: both rows
    got = d.unet_forward(x, [749], c, y)
    d.set_image_prompts([])
    d.close()
    ad.close()
    plus.close()
    waf, wpf = O.to_f32(wa), O.to_f32(wp)
    prompts = [(waf, IPO.prompt_tokens(waf, e).repeat(2, 1, 1), IPO.uniform_scales(SDXL_BASE, 0.8), left),
               (wpf, PO.plus_prompt_tokens(wpf, h).repeat(2, 1, 1), IPO.uniform_scales(SDXL_BASE, 0.7), right)]
    ref = O.unet_forward(SDXL_BASE, O.to_f32(w), x, torch.tensor([749]), c, y, O.Attach(prompts=prompts))
    err = rel_err(got, ref)
    print(f"SDXL base + base and Plus adapters, masked halves, {H}x{W} forward: rel err {err:.3e}")
    assert err < TOL
