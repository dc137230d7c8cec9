"""SDXL base (synthetic weights) with a ViT-H-sized IP-Adapter Plus (synthetic weights: image features 257 x 1280, Resampler of
depth 4, 20 heads, 16 tokens) at 1024x1024: one CFG-batched forward with a Plus prompt against the f32 oracle, with the bound of the
1024^2 forward (test_fullsize_gpu, test_ip_adapter_fullsize_gpu)."""
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


def test_ip_adapter_plus_1024(ctx):
    w = sdxl_b200.synth_weights(SDXL_BASE, seed=0)
    wa = synth_ip_adapter(SDXL_BASE, 1280, seed=1, resampler=SDXL_PLUS)
    d = Diffuser(ctx, SDXL_BASE, w)
    ad = IPAdapter(ctx, SDXL_BASE, 1280, wa)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 128, 128, generator=g)
    c = torch.randn(2, 77, 2048, generator=g).half().float()
    y = torch.randn(2, 2816, generator=g).half().float()
    h = torch.randn(1, 1, 257, 1280, generator=g)
    d.set_image_prompt(ad, h, 1.0, negative=torch.zeros_like(h))   # n_batch = 1: both rows use the image
    got = d.unet_forward(x, [749], c, y)
    d.set_image_prompt(None)
    d.close()
    ad.close()
    waf = O.to_f32(wa)
    tok = PO.plus_prompt_tokens(waf, h).repeat(2, 1, 1)
    ref = O.unet_forward(SDXL_BASE, O.to_f32(w), x, torch.tensor([749]), c, y, O.Attach(prompts=[(waf, tok, IPO.uniform_scales(SDXL_BASE, 1.0), None)]))
    err = rel_err(got, ref)
    print(f"SDXL base + IP-Adapter Plus 1024^2 forward: rel err {err:.3e}")
    assert err < TOL
