"""SDXL base (synthetic weights) with a ViT-H-sized IP-Adapter (synthetic weights, D = 1024, 4 tokens) at 1024x1024: one
CFG-batched forward with an image prompt against the f32 oracle, with the bound of the 1024^2 forward (test_fullsize_gpu)."""
import pytest
import torch

import sdxl_b200
from sdxl_b200 import SDXL_BASE, Diffuser, IPAdapter
from sdxl_b200.ip_adapter import synth_ip_adapter
from oracle import unet_oracle as O
import ip_adapter_oracle as IPO

pytestmark = pytest.mark.gpu
TOL = 1e-3


def rel_err(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def test_ip_adapter_1024(ctx):
    w = sdxl_b200.synth_weights(SDXL_BASE, seed=0)
    wa = synth_ip_adapter(SDXL_BASE, 1024, seed=1)
    d = Diffuser(ctx, SDXL_BASE, w)
    ad = IPAdapter(ctx, SDXL_BASE, 1024, wa)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 128, 128, generator=g)
    c = torch.randn(2, 77, 2048, generator=g).half().float()
    y = torch.randn(2, 2816, generator=g).half().float()
    e = torch.randn(1, 1, 1024, generator=g)
    d.set_image_prompt(ad, e, 1.0)              # n_batch = 1: both rows use the image
    got = d.unet_forward(x, [749], c, y)
    d.set_image_prompt(None)
    d.close()
    ad.close()
    waf = O.to_f32(wa)
    tok = IPO.prompt_tokens(waf, e).repeat(2, 1, 1)
    ref = O.unet_forward(SDXL_BASE, O.to_f32(w), x, torch.tensor([749]), c, y, O.Attach(prompts=[(waf, tok, IPO.uniform_scales(SDXL_BASE, 1.0), None)]))
    err = rel_err(got, ref)
    print(f"SDXL base + IP-Adapter 1024^2 forward: rel err {err:.3e}")
    assert err < TOL
