"""SDXL base (synthetic weights) with an SDXL ControlNet (synthetic weights, non-zero zero convs) at 1024x1024: the hint encoder
and one CFG-batched forward against the f32 oracle, with the bound of the uncontrolled 1024^2 forward (test_fullsize_gpu)."""
import pytest
import torch

import sdxl_b200
from sdxl_b200 import SDXL_BASE, SDXL_CONTROLNET, ControlNet, Diffuser
from oracle import unet_oracle as O

pytestmark = pytest.mark.gpu
TOL = 1e-3


def rel_err(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def test_controlnet_1024(ctx):
    w = sdxl_b200.synth_weights(SDXL_BASE, seed=0)
    wc = sdxl_b200.synth_weights(SDXL_CONTROLNET, seed=1)
    d = Diffuser(ctx, SDXL_BASE, w)
    net = ControlNet(ctx, SDXL_CONTROLNET, wc)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 128, 128, generator=g)
    c = torch.randn(2, 77, 2048, generator=g).half().float()
    y = torch.randn(2, 2816, generator=g).half().float()
    hint = torch.rand(1, 3, 1024, 1024, generator=g)
    wcf = O.to_f32(wc)
    emb = net.embed_hint(hint)
    emb_ref = O.hint_embedding(SDXL_CONTROLNET, wcf, hint)
    e_hint = rel_err(emb, emb_ref)
    d.set_controls([(net, hint, 1.0)])          # n_hint = 1: both CFG rows use the image's hint
    got = d.unet_forward(x, [749], c, y)
    d.set_controls([])
    base = d.unet_forward(x, [749], c, y)
    d.close()
    net.close()
    ref = O.unet_forward(SDXL_BASE, O.to_f32(w), x, torch.tensor([749]), c, y, O.Attach(controls=[(SDXL_CONTROLNET, wcf, hint, 1.0)]))
    e = rel_err(got, ref)
    print(f"SDXL ControlNet 1024^2: hint_emb rel err {e_hint:.2e}, CFG-batched forward rel err {e:.2e}, "
          f"the control moves the forward by {rel_err(got, base):.2e}")
    assert e_hint <= TOL and e <= TOL and rel_err(got, base) > 0.05
