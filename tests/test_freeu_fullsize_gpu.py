"""SDXL base (synthetic weights) at 1024x1024 with FreeU at the SDXL values the FreeU authors recommend: one CFG-batched forward against
the f32 oracle (oracle/unet_oracle.py), with the bound of the 1024^2 forward (test_fullsize_gpu)."""
import pytest
import torch

import sdxl_b200
from sdxl_b200 import SDXL_BASE, Diffuser
from oracle import unet_oracle as O
import freeu_oracle as FO

pytestmark = pytest.mark.gpu
TOL = 1e-3


def rel_err(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def test_freeu_1024(ctx):
    w = sdxl_b200.synth_weights(SDXL_BASE, seed=0)
    d = Diffuser(ctx, SDXL_BASE, w)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1, 4, 128, 128, generator=g).repeat(2, 1, 1, 1)
    c = torch.randn(2, 77, 2048, generator=g).half().float()
    y = torch.randn(2, 2816, generator=g).half().float()
    d.set_freeu(*FO.RECOMMENDED_SDXL)
    got = d.unet_forward(x, [749], c, y).cpu()
    d.set_freeu(None)
    base = d.unet_forward(x, [749], c, y).cpu()
    d.close()
    ref = O.unet_forward(SDXL_BASE, O.to_f32(w), x, torch.tensor([749]), c, y, O.Attach(freeu=FO.RECOMMENDED_SDXL))
    err, moved = rel_err(got, ref), rel_err(got, base)
    print(f"SDXL FreeU 1024^2: forward rel err {err:.3e}; FreeU moves the forward by {moved:.3e}")
    assert err < TOL and moved > 1e-2
