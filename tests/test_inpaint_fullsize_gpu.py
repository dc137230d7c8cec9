"""The SDXL inpainting UNet (SDXL base with 9 input channels, synthetic weights) at 1024x1024: one CFG-batched forward with an attached
condition against the f32 oracle, with the bound of the 1024^2 forward (test_fullsize_gpu)."""
import pytest
import torch

import sdxl_b200
from sdxl_b200 import SDXL_INPAINT, Diffuser
from oracle import unet_oracle as O
from harness import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-3


def test_inpaint_unet_1024(ctx):
    w = sdxl_b200.synth_weights(SDXL_INPAINT, seed=0)
    d = Diffuser(ctx, SDXL_INPAINT, w)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 128, 128, generator=g)
    c = torch.randn(2, 77, 2048, generator=g).half().float()
    y = torch.randn(2, 2816, generator=g).half().float()
    mask = torch.zeros(1, 1, 128, 128)
    mask[:, :, 20:90, 33:101] = 1.0
    cond = torch.cat([mask, torch.randn(1, 4, 128, 128, generator=g) * (1 - mask)], dim=1)
    d.set_inpaint_condition(cond)   # n = 1: the [cond | uncond] rows both read it
    got = d.unet_forward(x, [749], c, y)
    d.set_inpaint_condition(None)
    d.close()
    ref = O.unet_forward(SDXL_INPAINT, O.to_f32(w), x, torch.tensor([749]), c, y, O.Attach(concat=cond))
    err = rel_err(got, ref)
    print(f"SDXL inpainting UNet 1024^2: CFG-batched forward rel err {err:.3e}")
    assert got.shape == (2, 4, 128, 128) and err < TOL
