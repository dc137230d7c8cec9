"""SDXL base (synthetic weights) at 1024x1024 with perturbed-attention guidance on the 10 mid-block self-attentions: one batched
forward of the three row groups [cond | uncond | ptb] against the f32 oracle, with the bound of the 1024^2 forward (test_fullsize_gpu)."""
import pytest
import torch

import sdxl_b200
from sdxl_b200 import SDXL_BASE, Diffuser, pag_layer_mask
from oracle import unet_oracle as O
import pag_oracle as PO

pytestmark = pytest.mark.gpu
TOL = 1e-3


def rel_err(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def test_pag_mid_1024(ctx):
    w = sdxl_b200.synth_weights(SDXL_BASE, seed=0)
    d = Diffuser(ctx, SDXL_BASE, w)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1, 4, 128, 128, generator=g).repeat(3, 1, 1, 1)     # the sampler broadcasts one latent to every row group
    c = torch.randn(2, 77, 2048, generator=g).half().float()
    y = torch.randn(2, 2816, generator=g).half().float()
    c, y = torch.cat([c, c[:1]]), torch.cat([y, y[:1]])                  # the perturbed row repeats the conditional one
    mask = pag_layer_mask(SDXL_BASE, "mid")
    d.set_pag("mid", 3.0)
    got = d.unet_forward(x, [749], c, y, perturbed_rows=1).cpu()
    d.set_pag(None)
    base = d.unet_forward(x, [749], c, y).cpu()
    d.close()
    ref = PO.forward_rows(SDXL_BASE, O.to_f32(w), x, torch.tensor([749]), c, y, PO.paths_of_mask(SDXL_BASE, mask), 1)
    err, moved = rel_err(got, ref), rel_err(got[2], base[2])
    print(f"SDXL PAG (mid) 1024^2: forward rel err {err:.3e}; PAG moves the perturbed row by {moved:.3e}; "
          f"attended rows bit-identical to the unperturbed forward: {torch.equal(got[:2], base[:2])}")
    assert err < TOL and moved > 1e-2
    assert torch.equal(got[:2], base[:2])
