"""Instruction-based editing at full size: an SDXL-base-shaped edit UNet (8 input channels, synthetic weights) through libsdxl_b200.so at
768^2 (diffusers/sdxl-instructpix2pix-768's size) and 1024^2, a 4-step DDIM sample with guidance and image guidance, against the golden
the CPU f32 oracle chain produced (tests/golden/make_edit_golden.py, inputs in tests/fullsize_cases.py)."""
import os
import sys

import numpy as np
import pytest
import torch

import sdxl_b200
from sdxl_b200 import SDXL_EDIT, Conditioning, Diffuser
import fullsize_cases as FC

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
import make_edit_golden as MG  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "edit_fullsize.npz")
BOUND = 2e-3


@pytest.fixture(scope="module")
def d(ctx):
    w = sdxl_b200.synth_weights(SDXL_EDIT, seed=FC.BASE_WEIGHT_SEED, device="cpu")   # the generator the golden was made with
    d = Diffuser(ctx, SDXL_EDIT, sdxl_b200.build_pack(w))
    del w
    yield d
    d.close()


@pytest.mark.parametrize("res", MG.SIZES)
def test_edit_ddim_4_steps(d, res):
    d.set_edit_image(MG.source_latent(res), MG.IMAGE_GUIDANCE)
    out = d.sample_latent(Conditioning(**FC.base_conditioning(res)), MG.GUIDANCE, MG.N_STEPS, noise=FC.base_noise(res)).cpu()
    d.set_edit_image(None)
    g = torch.as_tensor(np.load(GOLD)[f"ddim_4_{res}"]).double()
    e = float((out.double() - g).norm() / g.norm())
    print(f"SDXL edit UNet {res}^2, DDIM 4 steps, guidance {MG.GUIDANCE}, image guidance {MG.IMAGE_GUIDANCE}: rel err vs the oracle "
          f"chain {e:.3e} (bound {BOUND:.0e})")
    assert bool(torch.isfinite(out).all()) and e <= BOUND
