"""UniPC and DPM++ 2M SDE (DESIGN.md §20) at SDXL-base size: libsdxl_b200.so at 1024^2 (latent 128x128, the full-size eps pitch,
fractional timesteps) against the goldens the CPU f32 oracle chain produced (tests/golden/make_samplers2_golden.py, inputs in
tests/fullsize_cases.py)."""
import os
import sys

import numpy as np
import pytest
import torch

import sdxl_b200
from sdxl_b200 import SDXL_BASE, Conditioning, Diffuser
from sdxl_b200.schedulers import Schedule
import fullsize_cases as FC

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
import make_samplers2_golden as MG  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "samplers2_1024.npz")
BOUND = 2e-3


def golden_rel_err(a, b):
    a, b = a.detach().double().cpu(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


@pytest.fixture(scope="module")
def base(ctx):
    w = sdxl_b200.synth_weights(SDXL_BASE, seed=FC.BASE_WEIGHT_SEED, device="cpu")   # the generator the goldens were made with
    d = Diffuser(ctx, SDXL_BASE, sdxl_b200.build_pack(w))
    del w
    yield d
    d.close()


def test_unipc_karras_8_steps_cfg(base):
    g = np.load(GOLD)
    cond = Conditioning(**FC.base_conditioning(MG.RES))
    out = base.sample_latent(cond, 7.5, 8, noise=FC.base_noise(MG.RES), schedule=Schedule("unipc", "karras", 8))
    e = golden_rel_err(out, g["unipc_karras_8"])
    print(f"SDXL base 1024^2, UniPC Karras, 8 steps, cfg 7.5: rel err vs the oracle chain {e:.3e} (bound {BOUND:.0e})")
    assert bool(torch.isfinite(out).all()) and e <= BOUND


def test_dpmpp_2m_sde_karras_8_steps_cfg(base):
    g = np.load(GOLD)
    cond = Conditioning(**FC.base_conditioning(MG.RES))
    out = base.sample_latent(cond, 7.5, 8, noise=FC.base_noise(MG.RES), step_noise=MG.sde_step_noise(),
                             schedule=Schedule("dpmpp_2m_sde", "karras", 8))
    e = golden_rel_err(out, g["dpmpp_2m_sde_karras_8"])
    print(f"SDXL base 1024^2, DPM++ 2M SDE Karras, 8 steps, cfg 7.5, injected noise: rel err vs the oracle chain {e:.3e} "
          f"(bound {BOUND:.0e})")
    assert bool(torch.isfinite(out).all()) and e <= BOUND
