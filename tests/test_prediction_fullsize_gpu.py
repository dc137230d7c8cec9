"""The v prediction with guidance rescale at SDXL-base size: libsdxl_b200.so at 1024^2 (latent 128x128) on the zero-terminal-SNR
table against the golden the CPU f32 oracle chain produced (tests/golden/make_prediction_golden.py, inputs in tests/fullsize_cases.py)."""
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
import make_prediction_golden as MG  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "prediction_1024.npz")
BOUND = 2e-3


def test_v_zero_snr_dpmpp_2m_trailing_4_steps_rescale(ctx):
    w = sdxl_b200.synth_weights(SDXL_BASE, seed=FC.BASE_WEIGHT_SEED, device="cpu")   # the generator the golden was made with
    d = Diffuser(ctx, SDXL_BASE, sdxl_b200.build_pack(w))
    del w
    d.set_prediction("v_prediction", MG.PHI, zero_terminal_snr=True)
    cond = Conditioning(**FC.base_conditioning(MG.RES))
    out = d.sample_latent(cond, MG.GUIDANCE, MG.N_STEPS, noise=FC.base_noise(MG.RES), schedule=Schedule("dpmpp_2m", "trailing", MG.N_STEPS))
    d.close()
    g = torch.as_tensor(np.load(GOLD)["v_zsnr_dpmpp_2m_trailing_4"]).double()
    e = float((out.double().cpu() - g).norm() / g.norm())
    print(f"SDXL base 1024^2, v, zero-SNR, DPM++ 2M trailing, 4 steps, cfg {MG.GUIDANCE}, rescale {MG.PHI}: rel err vs the oracle chain "
          f"{e:.3e} (bound {BOUND:.0e})")
    assert bool(torch.isfinite(out).all()) and e <= BOUND
