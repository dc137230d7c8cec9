#!/usr/bin/env python
"""Generates tests/golden/prediction_1024.npz with the CPU f32 oracle: a v-prediction, zero-terminal-SNR sample at SDXL-base size.

    python tests/golden/make_prediction_golden.py [--threads N]

SDXL-base synthetic weights and the inputs of tests/fullsize_cases.py at 1024^2 (latent 128x128), through the chain
oracle/unet_oracle.py forward + tests/prediction_oracle.py (guidance rescale, the v prediction) + tests/scheduler_oracle.py steps:

    v_zsnr_dpmpp_2m_trailing_4   DPM++ 2M on the trailing spacing of the zero-SNR table, 4 steps, cfg 7.5, guidance rescale 0.7
                                 (8 UNet forwards)

tests/test_prediction_fullsize_gpu.py runs the same inputs through libsdxl_b200.so. A few minutes on 8 cores, no GPU.
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "stable-diffusion-xl-burn_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import fullsize_cases as FC  # noqa: E402
import prediction_oracle as PR  # noqa: E402
import scheduler_oracle as SO  # noqa: E402
import sdxl_b200  # noqa: E402  (config + synthetic weights only; the .so is never loaded here)
from oracle import unet_oracle as O  # noqa: E402

RES = 1024
N_STEPS = 4
GUIDANCE = 7.5
PHI = 0.7


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--threads", type=int, default=os.cpu_count())
    args = ap.parse_args()
    torch.set_num_threads(args.threads)
    cfg = sdxl_b200.SDXL_BASE
    w = O.to_f32(sdxl_b200.synth_weights(cfg, seed=FC.BASE_WEIGHT_SEED, device="cpu"))
    c = O.OracleConditioning(**FC.base_conditioning(RES))
    z0 = FC.base_noise(RES)
    with torch.no_grad():
        t0 = time.time()
        t, sig = SO.schedule("trailing", N_STEPS, PR.zero_snr_alphas(cfg.n_steps))
        x = PR.sample(PR.model_fn(cfg, w, c, GUIDANCE, PHI), "dpmpp_2m", t, sig, z0.double() * (sig[0] ** 2 + 1) ** 0.5)
        print(f"v_zsnr_dpmpp_2m_trailing_4: {time.time() - t0:.0f} s", flush=True)
    np.savez_compressed(os.path.join(HERE, "prediction_1024.npz"), v_zsnr_dpmpp_2m_trailing_4=x.float().numpy())


if __name__ == "__main__":
    main()
