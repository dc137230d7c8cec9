#!/usr/bin/env python
"""Generates tests/golden/edit_fullsize.npz with the CPU f32 oracle: instruction-editing samples of an SDXL-base-shaped edit UNet.

    python tests/golden/make_edit_golden.py [--threads N]

Synthetic SDXL edit-UNet weights (sdxl_b200.SDXL_EDIT: 8 input channels) and tests/fullsize_cases.py's conditioning and noise, with
the source latent L ~ 0.5 N(0, 1) (seed 5), through oracle/unet_oracle.py's forward with L concatenated (tests/edit_oracle.py: rows
[cond | img | uncond], condition [L | L | 0]) and tests/prediction_oracle.py's DDIM loop on the f16-stored training table:

    ddim_4_<res>   the reference's DDIM loop, 4 steps, guidance 5.0, image guidance 1.5, at 768^2 (the checkpoint's size) and 1024^2
                   (12 UNet forwards each)

tests/test_edit_fullsize_gpu.py runs the same inputs through libsdxl_b200.so. About ten minutes on 8 cores, no GPU.
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

import edit_oracle as EO  # noqa: E402
import fullsize_cases as FC  # noqa: E402
import prediction_oracle as PR  # noqa: E402
import scheduler_oracle as SO  # noqa: E402
import sdxl_b200  # noqa: E402  (config + synthetic weights only; the .so is never loaded here)
from oracle import unet_oracle as O  # noqa: E402

SIZES = (768, 1024)
N_STEPS = 4
GUIDANCE = 5.0
IMAGE_GUIDANCE = 1.5


def source_latent(res: int) -> torch.Tensor:
    return 0.5 * torch.randn(1, 4, res // 8, res // 8, generator=torch.Generator().manual_seed(5))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--threads", type=int, default=os.cpu_count())
    args = ap.parse_args()
    torch.set_num_threads(args.threads)
    cfg = sdxl_b200.SDXL_EDIT
    w = O.to_f32(sdxl_b200.synth_weights(cfg, seed=FC.BASE_WEIGHT_SEED, device="cpu"))
    out = {}
    with torch.no_grad():
        for res in SIZES:
            t0 = time.time()
            c = O.OracleConditioning(**FC.base_conditioning(res))
            f = EO.model_fn(cfg, w, c, source_latent(res), GUIDANCE, IMAGE_GUIDANCE)
            x = PR.ddim(f, SO.sdxl_alphas(cfg.n_steps, f16=True), FC.base_noise(res).double(), N_STEPS, v=False)
            out[f"ddim_4_{res}"] = x.float().numpy()
            print(f"ddim_4_{res}: {time.time() - t0:.0f} s", flush=True)
    np.savez_compressed(os.path.join(HERE, "edit_fullsize.npz"), **out)


if __name__ == "__main__":
    main()
