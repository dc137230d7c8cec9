#!/usr/bin/env python
"""Generates tests/golden/samplers2_1024.npz with the CPU f32 oracle: two samplers of DESIGN.md §20 at SDXL-base size.

    python tests/golden/make_samplers2_golden.py [--threads N]

SDXL-base synthetic weights and the inputs of tests/fullsize_cases.py at 1024^2 (latent 128x128), through the chain
oracle/unet_oracle.py forward + tests/scheduler2_oracle.py sampler:

    unipc_karras_8          UniPC on a Karras schedule, 8 steps, cfg 7.5 (16 UNet forwards)
    dpmpp_2m_sde_karras_8   DPM++ 2M SDE on a Karras schedule, 8 steps, cfg 7.5, injected noise (seeds 500..506)

tests/test_samplers2_fullsize_gpu.py runs the same inputs through libsdxl_b200.so. A few minutes on 8 cores, no GPU.
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
import scheduler2_oracle as SO2  # noqa: E402
import scheduler_oracle as SO  # noqa: E402
import sdxl_b200  # noqa: E402  (config + synthetic weights only; the .so is never loaded here)
from oracle import unet_oracle as O  # noqa: E402

RES = 1024
SDE_NOISE_SEEDS = tuple(range(500, 507))


def sde_step_noise():
    return torch.stack([FC._randn(s, 1, 4, RES // 8, RES // 8) for s in SDE_NOISE_SEEDS])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--threads", type=int, default=os.cpu_count())
    args = ap.parse_args()
    torch.set_num_threads(args.threads)
    cfg = sdxl_b200.SDXL_BASE
    alphas = sdxl_b200.alphas_cumprod()
    a64 = np.array([O.get_alpha(alphas, i) for i in range(cfg.n_steps)])
    w = O.to_f32(sdxl_b200.synth_weights(cfg, seed=FC.BASE_WEIGHT_SEED, device="cpu"))
    c = O.OracleConditioning(**FC.base_conditioning(RES))
    z0 = FC.base_noise(RES)
    out = {}
    with torch.no_grad():
        t, sig = SO.schedule("karras", 8, a64)
        f = lambda x_in, tk: O.forward_diffuser(cfg, w, x_in.float(), torch.tensor([float(tk)]), c, 7.5)  # noqa: E731
        t0 = time.time()
        out["unipc_karras_8"] = SO2.sample2(f, "unipc", t, sig, z0 * (sig[0] ** 2 + 1) ** 0.5, where=torch.where).float().numpy()
        print(f"unipc_karras_8: {time.time() - t0:.0f} s", flush=True)
        t0 = time.time()
        it = iter(sde_step_noise())
        out["dpmpp_2m_sde_karras_8"] = SO2.sample2(f, "dpmpp_2m_sde", t, sig, z0 * (sig[0] ** 2 + 1) ** 0.5, lambda: next(it),
                                                  where=torch.where).float().numpy()
        print(f"dpmpp_2m_sde_karras_8: {time.time() - t0:.0f} s", flush=True)
    np.savez_compressed(os.path.join(HERE, "samplers2_1024.npz"), **out)


if __name__ == "__main__":
    main()
