"""Inputs of the full-size parity cases (BASELINE.json configs 1, 2, 4, 5 as SURVEY.md 8(d) spells them out).

Shared by tests/golden/make_fullsize_golden.py (which runs the CPU f32 oracle once, offline, and commits the
final latents under tests/golden/) and by tests/test_fullsize_parity_gpu.py (which runs the same inputs through
libsdxl_b200.so on the GPU and compares). Everything is drawn from torch CPU generators, so both sides see
bit-identical weights and inputs on any machine. Weights: sdxl_b200.synth_weights(cfg, seed, device="cpu").
"""
from __future__ import annotations

import torch

BASE_WEIGHT_SEED = 0
REFINER_WEIGHT_SEED = 2
N_CTX = 77


def _randn(seed: int, *shape) -> torch.Tensor:
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def h16(t: torch.Tensor) -> torch.Tensor:
    """conditioning is f16 in the reference's Diffuser (sample/main.rs:236-241): round once, keep f32 for the oracle"""
    return t.to(torch.float16).float()


def base_conditioning(res: int) -> dict:
    """SURVEY 8(d) configs 1/2: ctx, uctx ~ N(0,1) seeds 1,2; y, uy seeds 3,4."""
    return dict(context_full=h16(_randn(1, 1, N_CTX, 2048)), unconditional_context_full=h16(_randn(2, N_CTX, 2048)),
                channel_context=h16(_randn(3, 1, 2816)), unconditional_channel_context=h16(_randn(4, 2816)),
                resolution=(res, res))


def base_noise(res: int) -> torch.Tensor:
    """x0 ~ N(0,1) seed 0, [1,4,res/8,res/8]."""
    return _randn(0, 1, 4, res // 8, res // 8)


# ---- single forward at 1024^2 (the tile shapes the 1024^2 plan builds: BN-256 pair tiles, T = 4096 attention) ----
FWD_1024_T = 999


def fwd_1024_inputs():
    return _randn(100, 1, 4, 128, 128), h16(_randn(101, 1, N_CTX, 2048)), h16(_randn(102, 1, 2816))


# ---- config 1: base 256^2, 4 Euler/DDIM steps (t = 999, 749, 499, 249), cfg 1.0 (and 7.5) ----
CONFIG1 = dict(res=256, n_steps=4, guidances=(1.0, 7.5))

# ---- config 2: base 1024^2, n = 30 -> 31 iterations, cfg 7.5 ----
CONFIG2 = dict(res=1024, n_steps=30, guidance=7.5, checkpoints=(1, 2, 4, 8, 16, 24, 31))

# ---- config 4 (refiner leg): refine_latent(step_start = 800, n = 50) -> 10 iterations at 1024^2, no CFG ----
REFINER = dict(res=1024, step_start=800, n_steps=50, guidance=7.5)


def refiner_inputs():
    ctx = h16(_randn(202, 1, N_CTX, 1280))
    y = h16(_randn(203, 1, 2560))
    cond = dict(context_open_clip=ctx, channel_context_refiner=y, unconditional_context_open_clip=ctx[0].clone(),
                unconditional_channel_context_refiner=y[0].clone(), resolution=(1024, 1024))
    return _randn(200, 1, 4, 128, 128), _randn(201, 1, 4, 128, 128), cond   # base latent, entry noise, conditioning


# ---- config 5 shape: inpainting at 1024^2, mask = latent rows 0..25 (200 px), 10 iterations (n = 10), cfg 7.5 ----
INPAINT = dict(res=1024, n_steps=10, guidance=7.5, mask_rows=25)


def inpaint_inputs():
    ref = _randn(5, 1, 4, 128, 128)
    mask = torch.zeros(1, 4, 128, 128, dtype=torch.bool)
    mask[:, :, :INPAINT["mask_rows"]] = True
    init = _randn(300, 1, 4, 128, 128)
    step_noise = torch.stack([_randn(301 + i, 1, 4, 128, 128) for i in range(INPAINT["n_steps"])])
    return ref, mask, init, step_noise


# ---- latent decoder / encoder at 1024^2 (SURVEY 8(f) rows 1 and 4): one decode and one encode vs the f32 oracle ----
VAE_WEIGHT_SEED = 7


def vae_1024_inputs(scale_factor: float):
    """(latent [1,4,128,128] scaled like a sampler output, u8 RGB image [1,1024,1024,3])"""
    lat = _randn(301, 1, 4, 128, 128) * scale_factor
    rgb = torch.randint(0, 256, (1, 1024, 1024, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(302))
    return lat, rgb


def vae_image_digest(img: torch.Tensor):
    """The 12 MB f32 image is committed as two 196 KB digests that together see every pixel: 8x8 block means
    (all pixels, averaged) and one raw pixel per block (no averaging)."""
    pool = torch.nn.functional.avg_pool2d(img.double(), 8).float()
    samp = img[:, :, 3::8, 5::8].contiguous()
    return pool, samp
