"""Helpers the tests share: the relative error they bound, the reference's probe input, f16 rounding, the tiny-config CFG
conditioning and the UNet's plan-build counter."""
import numpy as np
import torch

from sdxl_b200 import TINY, TINY_REFINER


def rel_err(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def arb(*dims):
    """arb_tensor(dims) = sin(arange(prod(dims))) — the reference's probe input (src/bin/test/main.rs:51-54)."""
    n = int(np.prod(dims))
    return torch.sin(torch.arange(n, dtype=torch.float32)).reshape(*dims)


def h16f(t):
    return t.to(torch.float16).float()


def tiny_conditioning(B=2, n_ctx=7, res=(128, 128), cfg=TINY, refiner=False):
    """Conditioning keyword arguments drawn from arb: cfg's context_full and channel_context with their unconditional rows, and with
    refiner=True also TINY_REFINER's context_open_clip and channel_context_refiner, so one conditioning serves the base and the
    refiner."""
    kw = dict(context_full=h16f(arb(B, n_ctx, cfg.context_dim) * 0.9), unconditional_context_full=h16f(arb(n_ctx, cfg.context_dim).cos()),
              channel_context=h16f(arb(B, cfg.adm_in_channels)), unconditional_channel_context=h16f(arb(cfg.adm_in_channels).cos()),
              resolution=res)
    if refiner:
        r = TINY_REFINER
        kw.update(context_open_clip=h16f(arb(B, n_ctx, r.context_dim) * 0.8),
                  unconditional_context_open_clip=h16f(arb(n_ctx, r.context_dim).cos()),
                  channel_context_refiner=h16f(arb(B, r.adm_in_channels) * 0.5),
                  unconditional_channel_context_refiner=h16f(arb(r.adm_in_channels).cos()))
    return kw


def plan_builds(d):
    """How many times the Diffuser d has built its UNet plan (sdxl_unet_plan_builds)."""
    return int(d.ctx.lib.sdxl_unet_plan_builds(d.h))
