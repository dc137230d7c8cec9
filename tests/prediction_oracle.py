"""Float64 statement of DESIGN.md §18 (sdxl_unet_set_prediction), written from its sources and importing nothing from the engine:
the zero-terminal-SNR noise table (Lin et al. 2023, "Common Diffusion Noise Schedules and Sample Steps are Flawed", Algorithm 1,
with diffusers' last entry 2^-24), guidance rescale (their Eq. 15-16, diffusers' rescale_noise_cfg), and the v prediction
(Salimans & Ho 2022) in the reference's DDIM loop and in the scheduled samplers of tests/scheduler_oracle.py. The UNet forward is
oracle/unet_oracle.py's; the chains take any model function, so tests can also drive them with analytic models."""
import dataclasses
import math

import numpy as np
import torch

from oracle import unet_oracle as O
import scheduler_oracle as SO


def zero_snr_sqrt_alphas(n=1000, beta_start=0.00085, beta_end=0.012):
    """sqrt(alpha_bar) of the scaled-linear betas after Algorithm 1's shift and scale (before any clamp): ends at 0, starts unchanged."""
    betas = np.linspace(beta_start ** 0.5, beta_end ** 0.5, n, dtype=np.float64) ** 2
    s = np.sqrt(np.cumprod(1.0 - betas))
    return (s - s[-1]) * (s[0] / (s[0] - s[-1]))


def zero_snr_alphas(n=1000, beta_start=0.00085, beta_end=0.012):
    """alphas_cumprod of the zero-terminal-SNR schedule, the last entry (0 before the clamp) set to 2^-24."""
    a = zero_snr_sqrt_alphas(n, beta_start, beta_end) ** 2
    a[-1] = 2.0 ** -24
    return a


def rescale_noise_cfg(g, c, phi):
    """g <- phi * g * std(c) / std(g) + (1 - phi) * g per image (dim 0), unbiased std over the other dims; the ratio is 1 where
    std(g) = 0."""
    dims = list(range(1, g.dim()))
    sc, sg = c.std(dim=dims, keepdim=True), g.std(dim=dims, keepdim=True)
    ratio = torch.where(sg > 0, sc / torch.where(sg > 0, sg, torch.ones_like(sg)), torch.ones_like(sg))
    return phi * g * ratio + (1.0 - phi) * g


def guided(cfg, w, latent, timestep, c, guidance, phi=0.0, att=None, no_cfg=False):
    """oracle/unet_oracle.py's forward_diffuser (PAG as its only attachment) with guidance rescale on the CFG rows: the guided model
    output g of the rows [cond | uncond | ptb]. no_cfg: the conditional rows alone (the refiner always), where phi has no effect."""
    att = att or O.NOTHING
    n = latent.shape[0]
    if cfg.is_refiner:
        uctx, ctx, uy, y = c.unconditional_context_open_clip, c.context_open_clip, c.unconditional_channel_context_refiner, c.channel_context_refiner
    else:
        uctx, ctx, uy, y = c.unconditional_context_full, c.context_full, c.unconditional_channel_context, c.channel_context
    plain = dataclasses.replace(att, pag_layers=())
    cond = O.unet_forward(cfg, w, latent, timestep, ctx, y, plain)
    out = cond
    if not (cfg.is_refiner or no_cfg):
        unc = O.unet_forward(cfg, w, latent, timestep, uctx.unsqueeze(0).repeat(n, 1, 1), uy.unsqueeze(0).repeat(n, 1), plain)
        out = unc + (cond - unc) * guidance
    if att.pag_layers:
        ptb = O.unet_forward(cfg, w, latent, timestep, ctx, y, att)
        out = out + att.pag_scale(float(timestep[0])) * (cond - ptb)
    if phi > 0 and not (cfg.is_refiner or no_cfg):
        out = rescale_noise_cfg(out, cond, phi)
    return out


def model_fn(cfg, w, c, guidance, phi=0.0, att=None, no_cfg=False):
    """g(x_in, t) of `guided` with the timestep as the engine passes it (an int for the DDIM loop, a float for the schedules)."""
    def f(x_in, t):
        ts = torch.tensor([float(t)], dtype=torch.float32)
        return guided(cfg, w, x_in.float(), ts, c, guidance, phi, att, no_cfg)
    return f


def ddim(g_fn, alphas, latent, n_steps, v=True, step_start=0, n_total=None):
    """The reference's DDIM loop (unet_oracle.diffuse_latent: timesteps, eta = 0) on the float64 table `alphas`, the model output
    g = g_fn(x, t) read as v (x0 = sqrt(a) x - sqrt(1 - a) g, eps = sqrt(a) g + sqrt(1 - a) x) or as eps."""
    total = len(alphas) if n_total is None else n_total
    step = total // n_steps
    for t in range(total - step_start - 1, -1, -step):
        a = float(alphas[t])
        ap = float(alphas[t - step]) if t >= step else 1.0
        g = g_fn(latent, t)
        if v:
            x0 = math.sqrt(a) * latent - math.sqrt(1.0 - a) * g
            eps = math.sqrt(a) * g + math.sqrt(1.0 - a) * latent
        else:
            eps = g
            x0 = (latent - math.sqrt(1.0 - a) * eps) / math.sqrt(a)
        latent = math.sqrt(ap) * x0 + math.sqrt(1.0 - ap) * eps
    return latent


def sample(g_fn, sampler, t, sig, x, draw=None, v=True, k0=0, k1=None, eta=1.0, s_noise=1.0, blend=None, where=torch.where):
    """scheduler_oracle.sample with the denoised D of a v model, D = x / (sigma^2 + 1) - sigma / sqrt(sigma^2 + 1) * g (v), or of an
    eps model, D = x - sigma * g; the sampler steps are scheduler_oracle.step."""
    D_prev = None
    for k in range(k0, len(t) if k1 is None else k1):
        s = float(sig[k])
        if blend is not None:
            x = where(blend[1], x, blend[0] + s * draw())
        g = g_fn(x / (s * s + 1.0) ** 0.5, t[k])
        D = x / (s * s + 1.0) - (s / (s * s + 1.0) ** 0.5) * g if v else x - s * g
        x = SO.step(sampler, k, t, sig, x, D, D_prev if sampler == "dpmpp_2m" else None, draw, eta, s_noise)
        D_prev = D
    return x
