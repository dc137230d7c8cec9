"""f32 CPU oracle of FreeU (DESIGN.md §15), built from oracle/unet_oracle.py's block functions and tests/pag_oracle.py's (which carry
the PAG identity self-attentions and image prompts) and tests/controlnet_oracle.py (ControlNet residuals): UNet::forward with diffusers'
apply_freeu before the skip concatenations of up_blocks[0] and up_blocks[1] (this engine's output_blocks/0..5), and the CFG sampler
and the refiner's refine with it.

`freeu` is diffusers' (s1, s2, b1, b2). The skip filter is diffusers' fourier_filter, restated literally with torch.fft; the closed
form the kernel computes (fourier_filter_closed) is restated here too, in float64, as the kernel tests' reference. With freeu None,
or any of its values 0 (diffusers' is_freeu_enabled), unet_forward computes what pag_oracle.unet_forward computes."""
from __future__ import annotations

import math
from typing import Collection, Optional, Sequence

import torch

from oracle import unet_oracle as O
import controlnet_oracle as CN
import pag_oracle as PO

RECOMMENDED_SDXL = (0.9, 0.2, 1.3, 1.4)   # the FreeU authors' values for SDXL (s1, s2, b1, b2)


def fourier_filter(x_in: torch.Tensor, threshold: int, scale: float) -> torch.Tensor:
    """diffusers.utils.torch_utils.fourier_filter on a real [B, C, H, W] tensor (its f16 / bf16 upcast does not apply here)."""
    x = x_in
    B, C, H, W = x.shape
    x_freq = torch.fft.fftn(x, dim=(-2, -1))
    x_freq = torch.fft.fftshift(x_freq, dim=(-2, -1))
    mask = torch.ones((B, C, H, W), dtype=x.dtype, device=x.device)
    crow, ccol = H // 2, W // 2
    mask[..., crow - threshold:crow + threshold, ccol - threshold:ccol + threshold] = scale
    x_freq = x_freq * mask
    x_freq = torch.fft.ifftshift(x_freq, dim=(-2, -1))
    x_filtered = torch.fft.ifftn(x_freq, dim=(-2, -1)).real
    return x_filtered.to(dtype=x_in.dtype)


def fourier_filter_closed(r: torch.Tensor, scale: float) -> torch.Tensor:
    """fourier_filter(r, 1, scale) in closed form: r + (scale - 1) / N * sum_{k in K} Re(X_k e^{i theta_k}), K = {0, -1 mod H} x
    {0, -1 mod W} as a set, X_k = sum r e^{-i theta_k}, theta_k(h, w) = 2 pi (k_h h / H + k_w w / W). In r's dtype (float64 for
    the kernels' reference)."""
    B, C, H, W = r.shape
    N = H * W
    hh = torch.arange(H, dtype=torch.float64)[:, None]
    ww = torch.arange(W, dtype=torch.float64)[None, :]
    out = r.double().clone()
    for kh in sorted({0, (H - 1) % H}):
        for kw in sorted({0, (W - 1) % W}):
            theta = 2 * math.pi * (kh * hh / H + kw * ww / W)
            X = (r.double() * torch.exp(-1j * theta)).sum(dim=(-2, -1))
            out += (scale - 1) / N * (X[..., None, None] * torch.exp(1j * theta)).real
    return out.to(r.dtype)


def enabled(freeu: Optional[Sequence[float]]) -> bool:
    """diffusers' is_freeu_enabled: all four values given and nonzero."""
    return freeu is not None and all(freeu)


def apply_freeu(k: int, x: torch.Tensor, res: torch.Tensor, freeu: Sequence[float]):
    """diffusers' apply_freeu at resolution_idx k (0, 1): x's first half of channels times b, the skip filtered with s."""
    s, b = freeu[k], freeu[2 + k]
    half = x.shape[1] // 2
    x = torch.cat([x[:, :half] * b, x[:, half:]], dim=1)
    return x, fourier_filter(res, 1, s)


def unet_forward(cfg, w, x, timesteps, context, label, freeu: Optional[Sequence[float]] = None, layers: Collection[str] = (), ip=None,
                 controls: Optional[Sequence] = None):
    """UNet::forward with FreeU at the skip concatenations of output blocks 0..5, after the ControlNet residuals were added to the
    skips. layers, ip, controls: pag_oracle.unet_forward's."""
    x_in = x
    emb = CN._emb(cfg, w, timesteps, label)
    ins, mid, outs = O.unet_blocks(cfg)
    saved = []
    for kind, p, nh, d in ins:
        x = PO._run_block(kind, p, nh, d, x, emb, context, w, layers, ip)
        saved.append(x)
    _, mp, nh, d = mid
    x = O.res_block(x, emb, w, f"{mp}/res1")
    x = PO._spatial_transformer(x, context, w, f"{mp}/transformer", nh, d, layers, ip)
    x = O.res_block(x, emb, w, f"{mp}/res2")
    for ncfg, wc, hint, scale in controls or []:
        res, r_mid = CN.controlnet_forward(ncfg, wc, x_in, timesteps, context, label, CN.hint_embedding(ncfg, wc, hint))
        saved = [s + scale * r for s, r in zip(saved, res)]
        x = x + scale * r_mid
    for i, (kind, p, nh, d) in enumerate(outs):
        skip = saved.pop()
        if enabled(freeu) and i // 3 < 2:   # up_blocks[0] and [1]: three output blocks each
            x, skip = apply_freeu(i // 3, x, skip, freeu)
        x = torch.cat([x, skip], dim=1)
        x = PO._run_block(kind, p, nh, d, x, emb, context, w, layers, ip)
    x = O.group_norm(x, w["norm_out/weight"], w["norm_out/bias"])
    return O.conv2d(O.silu(x), w, "conv_out")


def forward_diffuser(cfg, w, latent, timestep, c, guidance, freeu):
    """unet_oracle.forward_diffuser with FreeU on every row."""
    n = latent.shape[0]
    if cfg.is_refiner:
        return unet_forward(cfg, w, latent, timestep, c.context_open_clip, c.channel_context_refiner, freeu)
    cond = unet_forward(cfg, w, latent, timestep, c.context_full, c.channel_context, freeu)
    unc = unet_forward(cfg, w, latent, timestep, c.unconditional_context_full.unsqueeze(0).repeat(n, 1, 1),
                       c.unconditional_channel_context.unsqueeze(0).repeat(n, 1), freeu)
    return unc + (cond - unc) * guidance


def diffuse_latent(cfg, w, alphas, latent, c, step_start, n_steps, guidance, freeu):
    """unet_oracle.diffuse_latent (DDIM, sigma = 0) with FreeU."""
    step_size = cfg.n_steps // n_steps
    for t in range(cfg.n_steps - step_start - 1, -1, -step_size):
        current_alpha = O.get_alpha(alphas, t)
        prev_alpha = O.get_alpha(alphas, t - step_size) if t >= step_size else 1.0
        e = forward_diffuser(cfg, w, latent, torch.tensor([t], dtype=torch.int32), c, guidance, freeu)
        predx0 = (latent - e * math.sqrt(1.0 - current_alpha)) / math.sqrt(current_alpha)
        latent = predx0 * math.sqrt(prev_alpha) + e * math.sqrt(1.0 - prev_alpha)
    return latent


def refine_latent(cfg, w, alphas, latent, c, guidance, step_start, n_steps, noise, freeu):
    """unet_oracle.refine_latent with FreeU."""
    a0 = O.get_alpha(alphas, cfg.n_steps - step_start)
    noised = latent * math.sqrt(a0) + noise * math.sqrt(1.0 - a0)
    return diffuse_latent(cfg, w, alphas, noised, c, step_start, n_steps, guidance, freeu)
