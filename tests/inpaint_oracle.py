"""f32 CPU oracle of the inpainting UNet (DESIGN.md §12), on oracle/unet_oracle.py: UNet::forward of cat([x, cond[b % n]]) and the
DDIM / CFG chain with the condition attached, plus a restatement of the condition's preparation (diffusers'
StableDiffusionXLInpaintPipeline.prepare_mask_latents) without the library.

cond: f32 [n, in_channels - out_channels, h, w], the mask (1 = repaint) then the masked image's latent; UNet row b reads row b % n,
the CFG rows of image b both read row b % n."""
from __future__ import annotations

import math
from typing import Callable, Optional, Tuple

import torch

from oracle import unet_oracle as O


def unet_forward(cfg, w, x, timesteps, context, label, cond):
    """The 9-channel forward: the latent x [B, out_channels, h, w] and the attached condition, concatenated on channels."""
    sel = torch.arange(x.shape[0]) % cond.shape[0]
    return O.unet_forward(cfg, w, torch.cat([x, cond[sel]], dim=1), timesteps, context, label)


def diffuse_latent(cfg, w, alphas, latent, c, n_steps, guidance, cond):
    """unet_oracle.diffuse_latent from step 0 (CFG, base model, no blending) with the condition on both branches."""
    step_size = cfg.n_steps // n_steps
    n_batch = latent.shape[0]
    for t in range(cfg.n_steps - 1, -1, -step_size):
        current_alpha = O.get_alpha(alphas, t)
        prev_alpha = O.get_alpha(alphas, t - step_size) if t >= step_size else 1.0
        sqrt_noise = math.sqrt(1.0 - current_alpha)
        ts = torch.tensor([t], dtype=torch.int32)
        cnd = unet_forward(cfg, w, latent, ts, c.context_full, c.channel_context, cond)
        unc = unet_forward(cfg, w, latent, ts, c.unconditional_context_full.unsqueeze(0).repeat(n_batch, 1, 1),
                           c.unconditional_channel_context.unsqueeze(0).repeat(n_batch, 1), cond)
        pred_noise = unc + (cnd - unc) * guidance
        predx0 = (latent - pred_noise * sqrt_noise) / math.sqrt(current_alpha)
        latent = predx0 * math.sqrt(prev_alpha) + pred_noise * math.sqrt(1.0 - prev_alpha)
    return latent


def pixel_mask(img_h: int, img_w: int, left: Optional[int], right: Optional[int], top: Optional[int], bottom: Optional[int],
               crop_out: bool) -> torch.Tensor:
    """The crop window as a pixel mask bool [1, 1, H, W]: True inside [top, bottom) x [left, right) (missing bounds: the image's
    edges), inverted by crop_out. True = repaint."""
    l, r = left or 0, img_w if right is None else right
    t, b = top or 0, img_h if bottom is None else bottom
    m = torch.zeros(img_h, img_w, dtype=torch.bool)
    m[t:b, l:r] = True
    return (~m if crop_out else m).reshape(1, 1, img_h, img_w)


def prepare(rgb: torch.Tensor, mask: torch.Tensor, factor: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """(the latent-resolution mask f32 [n, 1, H/f, W/f] = mask[f i, f j], the masked image f32 [n, 3, H, W] in [-1, 1]) of rgb u8
    [n, H, W, 3] and mask bool [n, 1, H, W]."""
    image = rgb.permute(0, 3, 1, 2).double() / 255.0 * 2.0 - 1.0
    keep = ~mask
    masked = torch.where(keep, image, torch.zeros_like(image))
    return mask[:, :, ::factor, ::factor].float(), masked.float()


def condition(rgb: torch.Tensor, mask: torch.Tensor, encode: Callable[[torch.Tensor], torch.Tensor], factor: int) -> torch.Tensor:
    """The condition f32 [n, 1 + latent_channels, H/f, W/f]: the mask, then encode(masked image)."""
    m, masked = prepare(rgb, mask, factor)
    return torch.cat([m, encode(masked)], dim=1)
