"""The inpainting UNet's condition (DESIGN.md §12), which the f32 CPU oracle concatenates to the latent (oracle/unet_oracle.py,
Attach.concat): a restatement of its preparation (diffusers' StableDiffusionXLInpaintPipeline.prepare_mask_latents) without the
library.

cond: f32 [n, in_channels - out_channels, h, w], the mask (1 = repaint) then the masked image's latent; UNet row b reads row b % n,
the CFG rows of image b both read row b % n."""
from __future__ import annotations

from typing import Callable, Optional, Tuple

import torch


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
