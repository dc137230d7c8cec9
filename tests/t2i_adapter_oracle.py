"""T2I-Adapter conditioning (DESIGN.md §11) for the f32 CPU oracle, which adds the features in the UNet's encoder as
UNet2DConditionModel(down_intrablock_additional_residuals=...) does (oracle/unet_oracle.py): the adapter forward of diffusers'
FullAdapterXL and the features of several adapters summed.

adapters: a list of (T2IAdapterConfig, f32 weights, hint [n_hint, C, H, W], scale); UNet row b uses feature set b % n_hint."""
from __future__ import annotations

from typing import List, Sequence

import torch
import torch.nn.functional as F

from oracle import unet_oracle as O


def pixel_unshuffle(x: torch.Tensor, r: int) -> torch.Tensor:
    """[n, C, H, W] -> [n, C*r*r, H/r, W/r]; channel c*r*r + i*r + j of pixel (y, x) is x[c, r*y + i, r*x + j]."""
    n, c, h, w = x.shape
    return x.reshape(n, c, h // r, r, w // r, r).permute(0, 1, 3, 5, 2, 4).reshape(n, c * r * r, h // r, w // r)


def adapter_features(acfg, w, hint: torch.Tensor) -> List[torch.Tensor]:
    """FullAdapterXL.forward: conv_in(pixel_unshuffle(hint, 16)), then per level k an average pool (k = 2), a 1x1 in_conv (k = 1, 2)
    and n_res_blocks resnets x + block2(relu(block1(x))); F_k is the level's output."""
    x = O.conv2d(pixel_unshuffle(hint, 16), w, "conv_in")
    feats = []
    for k in range(4):
        if k == 2:
            x = F.avg_pool2d(x, 2, ceil_mode=True)
        if k in (1, 2):
            x = O.conv2d(x, w, f"body/{k}/in_conv", padding=0)
        for j in range(acfg.n_res_blocks):
            p = f"body/{k}/resnets/{j}"
            x = x + O.conv2d(torch.relu(O.conv2d(x, w, f"{p}/block1")), w, f"{p}/block2", padding=0)
        feats.append(x)
    return feats


def summed_features(adapters: Sequence) -> List[torch.Tensor]:
    """sum_a s_a * F_{a,k}, adapters in order (diffusers MultiAdapter with adapter_weights): the features of Attach.t2i."""
    total = None
    for acfg, w, hint, scale in adapters:
        f = [scale * t for t in adapter_features(acfg, w, hint)]
        total = f if total is None else [a + b for a, b in zip(total, f)]
    return total
