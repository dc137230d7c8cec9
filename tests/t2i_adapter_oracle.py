"""f32 CPU oracle of T2I-Adapter conditioning (DESIGN.md §11), built from oracle/unet_oracle.py's block functions (and
tests/controlnet_oracle.py for a control): the adapter forward of diffusers' FullAdapterXL and UNet::forward / the DDIM sampler with
the features added in the UNet's encoder, as UNet2DConditionModel(down_intrablock_additional_residuals=...) does.

adapters: a list of (T2IAdapterConfig, f32 weights, hint [n_hint, C, H, W], scale); UNet row b uses feature set b % n_hint, the CFG
rows of image b both use set b % n_hint. The features are added when t >= t_min. With adapters=None every function computes exactly
what controlnet_oracle computes."""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import torch
import torch.nn.functional as F

from oracle import unet_oracle as O
import controlnet_oracle as CN


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
    """sum_a s_a * F_{a,k}, adapters in order (diffusers MultiAdapter with adapter_weights)."""
    total = None
    for acfg, w, hint, scale in adapters:
        f = [scale * t for t in adapter_features(acfg, w, hint)]
        total = f if total is None else [a + b for a, b in zip(total, f)]
    return total


def injection_blocks(cfg) -> List[str]:
    """Input blocks receiving F_0..F_2: a level's last resnet+transformer block, or for a transformer-free level its last block
    (its Downsample); F_3 follows the middle block."""
    ins, _, _ = O.unet_blocks(cfg)
    per_level, level = [[]], 0
    for kind, p, _, _ in ins[1:]:
        per_level[level].append((kind, p))
        if kind == "downsample":
            level += 1
            per_level.append([])
    out = []
    for blocks in per_level:
        tr = [p for kind, p in blocks if "transformer" in kind]
        out.append(tr[-1] if tr else blocks[-1][1])
    return out


def unet_forward(cfg, w, x, timesteps, context, label, adapters: Optional[Sequence] = None, t_min: int = 0,
                 controls: Optional[Sequence] = None):
    """controlnet_oracle.unet_forward with the adapters' features added in place to the outputs of the injection blocks and of the
    middle block (so the skips carry them), before the controls' residuals."""
    x_in = x
    emb = CN._emb(cfg, w, timesteps, label)
    ins, mid, outs = O.unet_blocks(cfg)
    feats = summed_features(adapters) if adapters and int(timesteps[0]) >= t_min else None
    points = injection_blocks(cfg)
    sel = torch.arange(x.shape[0]) % (adapters[0][2].shape[0] if adapters else 1)
    saved = []
    for kind, p, nh, d in ins:
        x = O._run_block(kind, p, nh, d, x, emb, context, w)
        if feats is not None and p in points:
            x = x + feats[points.index(p)][sel]
        saved.append(x)
    _, mp, nh, d = mid
    x = O.res_block(x, emb, w, f"{mp}/res1")
    x = O.spatial_transformer(x, context, w, f"{mp}/transformer", nh, d)
    x = O.res_block(x, emb, w, f"{mp}/res2")
    if feats is not None:
        x = x + feats[3][sel]
    for ncfg, wc, hint, scale in controls or []:
        res, r_mid = CN.controlnet_forward(ncfg, wc, x_in, timesteps, context, label, CN.hint_embedding(ncfg, wc, hint))
        saved = [s + scale * r for s, r in zip(saved, res)]
        x = x + scale * r_mid
    for kind, p, nh, d in outs:
        x = torch.cat([x, saved.pop()], dim=1)
        x = O._run_block(kind, p, nh, d, x, emb, context, w)
    x = O.group_norm(x, w["norm_out/weight"], w["norm_out/bias"])
    x = O.silu(x)
    return O.conv2d(x, w, "conv_out")


def diffuse_latent(cfg, w, alphas, latent, c, n_steps, guidance, adapters: Optional[Sequence] = None, t_min: int = 0):
    """unet_oracle.diffuse_latent from step 0 (CFG, base model) with adapters on both branches."""
    step_size = cfg.n_steps // n_steps
    n_batch = latent.shape[0]
    for t in range(cfg.n_steps - 1, -1, -step_size):
        current_alpha = O.get_alpha(alphas, t)
        prev_alpha = O.get_alpha(alphas, t - step_size) if t >= step_size else 1.0
        sqrt_noise = math.sqrt(1.0 - current_alpha)
        ts = torch.tensor([t], dtype=torch.int32)
        cond = unet_forward(cfg, w, latent, ts, c.context_full, c.channel_context, adapters, t_min)
        unc = unet_forward(cfg, w, latent, ts, c.unconditional_context_full.unsqueeze(0).repeat(n_batch, 1, 1),
                           c.unconditional_channel_context.unsqueeze(0).repeat(n_batch, 1), adapters, t_min)
        pred_noise = unc + (cond - unc) * guidance
        predx0 = (latent - pred_noise * sqrt_noise) / math.sqrt(current_alpha)
        latent = predx0 * math.sqrt(prev_alpha) + pred_noise * math.sqrt(1.0 - prev_alpha)
    return latent
