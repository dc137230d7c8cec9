"""f32 CPU oracle of ControlNet conditioning (DESIGN.md §8), built from oracle/unet_oracle.py's block functions: the hint
encoder, the control branch (residuals per skip tensor and for the middle block) and UNet::forward / the DDIM sampler with the
residuals added to the skip connections, as diffusers' down_block_additional_residuals / mid_block_additional_residual do.

controls: a list of (ControlNetConfig, f32 weights, hint [n_hint, 3, H, W], scale); UNet row b uses hint b % n_hint, the CFG
rows of image b both use hint b % n_hint. With controls=None every function computes exactly what unet_oracle computes."""
from __future__ import annotations

import math
from typing import Optional, Sequence

import torch

from oracle import unet_oracle as O


def hint_embedding(ncfg, w, hint: torch.Tensor) -> torch.Tensor:
    """SGM input_hint_block: conv(in -> c0), then SiLU + conv after each conv, stride 2 on every second, last conv(c_last -> mc)."""
    x = O.conv2d(hint, w, "input_hint_block/0")
    idx = 2
    for _ in range(len(ncfg.hint_block_channels) - 1):
        x = O.conv2d(O.silu(x), w, f"input_hint_block/{idx}")
        x = O.conv2d(O.silu(x), w, f"input_hint_block/{idx + 2}", stride=2)
        idx += 4
    return O.conv2d(O.silu(x), w, f"input_hint_block/{idx}")


def _emb(cfg, w, timesteps, label):
    t_emb = O.linear(O.silu(O.linear(O.timestep_embedding(timesteps, cfg.model_channels, 10000), w, "lin1_time_embed")), w, "lin2_time_embed")
    label_emb = O.linear(O.silu(O.linear(label, w, "lin1_label_embed")), w, "lin2_label_embed")
    return t_emb + label_emb


def controlnet_forward(ncfg, w, x, timesteps, context, label, hint_emb):
    """The control branch: (residuals r_i = zero_conv_i(h_i) for every input block, r_mid = middle_block_out(mid))."""
    cfg = ncfg.unet
    emb = _emb(cfg, w, timesteps, label)
    ins, mid, _ = O.unet_blocks(cfg)
    sel = torch.arange(x.shape[0]) % hint_emb.shape[0]
    res = []
    h = x
    for i, (kind, p, nh, d) in enumerate(ins):
        h = O._run_block(kind, p, nh, d, h, emb, context, w)
        if i == 0:
            h = h + hint_emb[sel]
        res.append(O.conv2d(h, w, f"zero_convs/{i}", padding=0))
    _, mp, nh, d = mid
    h = O.res_block(h, emb, w, f"{mp}/res1")
    h = O.spatial_transformer(h, context, w, f"{mp}/transformer", nh, d)
    h = O.res_block(h, emb, w, f"{mp}/res2")
    return res, O.conv2d(h, w, "middle_block_out", padding=0)


def unet_forward(cfg, w, x, timesteps, context, label, controls: Optional[Sequence] = None):
    """UNet::forward (unet_oracle.unet_forward) with the controls' residuals added after the middle block, controls in order."""
    x_in = x
    emb = _emb(cfg, w, timesteps, label)
    ins, mid, outs = O.unet_blocks(cfg)
    saved = []
    for kind, p, nh, d in ins:
        x = O._run_block(kind, p, nh, d, x, emb, context, w)
        saved.append(x)
    _, mp, nh, d = mid
    x = O.res_block(x, emb, w, f"{mp}/res1")
    x = O.spatial_transformer(x, context, w, f"{mp}/transformer", nh, d)
    x = O.res_block(x, emb, w, f"{mp}/res2")
    for ncfg, wc, hint, scale in controls or []:
        res, r_mid = controlnet_forward(ncfg, wc, x_in, timesteps, context, label, hint_embedding(ncfg, wc, hint))
        saved = [s + scale * r for s, r in zip(saved, res)]
        x = x + scale * r_mid
    for kind, p, nh, d in outs:
        x = torch.cat([x, saved.pop()], dim=1)
        x = O._run_block(kind, p, nh, d, x, emb, context, w)
    x = O.group_norm(x, w["norm_out/weight"], w["norm_out/bias"])
    x = O.silu(x)
    return O.conv2d(x, w, "conv_out")


def forward_diffuser(cfg, w, latent, timestep, c, guidance, controls: Optional[Sequence] = None):
    """unet_oracle.forward_diffuser (base model, CFG) with controls on both branches."""
    n_batch = latent.shape[0]
    conditional = unet_forward(cfg, w, latent, timestep, c.context_full, c.channel_context, controls)
    unconditional = unet_forward(cfg, w, latent, timestep, c.unconditional_context_full.unsqueeze(0).repeat(n_batch, 1, 1),
                                 c.unconditional_channel_context.unsqueeze(0).repeat(n_batch, 1), controls)
    return unconditional + (conditional - unconditional) * guidance


def diffuse_latent(cfg, w, alphas, latent, c, n_steps, guidance, reference=None, mask=None, step_noise=None,
                   controls: Optional[Sequence] = None):
    """unet_oracle.diffuse_latent from step 0 (sample_latent / sample_latent_with_inpainting) with controls."""
    step_size = cfg.n_steps // n_steps
    it = 0
    for t in range(cfg.n_steps - 1, -1, -step_size):
        current_alpha = O.get_alpha(alphas, t)
        prev_alpha = O.get_alpha(alphas, t - step_size) if t >= step_size else 1.0
        sqrt_noise = math.sqrt(1.0 - current_alpha)
        if reference is not None:
            latent = torch.where(mask.bool(), latent, reference * math.sqrt(current_alpha) + step_noise[it] * sqrt_noise)
        pred_noise = forward_diffuser(cfg, w, latent, torch.tensor([t], dtype=torch.int32), c, guidance, controls)
        predx0 = (latent - pred_noise * sqrt_noise) / math.sqrt(current_alpha)
        latent = predx0 * math.sqrt(prev_alpha) + pred_noise * math.sqrt(1.0 - prev_alpha)
        it += 1
    return latent
