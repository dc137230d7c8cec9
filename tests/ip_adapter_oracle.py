"""f32 CPU oracle of IP-Adapter image prompts (DESIGN.md §9), built from oracle/unet_oracle.py's block functions: the image-token
projection, decoupled cross-attention in every attn2 and UNet::forward / the DDIM CFG sampler with an image prompt.

ip: (f32 adapter weights (pack names), tokens [B, S_ip, context_dim], scales {transformer block path: s}) for unet_forward; the
sampler takes (weights, embeds [n_batch, n_images, D], negative or None, scales) and applies the engine's row rule: the CFG rows
of image b use prompt b % n_batch (cond) and negative b % n_batch (uncond), zeros when negative is None. With ip=None every
function computes exactly what unet_oracle computes."""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from oracle import unet_oracle as O


def project(wa, embeds: torch.Tensor, tokens_per_image: int = 4) -> torch.Tensor:
    """ImageProjection: LayerNorm(e @ proj + b).reshape(n, T, ctx); embeds [n, D] -> [n, T, ctx]."""
    y = O.linear(embeds, wa, "image_proj/proj")
    y = y.reshape(embeds.shape[0], tokens_per_image, -1)
    return O.layer_norm(y, wa["image_proj/norm/weight"], wa["image_proj/norm/bias"])


def prompt_tokens(wa, embeds: torch.Tensor) -> torch.Tensor:
    """[n_batch, n_images, D] -> tokens [n_batch, n_images * T, ctx], images concatenated in order."""
    nb, ni, d = embeds.shape
    return project(wa, embeds.reshape(nb * ni, d)).reshape(nb, -1, wa["image_proj/norm/weight"].shape[0])


def ip_attention(q, k, v, k_ip, v_ip, n_head: int, scale: float) -> torch.Tensor:
    """softmax(q k^T) v + scale * softmax(q k_ip^T) v_ip: two separate softmaxes, summed before the out projection."""
    return O.qkv_attention(q, k, v, None, n_head) + scale * O.qkv_attention(q, k_ip, v_ip, None, n_head)


def _transformer_block(x, context, w, p, n_head, ip):
    x = x + O.multi_head_attention(O.layer_norm(x, w[f"{p}/norm1/weight"], w[f"{p}/norm1/bias"]), None, w, f"{p}/attn1", n_head)
    h = O.layer_norm(x, w[f"{p}/norm2/weight"], w[f"{p}/norm2/bias"])
    a = f"{p}/attn2"
    q, k, v = O.linear(h, w, f"{a}/query"), O.linear(context, w, f"{a}/key"), O.linear(context, w, f"{a}/value")
    if ip is None:
        att = O.qkv_attention(q, k, v, None, n_head)
    else:
        wa, tokens, scales = ip
        att = ip_attention(q, k, v, O.linear(tokens, wa, f"{a}/ip_key"), O.linear(tokens, wa, f"{a}/ip_value"), n_head, scales[p])
    x = x + O.linear(att, w, f"{a}/out")
    h = O.layer_norm(x, w[f"{p}/norm3/weight"], w[f"{p}/norm3/bias"])
    return x + O.linear(O.geglu(h, w, f"{p}/mlp/geglu"), w, f"{p}/mlp/lin")


def _spatial_transformer(x, context, w, p, n_head, depth, ip):
    n_batch, n_channel, height, width = x.shape
    x_in = x
    x = O.group_norm(x, w[f"{p}/norm/weight"], w[f"{p}/norm/bias"])
    x = x.reshape(n_batch, n_channel, height * width).transpose(1, 2)
    x = O.linear(x, w, f"{p}/proj_in")
    for j in range(depth):
        x = _transformer_block(x, context, w, f"{p}/transformer_{j}", n_head, ip)
    x = O.linear(x, w, f"{p}/proj_out").transpose(1, 2).reshape(n_batch, n_channel, height, width)
    return x_in + x


def _run_block(kind, p, n_head, depth, x, emb, context, w, ip):
    if "transformer" not in kind:
        return O._run_block(kind, p, n_head, depth, x, emb, context, w)
    x = O.res_block(x, emb, w, f"{p}/res")
    x = _spatial_transformer(x, context, w, f"{p}/transformer", n_head, depth, ip)
    if kind.endswith("upsample"):
        x = O.upsample(x, w, f"{p}/upsample")
    return x


def unet_forward(cfg, w, x, timesteps, context, label, ip=None):
    """UNet::forward (unet_oracle.unet_forward) with decoupled cross-attention in every transformer block."""
    t_emb = O.linear(O.silu(O.linear(O.timestep_embedding(timesteps, cfg.model_channels, 10000), w, "lin1_time_embed")), w, "lin2_time_embed")
    emb = t_emb + O.linear(O.silu(O.linear(label, w, "lin1_label_embed")), w, "lin2_label_embed")
    ins, mid, outs = O.unet_blocks(cfg)
    saved = []
    for kind, p, nh, d in ins:
        x = _run_block(kind, p, nh, d, x, emb, context, w, ip)
        saved.append(x)
    _, mp, nh, d = mid
    x = O.res_block(x, emb, w, f"{mp}/res1")
    x = _spatial_transformer(x, context, w, f"{mp}/transformer", nh, d, ip)
    x = O.res_block(x, emb, w, f"{mp}/res2")
    for kind, p, nh, d in outs:
        x = torch.cat([x, saved.pop()], dim=1)
        x = _run_block(kind, p, nh, d, x, emb, context, w, ip)
    x = O.group_norm(x, w["norm_out/weight"], w["norm_out/bias"])
    return O.conv2d(O.silu(x), w, "conv_out")


def forward_diffuser(cfg, w, latent, timestep, c, guidance, ip=None):
    """unet_oracle.forward_diffuser (base model, CFG) with an image prompt (sampler form of `ip`, see the module doc)."""
    n_batch = latent.shape[0]
    ipc = ipu = None
    if ip is not None:
        wa, embeds, negative, scales = ip
        sel = torch.arange(n_batch) % embeds.shape[0]
        neg = torch.zeros_like(embeds) if negative is None else negative
        ipc = (wa, prompt_tokens(wa, embeds)[sel], scales)
        ipu = (wa, prompt_tokens(wa, neg)[sel], scales)
    conditional = unet_forward(cfg, w, latent, timestep, c.context_full, c.channel_context, ipc)
    unconditional = unet_forward(cfg, w, latent, timestep, c.unconditional_context_full.unsqueeze(0).repeat(n_batch, 1, 1),
                                 c.unconditional_channel_context.unsqueeze(0).repeat(n_batch, 1), ipu)
    return unconditional + (conditional - unconditional) * guidance


def sample_latent(cfg, w, alphas, latent, c, n_steps, guidance, ip=None):
    """unet_oracle.sample_latent (DDIM from step 0) with an image prompt."""
    step_size = cfg.n_steps // n_steps
    for t in range(cfg.n_steps - 1, -1, -step_size):
        current_alpha = O.get_alpha(alphas, t)
        prev_alpha = O.get_alpha(alphas, t - step_size) if t >= step_size else 1.0
        pred_noise = forward_diffuser(cfg, w, latent, torch.tensor([t], dtype=torch.int32), c, guidance, ip)
        predx0 = (latent - pred_noise * math.sqrt(1.0 - current_alpha)) / math.sqrt(current_alpha)
        latent = predx0 * math.sqrt(prev_alpha) + pred_noise * math.sqrt(1.0 - prev_alpha)
    return latent


def uniform_scales(cfg, s: float) -> Dict[str, float]:
    """s for every transformer block of cfg."""
    from sdxl_b200.ip_adapter import transformer_block_paths
    return {p: s for p in transformer_block_paths(cfg)}
