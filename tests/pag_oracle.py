"""f32 CPU oracle of perturbed-attention guidance (DESIGN.md §14), built from oracle/unet_oracle.py's block functions (and
tests/ip_adapter_oracle.py / tests/controlnet_oracle.py for the attachments it composes with): UNet::forward with the listed
self-attentions (attn1 of a transformer block) computing out(value(x)) instead of softmax attention, and the CFG + PAG DDIM sampler of
diffusers' StableDiffusionXLPAGPipeline in this engine's combine form

    e = (u + (c - u) * guidance) + p_t * (c - ptb)      (refiner, without CFG: e = c + p_t * (c - ptb))
    p_t = max(scale - adaptive * (n_steps - t), 0)       (adaptive = 0: p_t = scale)

Layers are transformer block paths (self_attention_paths). Every UNet op is per batch row, so a batch whose last rows are perturbed is
the concatenation of a plain forward of the attended rows and a perturbed forward of the others (forward_rows). With no layers
unet_forward computes exactly what unet_oracle.unet_forward computes."""
from __future__ import annotations

import math
from typing import Collection, List, Optional, Sequence

import torch

from oracle import unet_oracle as O
import controlnet_oracle as CN
import ip_adapter_oracle as IA


def self_attention_paths(cfg) -> List[str]:
    """Pack paths of the transformer blocks, in execution order (input blocks, middle block, output blocks): one self-attention each."""
    ins, mid, outs = O.unet_blocks(cfg)
    paths = []
    for kind, p, _, d in ins + [mid] + outs:
        if "transformer" in kind or kind == "middle":
            paths += [f"{p}/transformer/transformer_{j}" for j in range(d)]
    return paths


def paths_of_mask(cfg, mask: Sequence[int]) -> List[str]:
    return [p for p, m in zip(self_attention_paths(cfg), mask) if m]


def _transformer_block(x, context, w, p, n_head, identity: bool, ip):
    h = O.layer_norm(x, w[f"{p}/norm1/weight"], w[f"{p}/norm1/bias"])
    if identity:
        x = x + O.linear(O.linear(h, w, f"{p}/attn1/value"), w, f"{p}/attn1/out")
    else:
        x = x + O.multi_head_attention(h, None, w, f"{p}/attn1", n_head)
    h = O.layer_norm(x, w[f"{p}/norm2/weight"], w[f"{p}/norm2/bias"])
    if ip is None:
        x = x + O.multi_head_attention(h, context, w, f"{p}/attn2", n_head)
    else:
        a = f"{p}/attn2"
        wa, tokens, scales = ip
        q, k, v = O.linear(h, w, f"{a}/query"), O.linear(context, w, f"{a}/key"), O.linear(context, w, f"{a}/value")
        att = IA.ip_attention(q, k, v, O.linear(tokens, wa, f"{a}/ip_key"), O.linear(tokens, wa, f"{a}/ip_value"), n_head, scales[p])
        x = x + O.linear(att, w, f"{a}/out")
    h = O.layer_norm(x, w[f"{p}/norm3/weight"], w[f"{p}/norm3/bias"])
    return x + O.linear(O.geglu(h, w, f"{p}/mlp/geglu"), w, f"{p}/mlp/lin")


def _spatial_transformer(x, context, w, p, n_head, depth, layers, ip):
    n_batch, n_channel, height, width = x.shape
    x_in = x
    x = O.group_norm(x, w[f"{p}/norm/weight"], w[f"{p}/norm/bias"])
    x = x.reshape(n_batch, n_channel, height * width).transpose(1, 2)
    x = O.linear(x, w, f"{p}/proj_in")
    for j in range(depth):
        bp = f"{p}/transformer_{j}"
        x = _transformer_block(x, context, w, bp, n_head, bp in layers, ip)
    x = O.linear(x, w, f"{p}/proj_out").transpose(1, 2).reshape(n_batch, n_channel, height, width)
    return x_in + x


def _run_block(kind, p, n_head, depth, x, emb, context, w, layers, ip):
    if "transformer" not in kind:
        return O._run_block(kind, p, n_head, depth, x, emb, context, w)
    x = O.res_block(x, emb, w, f"{p}/res")
    x = _spatial_transformer(x, context, w, f"{p}/transformer", n_head, depth, layers, ip)
    if kind.endswith("upsample"):
        x = O.upsample(x, w, f"{p}/upsample")
    return x


def unet_forward(cfg, w, x, timesteps, context, label, layers: Collection[str] = (), ip=None, controls: Optional[Sequence] = None):
    """UNet::forward with the self-attentions of `layers` as the identity on every row. ip: ip_adapter_oracle's forward form (weights,
    tokens [B, S_ip, ctx], scales); controls: controlnet_oracle's (ControlNetConfig, weights, hint, scale), whose nets run unperturbed."""
    x_in = x
    emb = CN._emb(cfg, w, timesteps, label)
    ins, mid, outs = O.unet_blocks(cfg)
    saved = []
    for kind, p, nh, d in ins:
        x = _run_block(kind, p, nh, d, x, emb, context, w, layers, ip)
        saved.append(x)
    _, mp, nh, d = mid
    x = O.res_block(x, emb, w, f"{mp}/res1")
    x = _spatial_transformer(x, context, w, f"{mp}/transformer", nh, d, layers, ip)
    x = O.res_block(x, emb, w, f"{mp}/res2")
    for ncfg, wc, hint, scale in controls or []:
        res, r_mid = CN.controlnet_forward(ncfg, wc, x_in, timesteps, context, label, CN.hint_embedding(ncfg, wc, hint))
        saved = [s + scale * r for s, r in zip(saved, res)]
        x = x + scale * r_mid
    for kind, p, nh, d in outs:
        x = torch.cat([x, saved.pop()], dim=1)
        x = _run_block(kind, p, nh, d, x, emb, context, w, layers, ip)
    x = O.group_norm(x, w["norm_out/weight"], w["norm_out/bias"])
    return O.conv2d(O.silu(x), w, "conv_out")


def forward_rows(cfg, w, x, timesteps, context, label, layers: Collection[str], n_ptb: int):
    """A batch whose last n_ptb rows are perturbed (the engine's direct forward with forward_perturbed_rows = n_ptb)."""
    a = len(x) - n_ptb
    return torch.cat([unet_forward(cfg, w, x[:a], timesteps, context[:a], label[:a]),
                      unet_forward(cfg, w, x[a:], timesteps, context[a:], label[a:], layers)])


def pag_scale(t: int, scale: float, adaptive: float, total: int) -> float:
    return max(scale - adaptive * (total - t), 0.0) if adaptive else scale


def guided_noise(cfg, w, latent, t, c, guidance, layers, scale, adaptive=0.0, ip=None, controls=None):
    """The guided noise of one step. ip: ip_adapter_oracle's sampler form (weights, embeds [n_batch, n_images, D], negative or None,
    scales): the conditional and the perturbed rows of image b use prompt b % n_batch, the unconditional rows the negative."""
    n = latent.shape[0]
    ts = torch.tensor([t], dtype=torch.int32)
    ipc = ipu = None
    if ip is not None:
        wa, embeds, negative, scales = ip
        sel = torch.arange(n) % embeds.shape[0]
        neg = torch.zeros_like(embeds) if negative is None else negative
        ipc = (wa, IA.prompt_tokens(wa, embeds)[sel], scales)
        ipu = (wa, IA.prompt_tokens(wa, neg)[sel], scales)
    if cfg.is_refiner:
        ctx, y = c.context_open_clip, c.channel_context_refiner
    else:
        ctx, y = c.context_full, c.channel_context
    cond = unet_forward(cfg, w, latent, ts, ctx, y, (), ipc, controls)
    ptb = unet_forward(cfg, w, latent, ts, ctx, y, layers, ipc, controls)
    p_t = pag_scale(t, scale, adaptive, cfg.n_steps)
    if cfg.is_refiner:
        return cond + p_t * (cond - ptb)
    unc = unet_forward(cfg, w, latent, ts, c.unconditional_context_full.unsqueeze(0).repeat(n, 1, 1),
                       c.unconditional_channel_context.unsqueeze(0).repeat(n, 1), (), ipu, controls)
    return (unc + (cond - unc) * guidance) + p_t * (cond - ptb)


def diffuse_latent(cfg, w, alphas, latent, c, step_start, n_steps, guidance, layers, scale, adaptive=0.0, ip=None, controls=None):
    """unet_oracle.diffuse_latent (DDIM, sigma = 0) with the PAG-guided noise."""
    step_size = cfg.n_steps // n_steps
    for t in range(cfg.n_steps - step_start - 1, -1, -step_size):
        current_alpha = O.get_alpha(alphas, t)
        prev_alpha = O.get_alpha(alphas, t - step_size) if t >= step_size else 1.0
        e = guided_noise(cfg, w, latent, t, c, guidance, layers, scale, adaptive, ip, controls)
        predx0 = (latent - e * math.sqrt(1.0 - current_alpha)) / math.sqrt(current_alpha)
        latent = predx0 * math.sqrt(prev_alpha) + e * math.sqrt(1.0 - prev_alpha)
    return latent


def refine_latent(cfg, w, alphas, latent, c, step_start, n_steps, noise, layers, scale, adaptive=0.0):
    """unet_oracle.refine_latent with PAG."""
    a0 = O.get_alpha(alphas, cfg.n_steps - step_start)
    noised = latent * math.sqrt(a0) + noise * math.sqrt(1.0 - a0)
    return diffuse_latent(cfg, w, alphas, noised, c, step_start, n_steps, 1.0, layers, scale, adaptive)
