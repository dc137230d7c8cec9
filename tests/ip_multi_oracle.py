"""f32 CPU oracle of image-prompt sets (DESIGN.md §13), beside tests/ip_adapter_oracle.py and ip_adapter_plus_oracle.py, whose token
functions it reuses: several prompts in every attn2, each unmasked (one softmax over all its tokens) or masked (one softmax per image,
weighted per query by the image's mask downsampled as diffusers' IPAdapterMaskProcessor.downsample does).

A prompt for unet_forward is (f32 adapter weights (pack names), tokens [B, S_ip, context_dim], scales {transformer block path: s},
mask [n_images, H, W] or None). The sampler form is (weights, cond tokens [n_batch, S_ip, ctx], uncond tokens, scales, mask) and
applies the engine's row rule: the CFG rows of image b use prompt row b % n_batch."""
from __future__ import annotations

import math
from typing import Optional, Sequence

import torch
import torch.nn.functional as F

from oracle import unet_oracle as O


def mask_grid(H: int, W: int, T: int):
    """(mh, mw) of diffusers' downsample for T queries and an H x W mask, both kept >= 1 (diffusers divides by zero there)."""
    ratio = W / H
    mh = max(1, int(math.sqrt(T / ratio)))
    mh += int(T % mh != 0)
    return mh, max(1, T // mh)


def downsample_mask(mask: torch.Tensor, T: int) -> torch.Tensor:
    """[n, H, W] -> [n, T]: bicubic to mask_grid, flattened row-major, zero-padded or cut to T."""
    n, H, W = mask.shape
    mh, mw = mask_grid(H, W, T)
    m = F.interpolate(mask[:, None].float(), size=(mh, mw), mode="bicubic", align_corners=False)[:, 0].reshape(n, -1)
    if m.shape[1] < T:
        return torch.cat([m, m.new_zeros(n, T - m.shape[1])], 1)
    return m[:, :T]


def sdpa(q, k, v, n_head: int) -> torch.Tensor:
    """Multi-head F.scaled_dot_product_attention on [B, T, C] / [B, S, C] (head dim C / n_head)."""
    B, T, C = q.shape
    split = lambda t: t.reshape(B, t.shape[1], n_head, C // n_head).transpose(1, 2)  # noqa: E731
    return F.scaled_dot_product_attention(split(q), split(k), split(v)).transpose(1, 2).reshape(B, T, C)


def multi_attention(q, k, v, sources: Sequence, n_head: int) -> torch.Tensor:
    """softmax(q k^T) v + sum over sources (k_s, v_s, s, m) of s * m[t] * softmax(q k_s^T) v_s (m None: 1), in order."""
    h = sdpa(q, k, v, n_head)
    for k_s, v_s, s, m in sources:
        a = s * sdpa(q, k_s, v_s, n_head)
        h = h + (a if m is None else a * m[None, :, None])
    return h


def _sources(h, prompts, a: str, p: str):
    T = h.shape[1]
    out = []
    for wa, tokens, scales, mask in prompts:
        k, v = O.linear(tokens, wa, f"{a}/ip_key"), O.linear(tokens, wa, f"{a}/ip_value")
        if mask is None:
            out.append((k, v, scales[p], None))
            continue
        n = mask.shape[0]
        m = downsample_mask(mask, T)
        per = k.shape[1] // n
        out += [(k[:, i * per:(i + 1) * per], v[:, i * per:(i + 1) * per], scales[p], m[i]) for i in range(n)]
    return out


def _transformer_block(x, context, w, p, n_head, prompts):
    x = x + O.multi_head_attention(O.layer_norm(x, w[f"{p}/norm1/weight"], w[f"{p}/norm1/bias"]), None, w, f"{p}/attn1", n_head)
    h = O.layer_norm(x, w[f"{p}/norm2/weight"], w[f"{p}/norm2/bias"])
    a = f"{p}/attn2"
    q, k, v = O.linear(h, w, f"{a}/query"), O.linear(context, w, f"{a}/key"), O.linear(context, w, f"{a}/value")
    att = multi_attention(q, k, v, _sources(q, prompts, a, p), n_head)
    x = x + O.linear(att, w, f"{a}/out")
    h = O.layer_norm(x, w[f"{p}/norm3/weight"], w[f"{p}/norm3/bias"])
    return x + O.linear(O.geglu(h, w, f"{p}/mlp/geglu"), w, f"{p}/mlp/lin")


def _spatial_transformer(x, context, w, p, n_head, depth, prompts):
    n_batch, n_channel, height, width = x.shape
    x_in = x
    x = O.group_norm(x, w[f"{p}/norm/weight"], w[f"{p}/norm/bias"])
    x = x.reshape(n_batch, n_channel, height * width).transpose(1, 2)
    x = O.linear(x, w, f"{p}/proj_in")
    for j in range(depth):
        x = _transformer_block(x, context, w, f"{p}/transformer_{j}", n_head, prompts)
    x = O.linear(x, w, f"{p}/proj_out").transpose(1, 2).reshape(n_batch, n_channel, height, width)
    return x_in + x


def _run_block(kind, p, n_head, depth, x, emb, context, w, prompts):
    if "transformer" not in kind:
        return O._run_block(kind, p, n_head, depth, x, emb, context, w)
    x = O.res_block(x, emb, w, f"{p}/res")
    x = _spatial_transformer(x, context, w, f"{p}/transformer", n_head, depth, prompts)
    if kind.endswith("upsample"):
        x = O.upsample(x, w, f"{p}/upsample")
    return x


def unet_forward(cfg, w, x, timesteps, context, label, prompts: Sequence = ()):
    """UNet::forward (unet_oracle.unet_forward) with every prompt of the set in each transformer block."""
    t_emb = O.linear(O.silu(O.linear(O.timestep_embedding(timesteps, cfg.model_channels, 10000), w, "lin1_time_embed")), w, "lin2_time_embed")
    emb = t_emb + O.linear(O.silu(O.linear(label, w, "lin1_label_embed")), w, "lin2_label_embed")
    ins, mid, outs = O.unet_blocks(cfg)
    saved = []
    for kind, p, nh, d in ins:
        x = _run_block(kind, p, nh, d, x, emb, context, w, prompts)
        saved.append(x)
    _, mp, nh, d = mid
    x = O.res_block(x, emb, w, f"{mp}/res1")
    x = _spatial_transformer(x, context, w, f"{mp}/transformer", nh, d, prompts)
    x = O.res_block(x, emb, w, f"{mp}/res2")
    for kind, p, nh, d in outs:
        x = torch.cat([x, saved.pop()], dim=1)
        x = _run_block(kind, p, nh, d, x, emb, context, w, prompts)
    x = O.group_norm(x, w["norm_out/weight"], w["norm_out/bias"])
    return O.conv2d(O.silu(x), w, "conv_out")


def forward_diffuser(cfg, w, latent, timestep, c, guidance, prompts: Sequence):
    """unet_oracle.forward_diffuser (base model, CFG) with a prompt set in sampler form (module doc)."""
    n_batch = latent.shape[0]
    sel = lambda t: t[torch.arange(n_batch) % t.shape[0]]  # noqa: E731
    pc = [(wa, sel(tc), s, m) for wa, tc, tu, s, m in prompts]
    pu = [(wa, sel(tu), s, m) for wa, tc, tu, s, m in prompts]
    conditional = unet_forward(cfg, w, latent, timestep, c.context_full, c.channel_context, pc)
    unconditional = unet_forward(cfg, w, latent, timestep, c.unconditional_context_full.unsqueeze(0).repeat(n_batch, 1, 1),
                                 c.unconditional_channel_context.unsqueeze(0).repeat(n_batch, 1), pu)
    return unconditional + (conditional - unconditional) * guidance


def sample_latent(cfg, w, alphas, latent, c, n_steps, guidance, prompts: Sequence):
    """unet_oracle.sample_latent (DDIM from step 0) with a prompt set."""
    step_size = cfg.n_steps // n_steps
    for t in range(cfg.n_steps - 1, -1, -step_size):
        current_alpha = O.get_alpha(alphas, t)
        prev_alpha = O.get_alpha(alphas, t - step_size) if t >= step_size else 1.0
        pred_noise = forward_diffuser(cfg, w, latent, torch.tensor([t], dtype=torch.int32), c, guidance, prompts)
        predx0 = (latent - pred_noise * math.sqrt(1.0 - current_alpha)) / math.sqrt(current_alpha)
        latent = predx0 * math.sqrt(prev_alpha) + pred_noise * math.sqrt(1.0 - prev_alpha)
    return latent


def binarize(mask: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """diffusers' mask processor binarisation at 0.5 (what set_image_prompts applies)."""
    return None if mask is None else (mask.float() >= 0.5).float()
