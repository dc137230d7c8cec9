"""IP-Adapter image prompts (DESIGN.md §9) for the f32 CPU oracle, whose transformer blocks run the decoupled cross-attention
(oracle/unet_oracle.py): the image-token projection, the two-source attention of one prompt, and the sampler's attachment with the
engine's row rule. A prompt in forward form is (f32 adapter weights (pack names), tokens [B, S_ip, context_dim], scales
{transformer block path: s}, None)."""
from __future__ import annotations

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


def attach(wa, embeds: torch.Tensor, negative: Optional[torch.Tensor], scales: Dict[str, float]) -> O.Attach:
    """The sampler's image prompt: the CFG rows of image b use prompt b % n_batch (cond) and negative
    b % n_batch (uncond), the projection of zero embeddings when negative is None."""
    neg = torch.zeros_like(embeds) if negative is None else negative
    return O.Attach(prompts=[(wa, prompt_tokens(wa, embeds), scales, None)], uncond_tokens=[prompt_tokens(wa, neg)])


def uniform_scales(cfg, s: float) -> Dict[str, float]:
    """s for every transformer block of cfg."""
    from sdxl_b200.ip_adapter import transformer_block_paths
    return {p: s for p in transformer_block_paths(cfg)}
