"""IP-Adapter Plus image prompts (DESIGN.md §10) for the f32 CPU oracle, beside tests/ip_adapter_oracle.py: the perceiver
Resampler (h94 resampler.py, diffusers IPAdapterPlusImageProjection), the Plus prompt tokens and the sampler's attachment of a Plus
prompt (f32 adapter weights (pack names), hidden states [n_batch, n_images, L, D], negative hidden states of the same shape, scales
{transformer block path: s})."""
from __future__ import annotations

import torch

from oracle import unet_oracle as O


def perceiver_attention(x, lat, wa, p: str, n_head: int) -> torch.Tensor:
    """PerceiverAttention (h94 resampler.py) for one image: x [L, W], lat [Q, W] -> [Q, W], before the residual add. Keys and values
    are projections of cat(LN1(x), LN2(lat)); scale 1 / sqrt(64) (h94 scales q and k by 64^-1/4 each)."""
    xn = O.layer_norm(x, wa[f"{p}/norm1/weight"], wa[f"{p}/norm1/bias"])
    ln = O.layer_norm(lat, wa[f"{p}/norm2/weight"], wa[f"{p}/norm2/bias"])
    q = ln @ wa[f"{p}/to_q/weight"]
    kv = torch.cat([xn, ln], 0) @ wa[f"{p}/to_kv/weight"]
    k, v = kv.chunk(2, dim=-1)
    return O.qkv_attention(q[None], k[None], v[None], None, n_head)[0] @ wa[f"{p}/to_out/weight"]


def resample(wa, hidden: torch.Tensor) -> torch.Tensor:
    """IP-Adapter Plus Resampler (include/sdxl_b200.h): hidden [n, L, D] -> tokens [n, Q, context_dim]."""
    lat0 = wa["image_proj/latents"]
    n_head = lat0.shape[1] // 64
    depth = len({k.split("/")[2] for k in wa if k.startswith("image_proj/layers/")})
    out = []
    for h in hidden:
        x = O.linear(h, wa, "image_proj/proj_in")
        lat = lat0
        for i in range(depth):
            p = f"image_proj/layers/{i}"
            lat = lat + perceiver_attention(x, lat, wa, f"{p}/attn", n_head)
            f = O.layer_norm(lat, wa[f"{p}/ff/norm/weight"], wa[f"{p}/ff/norm/bias"])
            lat = lat + torch.nn.functional.gelu(f @ wa[f"{p}/ff/fc1/weight"]) @ wa[f"{p}/ff/fc2/weight"]
        y = O.linear(lat, wa, "image_proj/proj_out")
        out.append(O.layer_norm(y, wa["image_proj/norm_out/weight"], wa["image_proj/norm_out/bias"]))
    return torch.stack(out)


def plus_prompt_tokens(wa, hidden: torch.Tensor) -> torch.Tensor:
    """[n_batch, n_images, L, D] -> tokens [n_batch, n_images * Q, ctx], images concatenated in order."""
    nb, ni, L, d = hidden.shape
    return resample(wa, hidden.reshape(nb * ni, L, d)).reshape(nb, -1, wa["image_proj/norm_out/weight"].shape[0])


def attach(wa, hidden: torch.Tensor, negative: torch.Tensor, scales) -> O.Attach:
    """The sampler's Plus prompt: the CFG rows of image b use prompt b % n_batch (cond) and negative
    b % n_batch (uncond)."""
    return O.Attach(prompts=[(wa, plus_prompt_tokens(wa, hidden), scales, None)], uncond_tokens=[plus_prompt_tokens(wa, negative)])
