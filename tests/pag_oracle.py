"""Perturbed-attention guidance (DESIGN.md §14) for the f32 CPU oracle: the self-attention paths a layer selection names, a batch
with perturbed rows, and the sampler's PAG attachment. oracle/unet_oracle.py runs the listed self-attentions (attn1 of a
transformer block) as out(value(x)) instead of softmax attention and combines the noise as diffusers' StableDiffusionXLPAGPipeline
does, in this engine's form

    e = (u + (c - u) * guidance) + p_t * (c - ptb)      (refiner, without CFG: e = c + p_t * (c - ptb))
    p_t = max(scale - adaptive * (n_steps - t), 0)       (adaptive = 0: p_t = scale)

Every UNet op is per batch row, so a batch whose last rows are perturbed is the concatenation of a plain forward of the attended
rows and a perturbed forward of the others (forward_rows)."""
from __future__ import annotations

from typing import Collection, List, Sequence

import torch

from oracle import unet_oracle as O


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


def forward_rows(cfg, w, x, timesteps, context, label, layers: Collection[str], n_ptb: int):
    """A batch whose last n_ptb rows are perturbed (the engine's direct forward with forward_perturbed_rows = n_ptb)."""
    a = len(x) - n_ptb
    return torch.cat([O.unet_forward(cfg, w, x[:a], timesteps, context[:a], label[:a]),
                      O.unet_forward(cfg, w, x[a:], timesteps, context[a:], label[a:], O.Attach(pag_layers=layers))])


def pag_scale(t: int, scale: float, adaptive: float, total: int) -> float:
    return max(scale - adaptive * (total - t), 0.0) if adaptive else scale


def attach(cfg, layers: Collection[str], scale: float, adaptive: float = 0.0, **kw) -> O.Attach:
    """The sampler's PAG attachment (beside the attachments kw): the identity in `layers`, guidance p_t = pag_scale(t, ...)."""
    return O.Attach(pag_layers=layers, pag_scale=lambda t: pag_scale(t, scale, adaptive, cfg.n_steps), **kw)
