"""Perturbed-attention guidance (DESIGN.md §14): diffusers' `pag_applied_layers` ids resolved to the engine's self-attention mask
(Diffuser.set_pag, sdxl_unet_set_pag), and the per-step PAG scale."""
from __future__ import annotations

import re
from typing import List, Sequence, Union

from ._lib import SdxlError
from .config import UNetConfig
from .diffusers_unet import name_map


def self_attention_names(cfg: UNetConfig) -> List[str]:
    """diffusers module names of the UNet's self-attentions (`down_blocks.1.attentions.0.transformer_blocks.1.attn1`, ...), in the
    engine's order: one per transformer block in execution order (down blocks, middle block, up blocks)."""
    tail = ".to_q.weight"
    return [k[:-len(tail)] for k in name_map(cfg) if k.endswith(".attn1" + tail)]


def _fake_integral_match(layer_id: str, name: str) -> bool:
    """diffusers' PAGMixin guard: an id ending in a number does not match a name ending in the same number by accident."""
    a, b = layer_id.split(".")[-1], name.split(".")[-1]
    return a.isnumeric() and b.isnumeric() and a == b


def layer_mask(cfg: UNetConfig, layers: Union[str, Sequence[str]]) -> List[int]:
    """The engine's layer mask (one 0/1 per self-attention, self_attention_names order) of diffusers' pag_applied_layers: each id is a
    regular expression searched (re.search) in every self-attention's module name, as PAGMixin._set_pag_attn_processor does. An id
    that matches nothing raises SdxlError."""
    ids = [layers] if isinstance(layers, str) else list(layers)
    if not ids:
        raise SdxlError("PAG: no layer ids given")
    names = self_attention_names(cfg)
    mask = [0] * len(names)
    for lid in ids:
        hits = [i for i, n in enumerate(names) if re.search(lid, n) is not None and not _fake_integral_match(lid, n)]
        if not hits:
            raise SdxlError(f"PAG: layer id {lid!r} matches no self-attention of this UNet")
        for i in hits:
            mask[i] = 1
    return mask


def pag_scale_at(t: int, scale: float, adaptive: float = 0.0, total: int = 1000) -> float:
    """The PAG scale of the step at timestep t: scale, or with adaptive scaling max(scale - adaptive * (total - t), 0) (diffusers'
    _get_pag_scale with total = 1000, the engine's cfg.n_steps)."""
    if not adaptive:
        return float(scale)
    return max(float(scale) - float(adaptive) * (total - t), 0.0)
