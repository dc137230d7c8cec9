"""diffusers UNet2DConditionModel files -> this engine's UNet (DESIGN.md §12): the config, the key map and the loader behind
Diffuser.from_diffusers_dir. Any SDXL-base-shaped UNet loads, with 4 input channels (SDXL base and its fine-tunes) or 9 (the inpainting
UNet, stable-diffusion-xl-1.0-inpainting-0.1). The encoder half of the map and the config rules are shared with sdxl_b200.controlnet,
whose ControlNetModel copies that half."""
from __future__ import annotations

import json
import os
from dataclasses import replace
from typing import Callable, Dict, Tuple

import torch

from ._lib import SdxlError
from .config import UNetConfig, block_program
from .weights import alphas_cumprod, unet_tensor_specs

SDXL_DOWN_BLOCK_TYPES = ["DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"]
SDXL_UP_BLOCK_TYPES = ["CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"]

_RES = {"norm1": "norm_in", "conv1": "conv_in", "time_emb_proj": "lin_embed", "norm2": "norm_out", "conv2": "conv_out",
        "conv_shortcut": "skip_connection"}
_ATTN = {"to_q": "query", "to_k": "key", "to_v": "value", "to_out.0": "out"}

# config.json fields the engine computes one way only: (field, diffusers default, the value this engine runs)
_FIXED = [("addition_embed_type", None, "text_time"), ("class_embed_type", None, None), ("use_linear_projection", False, True),
          ("layers_per_block", 2, 2), ("norm_num_groups", 32, 32), ("flip_sin_to_cos", True, True), ("freq_shift", 0, 0),
          ("time_embedding_type", "positional", "positional"), ("resnet_time_scale_shift", "default", "default"),
          ("mid_block_type", "UNetMidBlock2DCrossAttn", "UNetMidBlock2DCrossAttn"), ("encoder_hid_dim_type", None, None),
          ("time_cond_proj_dim", None, None), ("conv_in_kernel", 3, 3), ("conv_out_kernel", 3, 3)]

Names = Dict[str, Tuple[str, bool]]


def read_config(config_json) -> Dict:
    """config.json as a dict, JSON text or path."""
    if isinstance(config_json, str):
        if os.path.exists(config_json):
            with open(config_json) as f:
                return json.load(f)
        return json.loads(config_json)
    return dict(config_json)


def encoder_config(cfg: Dict, what: str, in_channels: int, out_channels: int = 4) -> UNetConfig:
    """The UNetConfig of the fields a UNet2DConditionModel and a ControlNetModel config.json share (the encoder half): SDXL base's
    down blocks and head dim 64 only, refused by field name with `what` as the message prefix."""
    dbt = list(cfg.get("down_block_types", []))
    if dbt != SDXL_DOWN_BLOCK_TYPES:
        raise SdxlError(f"{what}: down_block_types {dbt} is not SDXL base's {SDXL_DOWN_BLOCK_TYPES}")
    ch = list(cfg["block_out_channels"])
    mc = ch[0]
    heads = cfg.get("num_attention_heads") or cfg.get("attention_head_dim")
    heads = list(heads) if isinstance(heads, (list, tuple)) else [heads] * len(ch)
    for lvl, t in enumerate(dbt):
        if t.startswith("CrossAttn") and ch[lvl] != 64 * heads[lvl]:
            raise SdxlError(f"{what}: attention_head_dim gives head dim {ch[lvl] // heads[lvl]} at level {lvl}; only 64 is supported")
    tl = cfg.get("transformer_layers_per_block", 1)
    tl = list(tl) if isinstance(tl, (list, tuple)) else [tl] * len(ch)
    depths = tuple(tl[lvl] if t.startswith("CrossAttn") else 0 for lvl, t in enumerate(dbt))
    return UNetConfig(adm_in_channels=int(cfg["projection_class_embeddings_input_dim"]), model_channels=mc,
                      channel_mults=tuple(c // mc for c in ch), transformer_depths=depths, context_dim=int(cfg["cross_attention_dim"]),
                      in_channels=in_channels, out_channels=out_channels)


def config_from_diffusers(config_json) -> UNetConfig:
    """UNetConfig of a diffusers UNet2DConditionModel config.json (dict, JSON text or path). SDXL-base-shaped UNets with
    in_channels = out_channels (4), 2 * out_channels + 1 (9, the inpainting layout) or 2 * out_channels (8, the InstructPix2Pix edit
    layout) are accepted; every other field this engine does not run is refused by name."""
    cfg = read_config(config_json)
    what = "unet config"
    ubt = list(cfg.get("up_block_types", []))
    if ubt != SDXL_UP_BLOCK_TYPES:
        raise SdxlError(f"{what}: up_block_types {ubt} is not SDXL base's {SDXL_UP_BLOCK_TYPES}")
    for field, default, want in _FIXED:
        got = cfg.get(field, default)
        if got != want:
            raise SdxlError(f"{what}: {field} = {got!r} is not supported (only {want!r})")
    rev = cfg.get("reverse_transformer_layers_per_block")
    if rev is not None:
        raise SdxlError(f"{what}: reverse_transformer_layers_per_block is not supported (the up blocks mirror the down blocks)")
    out_ch = int(cfg.get("out_channels", 4))
    in_ch = int(cfg.get("in_channels", 4))
    if out_ch != 4:
        raise SdxlError(f"{what}: out_channels = {out_ch} is not supported (only 4)")
    if in_ch not in (out_ch, 2 * out_ch + 1, 2 * out_ch):
        raise SdxlError(f"{what}: in_channels = {in_ch} is not supported (only {out_ch}, {2 * out_ch + 1} for inpainting or "
                        f"{2 * out_ch} for editing)")
    return replace(encoder_config(cfg, what, in_ch, out_ch), is_edit=in_ch == 2 * out_ch)


def _put(m: Names, src: str, dst: str, lin: bool = False) -> None:
    """weight and bias of one layer; lin: a Linear ([out, in] in diffusers, [in, out] in the pack)."""
    m[f"{src}.weight"] = (f"{dst}/weight", lin)
    m[f"{src}.bias"] = (f"{dst}/bias", False)


def _res(m: Names, src: str, dst: str, has_skip: bool) -> None:
    for a, b in _RES.items():
        if a != "conv_shortcut" or has_skip:
            _put(m, f"{src}.{a}", f"{dst}/{b}", a == "time_emb_proj")


def _st(m: Names, src: str, dst: str, depth: int) -> None:
    _put(m, f"{src}.norm", f"{dst}/norm")
    _put(m, f"{src}.proj_in", f"{dst}/proj_in", True)
    _put(m, f"{src}.proj_out", f"{dst}/proj_out", True)
    for j in range(depth):
        s, d = f"{src}.transformer_blocks.{j}", f"{dst}/transformer_{j}"
        for n in ("norm1", "norm2", "norm3"):
            _put(m, f"{s}.{n}", f"{d}/{n}")
        for a in ("attn1", "attn2"):
            for x, y in _ATTN.items():
                if x == "to_out.0":
                    _put(m, f"{s}.{a}.{x}", f"{d}/{a}/{y}", True)
                else:
                    m[f"{s}.{a}.{x}.weight"] = (f"{d}/{a}/{y}/weight", True)
        _put(m, f"{s}.ff.net.0.proj", f"{d}/mlp/geglu/proj", True)
        _put(m, f"{s}.ff.net.2", f"{d}/mlp/lin", True)


def encoder_name_map(cfg: UNetConfig, extra: Callable[[Names], None] = None) -> Names:
    """diffusers key -> (pack name, transpose) of the embeddings, conv_in, the down blocks and the middle block. extra(m) runs after
    the embeddings (a ControlNet's hint encoder); a ControlNet adds its zero convs around the middle block itself."""
    m: Names = {}
    ins, mid, _ = block_program(cfg)
    _put(m, "conv_in", ins[0].path)
    _put(m, "time_embedding.linear_1", "lin1_time_embed", True)
    _put(m, "time_embedding.linear_2", "lin2_time_embed", True)
    _put(m, "add_embedding.linear_1", "lin1_label_embed", True)
    _put(m, "add_embedding.linear_2", "lin2_label_embed", True)
    if extra is not None:
        extra(m)
    lvl, j = 0, 0   # diffusers numbers the blocks of a level: resnets.{j} / attentions.{j}, then the level's downsampler
    for b in ins[1:]:
        if b.kind == "downsample":
            _put(m, f"down_blocks.{lvl}.downsamplers.0.conv", b.path)
            lvl, j = lvl + 1, 0
            continue
        tr = b.kind == "resnet_transformer"
        _res(m, f"down_blocks.{lvl}.resnets.{j}", f"{b.path}/res" if tr else b.path, b.c_in != b.c_out)
        if tr:
            _st(m, f"down_blocks.{lvl}.attentions.{j}", f"{b.path}/transformer", b.depth)
        j += 1
    return m


def middle_name_map(m: Names, cfg: UNetConfig) -> None:
    _, mid, _ = block_program(cfg)
    _res(m, "mid_block.resnets.0", f"{mid.path}/res1", False)
    _st(m, "mid_block.attentions.0", f"{mid.path}/transformer", mid.depth)
    _res(m, "mid_block.resnets.1", f"{mid.path}/res2", False)


def name_map(cfg: UNetConfig) -> Names:
    """diffusers UNet2DConditionModel key -> (pack name, transpose) for the whole UNet: output block i is up_blocks.{i // 3}
    resnets / attentions.{i % 3}, the level's upsampler after its third block; then conv_norm_out and conv_out."""
    m = encoder_name_map(cfg)
    middle_name_map(m, cfg)
    _, _, outs = block_program(cfg)
    for i, b in enumerate(outs):
        k, j = divmod(i, 3)
        res_dst = b.path if b.kind == "resnet" else f"{b.path}/res"
        _res(m, f"up_blocks.{k}.resnets.{j}", res_dst, b.c_in != b.c_out)
        if "transformer" in b.kind:
            _st(m, f"up_blocks.{k}.attentions.{j}", f"{b.path}/transformer", b.depth)
        if b.kind.endswith("upsample"):
            _put(m, f"up_blocks.{k}.upsamplers.0.conv", f"{b.path}/upsample/conv")
    _put(m, "conv_norm_out", "norm_out")
    _put(m, "conv_out", "conv_out")
    return m


def from_diffusers(state_dict: Dict[str, torch.Tensor], config_json) -> Tuple[UNetConfig, Dict[str, torch.Tensor]]:
    """A diffusers SDXL UNet2DConditionModel (state dict + config.json as dict, JSON text or path) -> (config, pack-named f16 weights
    with alphas_cumprod, ready for Diffuser). Unknown keys, missing keys and wrong shapes raise SdxlError naming the key. The alphas
    are SDXL's scaled-linear schedule (weights.alphas_cumprod), which the UNet's files do not carry."""
    cfg = config_from_diffusers(config_json)
    names = name_map(cfg)
    shapes = {n: s for n, s, *_ in unet_tensor_specs(cfg)}
    out: Dict[str, torch.Tensor] = {}
    for k, t in state_dict.items():
        if k not in names:
            raise SdxlError(f"unet: unexpected key '{k}' for an SDXL UNet2DConditionModel")
        dst, lin = names[k]
        want = shapes[dst][::-1] if lin else shapes[dst]
        if tuple(t.shape) != tuple(want):
            raise SdxlError(f"unet: key '{k}' has shape {tuple(t.shape)}, expected {tuple(want)}")
        t = t.detach().to("cpu")
        out[dst] = (t.t() if lin else t).to(torch.float16).contiguous()
    missing = [k for k, (dst, _) in names.items() if dst not in out]
    if missing:
        raise SdxlError(f"unet: key '{missing[0]}' is missing ({len(missing)} in all)")
    out["alphas_cumprod"] = alphas_cumprod(cfg.n_steps)
    return cfg, out


def read_model_dir(path: str) -> Tuple[Dict[str, torch.Tensor], str]:
    """(state dict, config.json path) of a diffusers model directory (a UNet, ControlNetModel or T2IAdapter): config.json +
    diffusion_pytorch_model[.fp16].safetensors, the fp16 file when both are there."""
    from .lora import read_safetensors
    files = [f for f in ("diffusion_pytorch_model.fp16.safetensors", "diffusion_pytorch_model.safetensors")
             if os.path.exists(os.path.join(path, f))]
    if not files:
        raise SdxlError(f"{path}: no diffusion_pytorch_model[.fp16].safetensors")
    return read_safetensors(os.path.join(path, files[0])), os.path.join(path, "config.json")
