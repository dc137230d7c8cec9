"""ControlNet (DESIGN.md §8): diffusers SDXL ControlNetModel files -> pack names, and the device-resident net of
sdxl_controlnet_load. A net is attached to a UNet with Diffuser.set_controls or sample(..., controls=...)."""
from __future__ import annotations

from typing import Dict, List, Tuple

import torch

from . import _lib
from ._lib import SdxlError
from .config import ControlNetConfig, block_program
from .diffusers_unet import (SDXL_DOWN_BLOCK_TYPES, _put, encoder_config, encoder_name_map, middle_name_map,  # noqa: F401
                             read_config, read_model_dir)
from .engine import AttachableModel, _cfg_struct
from .weights import controlnet_tensor_specs

# ControlNet variants this loader does not implement, recognised by a key prefix or substring
_FOREIGN = [("control_model.", "an SGM/ldm ControlNet checkpoint (convert it to diffusers format)"),
            ("task_embedding", "a ControlNet-Union checkpoint"), ("control_type_proj", "a ControlNet-Union checkpoint"),
            ("transformer_layes", "a ControlNet-Union checkpoint"), ("lora", "a Control-LoRA checkpoint"),
            ("adapter.", "a T2I-Adapter checkpoint"), ("body.", "a T2I-Adapter checkpoint")]

def config_from_diffusers(cfg: Dict) -> ControlNetConfig:
    """ControlNetConfig of a diffusers ControlNetModel config.json; everything this engine does not run is rejected by name."""
    if cfg.get("global_pool_conditions"):
        raise SdxlError("controlnet config: global_pool_conditions = true is not supported")
    unet = encoder_config(cfg, "controlnet config", int(cfg.get("in_channels", 4)))
    return ControlNetConfig(unet, hint_in_channels=int(cfg.get("conditioning_channels", 3)),
                            hint_block_channels=tuple(cfg.get("conditioning_embedding_out_channels", (16, 32, 96, 256))))


def diffusers_name_map(cfg: ControlNetConfig) -> Dict[str, Tuple[str, bool]]:
    """diffusers key -> (pack name, transpose): Linear weights are [out, in] in diffusers and [in, out] in the pack. The UNet's
    encoder half (diffusers_unet.encoder_name_map), the hint encoder, one zero conv per skip and middle_block_out."""
    def hint_encoder(m):
        _put(m, "controlnet_cond_embedding.conv_in", "input_hint_block/0")
        for k in range(2 * (len(cfg.hint_block_channels) - 1)):
            _put(m, f"controlnet_cond_embedding.blocks.{k}", f"input_hint_block/{2 * k + 2}")
        _put(m, "controlnet_cond_embedding.conv_out", f"input_hint_block/{4 * len(cfg.hint_block_channels) - 2}")

    m = encoder_name_map(cfg.unet, hint_encoder)
    ins, _, _ = block_program(cfg.unet)
    for i in range(len(ins)):
        _put(m, f"controlnet_down_blocks.{i}", f"zero_convs/{i}")
    middle_name_map(m, cfg.unet)
    _put(m, "controlnet_mid_block", "middle_block_out")
    return m


def from_diffusers(state_dict: Dict[str, torch.Tensor], config_json) -> Tuple[ControlNetConfig, Dict[str, torch.Tensor]]:
    """A diffusers SDXL ControlNetModel (state dict + config.json as dict, JSON text or path) -> (config, pack-named f16 weights).
    Unsupported variants raise SdxlError naming the key or config field. A "bgr" conditioning_channel_order is folded into the
    first hint conv (its input channels are reversed), so hints are always passed as RGB."""
    config_json = read_config(config_json)
    for k in state_dict:
        for pat, what in _FOREIGN:
            if (k.startswith(pat) if pat.endswith(".") else pat in k):
                raise SdxlError(f"controlnet: key '{k}' belongs to {what}, which is not supported")
    cfg = config_from_diffusers(config_json)
    names = diffusers_name_map(cfg)
    out: Dict[str, torch.Tensor] = {}
    for k, t in state_dict.items():
        if k not in names:
            raise SdxlError(f"controlnet: unexpected key '{k}' for an SDXL ControlNetModel")
        dst, lin = names[k]
        t = t.detach().to("cpu")
        if lin:
            t = t.reshape(t.shape[0], t.shape[1]).t()     # proj_in / proj_out may be stored as 1x1 convs
        out[dst] = t.to(torch.float16).contiguous()
    if config_json.get("controlnet_conditioning_channel_order", "rgb") == "bgr":
        out["input_hint_block/0/weight"] = out["input_hint_block/0/weight"].flip(1).contiguous()
    missing = [n for n, *_ in controlnet_tensor_specs(cfg) if n not in out]
    if missing:
        raise SdxlError(f"controlnet: tensor '{missing[0]}' is missing ({len(missing)} in all)")
    return cfg, out


def cfg_struct(cfg: ControlNetConfig) -> _lib.ControlNetCfg:
    s = _lib.ControlNetCfg()
    s.unet = _cfg_struct(cfg.unet)
    s.hint_in_channels = cfg.hint_in_channels
    s.n_hint_blocks = len(cfg.hint_block_channels)
    for i, c in enumerate(cfg.hint_block_channels):
        s.hint_block_channels[i] = c
    return s


class ControlNet(AttachableModel):
    """A device-resident ControlNet (sdxl_controlnet_load). weights: pack-named tensor dict or a built pack."""
    _load_fn, _destroy_fn, _detach_call = "sdxl_controlnet_load", "sdxl_controlnet_destroy", "set_controls([])"

    def __init__(self, ctx, cfg: ControlNetConfig, weights):
        self.cfg = cfg
        self._load(ctx, cfg_struct(cfg), weights)

    @classmethod
    def from_diffusers_dir(cls, ctx, path: str) -> "ControlNet":
        """A diffusers ControlNetModel directory: config.json + diffusion_pytorch_model[.fp16].safetensors."""
        return cls(ctx, *from_diffusers(*read_model_dir(path)))

    def embed_hint(self, hint: torch.Tensor) -> torch.Tensor:
        """hint_emb [n, mc, H/8, W/8] f32 of hint f32 [n, 3, H, W] in [0, 1] (test aid)."""
        ctx = self.ctx
        h = self.handle()
        hint = hint_tensor(hint, self.cfg.hint_in_channels).to(ctx.device).contiguous()
        n, _, H, W = hint.shape
        out = torch.empty(n, self.cfg.unet.model_channels, H // 8, W // 8, device=ctx.device, dtype=torch.float32)
        ctx.call("sdxl_controlnet_embed_hint", ctx.lib.sdxl_controlnet_embed_hint, h, n, H, W, hint.data_ptr(), 0, out.data_ptr())
        return out


def hint_tensor(hint: torch.Tensor, channels: int) -> torch.Tensor:
    """A control image as the engine takes it: f32 [n, channels, H, W] in [0, 1] is used as is, u8 [n, H, W, channels] is
    scaled by 1/255. The engine reads n * channels * H * W floats from the pointer, so any other shape is refused here."""
    if hint.dtype == torch.uint8:
        if hint.dim() != 4 or hint.shape[3] != channels:
            raise SdxlError(f"u8 control image must be [n, H, W, {channels}], got {tuple(hint.shape)}")
        return hint.permute(0, 3, 1, 2).to(torch.float32) / 255.0
    if hint.dim() != 4 or hint.shape[1] != channels:
        raise SdxlError(f"control image must be f32 [n, {channels}, H, W] or u8 [n, H, W, {channels}], got {tuple(hint.shape)}")
    return hint.to(torch.float32)


def set_controls(diffuser, controls: List) -> None:
    """sdxl_unet_set_controls with [(ControlNet, hint, scale), ...]; [] detaches."""
    ctx = diffuser.ctx
    controls = list(controls)
    if len(controls) > _lib.MAX_CONTROLS:
        raise SdxlError(f"sdxl_unet_set_controls: at most {_lib.MAX_CONTROLS} controls, got {len(controls)}")
    handles = [net.handle() for net, _, _ in controls]
    hints = [hint_tensor(h, net.cfg.hint_in_channels) for net, h, _ in controls]   # every check before any device work
    hints = [h.to(ctx.device).contiguous() for h in hints]
    arr = (_lib.Control * max(1, len(controls)))()
    for i, ((net, _, scale), h) in enumerate(zip(controls, hints)):
        arr[i].net = handles[i]
        arr[i].hint = h.data_ptr()
        arr[i].hint_on_host = 0
        arr[i].n_hint, arr[i].height, arr[i].width = h.shape[0], h.shape[2], h.shape[3]
        arr[i].scale = float(scale)
    ctx.call("sdxl_unet_set_controls", ctx.lib.sdxl_unet_set_controls, diffuser.h, len(controls), arr)
    diffuser._attach("controls", [net for net, _, _ in controls])
