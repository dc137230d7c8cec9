"""T2I-Adapter (DESIGN.md §11): diffusers SDXL T2IAdapter files (adapter_type "full_adapter_xl") -> pack names, the device-resident
adapter of sdxl_t2i_adapter_load, and its attachment to a UNet with Diffuser.set_t2i_adapters or sample(..., t2i_adapters=...)."""
from __future__ import annotations

import re
from typing import Dict, List, Sequence, Tuple

import torch

from . import _lib
from ._lib import SdxlError
from .config import SDXL_BASE, T2IAdapterConfig, UNetConfig, block_program
from .controlnet import hint_tensor
from .diffusers_unet import read_config, read_model_dir
from .engine import AttachableModel, _cfg_struct, ddim_timesteps
from .weights import t2i_adapter_tensor_specs

# adapter types diffusers' T2IAdapter knows that this engine does not run
_OTHER_TYPES = {"full_adapter": "the SD1.5 full adapter", "light_adapter": "the SD1.5 light adapter",
                "multi_adapter": "a MultiAdapter config (attach several adapters instead)"}


def config_from_diffusers(cfg: Dict, unet: UNetConfig = SDXL_BASE) -> T2IAdapterConfig:
    """T2IAdapterConfig of a diffusers T2IAdapter config.json for `unet`; everything this engine does not run is rejected by name."""
    kind = cfg.get("adapter_type", "full_adapter")
    if kind != "full_adapter_xl":
        raise SdxlError(f"t2i-adapter config: adapter_type '{kind}' ({_OTHER_TYPES.get(kind, 'unknown')}) is not supported; "
                        "only 'full_adapter_xl' is")
    if int(cfg.get("downscale_factor", 8)) != 16:
        raise SdxlError(f"t2i-adapter config: downscale_factor {cfg.get('downscale_factor', 8)} is not 16")
    out = T2IAdapterConfig(unet, in_channels=int(cfg.get("in_channels", 3)), n_res_blocks=int(cfg.get("num_res_blocks", 2)))
    ch = tuple(cfg.get("channels", ()))
    if ch != out.channels:
        raise SdxlError(f"t2i-adapter config: channels {list(ch)} are not the widths {list(out.channels)} of the UNet")
    return out


_KEY = re.compile(r"adapter\.(conv_in|body\.[0-9]+\.in_conv|body\.[0-9]+\.resnets\.[0-9]+\.block[12])\.(weight|bias)")


def from_diffusers(state_dict: Dict[str, torch.Tensor], config_json, unet: UNetConfig = SDXL_BASE
                   ) -> Tuple[T2IAdapterConfig, Dict[str, torch.Tensor]]:
    """A diffusers SDXL T2IAdapter (state dict + config.json as dict, JSON text or path) -> (config, pack-named f16 weights).
    Unknown keys, missing tensors and wrong shapes raise SdxlError naming the key."""
    cfg = config_from_diffusers(read_config(config_json), unet)
    specs = {name: shape for name, shape, _, _ in t2i_adapter_tensor_specs(cfg)}
    out: Dict[str, torch.Tensor] = {}
    for k, t in state_dict.items():
        m = _KEY.fullmatch(k)
        name = f"{m.group(1).replace('.', '/')}/{m.group(2)}" if m else None
        if name not in specs:
            raise SdxlError(f"t2i-adapter: unexpected key '{k}' for an SDXL full_adapter_xl")
        if tuple(t.shape) != specs[name]:
            raise SdxlError(f"t2i-adapter: '{k}' has shape {list(t.shape)}, expected {list(specs[name])}")
        out[name] = t.detach().to("cpu", torch.float16).contiguous()
    missing = [n for n in specs if n not in out]
    if missing:
        raise SdxlError(f"t2i-adapter: tensor '{missing[0]}' is missing ({len(missing)} in all)")
    return cfg, out


def cfg_struct(cfg: T2IAdapterConfig) -> _lib.T2IAdapterCfg:
    s = _lib.T2IAdapterCfg()
    s.unet = _cfg_struct(cfg.unet)
    s.in_channels = cfg.in_channels
    s.n_res_blocks = cfg.n_res_blocks
    return s


def injection_points(cfg: UNetConfig) -> List[str]:
    """The blocks whose outputs receive F_0..F_3: per level the last input block with a transformer or, on a level without one,
    its last input block (the Downsample where it has one); then the middle block. Refuses cfgs that are not SDXL-base-shaped."""
    if cfg.is_refiner or cfg.n_levels != 3 or cfg.transformer_depths[0] != 0:
        raise SdxlError("t2i-adapter: only an SDXL-base-shaped UNet (3 levels, no refiner, no transformer on level 0) takes one")
    ins, mid, _ = block_program(cfg)
    levels: List[List] = [[], [], []]
    lv = 0
    for b in ins[1:]:   # a Downsample reads its level; the blocks after it run at the next
        levels[lv].append(b)
        lv += b.kind == "downsample"
    pts = []
    for blocks in levels:
        tr = [b for b in blocks if "transformer" in b.kind]
        pts.append((tr or blocks)[-1].path)
    return pts + [mid.path]


def t2i_t_min(n_steps: int, factor: float, step_start: int = 0, total: int = 1000) -> int:
    """t_min of diffusers' adapter_conditioning_factor: the features are added on the first int(n_iter * factor) sampler
    iterations, i.e. at timesteps t >= t_min; a t_min above every timestep when that count is 0."""
    ts = ddim_timesteps(n_steps, step_start, total)
    k = int(len(ts) * factor)
    return total if k <= 0 else ts[min(k, len(ts)) - 1]


class T2IAdapter(AttachableModel):
    """A device-resident T2I-Adapter (sdxl_t2i_adapter_load). weights: pack-named tensor dict or a built pack."""
    _load_fn, _destroy_fn, _detach_call = "sdxl_t2i_adapter_load", "sdxl_t2i_adapter_destroy", "set_t2i_adapters([])"

    def __init__(self, ctx, cfg: T2IAdapterConfig, weights):
        self.cfg = cfg
        self._load(ctx, cfg_struct(cfg), weights)

    @classmethod
    def from_diffusers_dir(cls, ctx, path: str, unet: UNetConfig = SDXL_BASE) -> "T2IAdapter":
        """A diffusers T2IAdapter directory: config.json + diffusion_pytorch_model[.fp16].safetensors."""
        return cls(ctx, *from_diffusers(*read_model_dir(path), unet))

    def features(self, hint: torch.Tensor) -> List[torch.Tensor]:
        """The four features F_k f32 [n, ch_k, H/16 or H/32, ...] of hint f32 [n, C, H, W] in [0, 1] or u8 [n, H, W, C] (test aid)."""
        ctx = self.ctx
        h = self.handle()
        hint = hint_tensor(hint, self.cfg.in_channels).to(ctx.device).contiguous()
        n, _, H, W = hint.shape
        shapes = [(n, c, H // d, W // d) for c, d in zip(self.cfg.channels, (16, 16, 32, 32))]
        out = torch.empty(sum(int(torch.Size(s).numel()) for s in shapes), device=ctx.device, dtype=torch.float32)
        ctx.call("sdxl_t2i_adapter_features", ctx.lib.sdxl_t2i_adapter_features, h, n, H, W, hint.data_ptr(), 0, out.data_ptr())
        return [p.reshape(s) for p, s in zip(out.split([int(torch.Size(s).numel()) for s in shapes]), shapes)]


def set_t2i_adapters(diffuser, items: Sequence, t_min: int = 0) -> None:
    """sdxl_unet_set_t2i_adapters with [(T2IAdapter, hint, scale), ...]; [] detaches. hint: u8 [n, H, W, C] or f32 [n, C, H, W]."""
    ctx = diffuser.ctx
    items = list(items)
    if len(items) > _lib.MAX_T2I_ADAPTERS:
        raise SdxlError(f"sdxl_unet_set_t2i_adapters: at most {_lib.MAX_T2I_ADAPTERS} adapters, got {len(items)}")
    handles = [ad.handle() for ad, _, _ in items]
    # the C call reads n * in_channels * H * W floats from each pointer: the channel count is checked here
    hints = [hint_tensor(h, ad.cfg.in_channels).to(ctx.device).contiguous() for ad, h, _ in items]
    arr = (_lib.T2IControl * max(1, len(items)))()
    for i, ((_, _, scale), h) in enumerate(zip(items, hints)):
        arr[i].adapter = handles[i]
        arr[i].hint = h.data_ptr()
        arr[i].hint_on_host = 0
        arr[i].n_hint, arr[i].height, arr[i].width = h.shape[0], h.shape[2], h.shape[3]
        arr[i].scale = float(scale)
    ctx.call("sdxl_unet_set_t2i_adapters", ctx.lib.sdxl_unet_set_t2i_adapters, diffuser.h, len(items), arr, int(t_min))
    diffuser._attach("t2i_adapters", [ad for ad, _, _ in items])
