"""CLIP vision encoder (DESIGN.md §9): HF CLIPVisionModelWithProjection weights -> pack names, the device-resident encoder of
sdxl_clip_vision_load, and clip_preprocess, the CLIPImageProcessor pipeline in torch. Its image_embeds feed IP-Adapter."""
from __future__ import annotations

import ctypes as C
import json
from dataclasses import dataclass
from typing import Dict, Optional, Tuple, Union

import torch
import torch.nn.functional as F

from . import _lib
from ._lib import SdxlError
from .weights import build_pack

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


@dataclass(frozen=True)
class ClipVisionConfig:
    """HF CLIPVisionConfig fields the encoder runs (hidden_size, num_attention_heads, num_hidden_layers, intermediate_size,
    image_size, patch_size, projection_dim, hidden_act)."""
    n_state: int
    n_head: int
    n_layer: int
    mlp_dim: int
    proj_dim: int
    image_size: int = 224
    patch_size: int = 14
    quick_gelu: bool = False

    @property
    def n_tokens(self) -> int:
        return (self.image_size // self.patch_size) ** 2 + 1


# the image encoders of h94's SDXL adapters: ip-adapter_sdxl_vit-h (ViT-H/14) and ip-adapter_sdxl (ViT-bigG/14)
SDXL_VIT_H = ClipVisionConfig(n_state=1280, n_head=16, n_layer=32, mlp_dim=5120, proj_dim=1024)
SDXL_VIT_BIGG = ClipVisionConfig(n_state=1664, n_head=16, n_layer=48, mlp_dim=8192, proj_dim=1280)
# small instances for known-answer tests: head dims 80 and 104, an MLP width that is not 4 * n_state
TINY_VIT_80 = ClipVisionConfig(n_state=160, n_head=2, n_layer=2, mlp_dim=384, proj_dim=48, image_size=56)
TINY_VIT_104 = ClipVisionConfig(n_state=208, n_head=2, n_layer=3, mlp_dim=512, proj_dim=64, image_size=42)


def vision_tensor_specs(cfg: ClipVisionConfig):
    """(pack name, shape, kind) of every tensor; Linear weights [in, out]."""
    C_, p = cfg.n_state, cfg.patch_size
    specs = [("patch_embedding/weight", (C_, 3, p, p), "conv"), ("class_embedding", (C_,), "embed"),
             ("position_embedding/weight", (cfg.n_tokens, C_), "embed"),
             ("pre_layernorm/weight", (C_,), "gamma"), ("pre_layernorm/bias", (C_,), "beta")]
    for i in range(cfg.n_layer):
        b = f"blocks/{i}"
        for n in ("attn_ln", "mlp_ln"):
            specs += [(f"{b}/{n}/weight", (C_,), "gamma"), (f"{b}/{n}/bias", (C_,), "beta")]
        for n in ("query", "key", "value", "out"):
            specs += [(f"{b}/attn/{n}/weight", (C_, C_), "linear"), (f"{b}/attn/{n}/bias", (C_,), "bias")]
        specs += [(f"{b}/mlp/fc1/weight", (C_, cfg.mlp_dim), "linear"), (f"{b}/mlp/fc1/bias", (cfg.mlp_dim,), "bias"),
                  (f"{b}/mlp/fc2/weight", (cfg.mlp_dim, C_), "linear"), (f"{b}/mlp/fc2/bias", (C_,), "bias")]
    specs += [("post_layernorm/weight", (C_,), "gamma"), ("post_layernorm/bias", (C_,), "beta"),
              ("visual_projection", (C_, cfg.proj_dim), "linear")]
    return specs


def synth_vision_weights(cfg: ClipVisionConfig, seed: int = 0, device: str = "cpu") -> Dict[str, torch.Tensor]:
    """Deterministic (per device type) synthetic f16 weights in pack names."""
    gen = torch.Generator(device=device).manual_seed(seed)
    out = {}
    for name, shape, kind in vision_tensor_specs(cfg):
        r = torch.randn(shape, generator=gen, device=device)
        if kind == "linear":
            t = r / shape[0] ** 0.5
        elif kind == "conv":
            t = r / (shape[1] * shape[2] * shape[3]) ** 0.5
        elif kind == "embed":
            t = r * 0.5
        elif kind == "gamma":
            t = 1.0 + 0.05 * r
        else:
            t = 0.05 * r
        out[name] = t.to(torch.float16)
    return out


_HF_BLOCK = {"layer_norm1": "attn_ln", "layer_norm2": "mlp_ln", "self_attn.q_proj": "attn/query", "self_attn.k_proj": "attn/key",
             "self_attn.v_proj": "attn/value", "self_attn.out_proj": "attn/out", "mlp.fc1": "mlp/fc1", "mlp.fc2": "mlp/fc2"}


def hf_name_map(cfg: ClipVisionConfig) -> Dict[str, Tuple[str, bool]]:
    """HF key -> (pack name, transpose): HF Linear weights are [out, in], the pack's [in, out]."""
    m = {"vision_model.embeddings.patch_embedding.weight": ("patch_embedding/weight", False),
         "vision_model.embeddings.class_embedding": ("class_embedding", False),
         "vision_model.embeddings.position_embedding.weight": ("position_embedding/weight", False),
         "vision_model.pre_layrnorm.weight": ("pre_layernorm/weight", False), "vision_model.pre_layrnorm.bias": ("pre_layernorm/bias", False),
         "vision_model.post_layernorm.weight": ("post_layernorm/weight", False),
         "vision_model.post_layernorm.bias": ("post_layernorm/bias", False), "visual_projection.weight": ("visual_projection", True)}
    for i in range(cfg.n_layer):
        for src, dst in _HF_BLOCK.items():
            lin = "proj" in src or "fc" in src
            m[f"vision_model.encoder.layers.{i}.{src}.weight"] = (f"blocks/{i}/{dst}/weight", lin)
            m[f"vision_model.encoder.layers.{i}.{src}.bias"] = (f"blocks/{i}/{dst}/bias", False)
    return m


def config_from_hf(cfg: Union[Dict, str]) -> ClipVisionConfig:
    """ClipVisionConfig of an HF CLIPVisionConfig (dict, JSON text or path; a full CLIPConfig's vision_config is accepted)."""
    if isinstance(cfg, str):
        cfg = json.loads(cfg) if cfg.lstrip().startswith("{") else json.load(open(cfg))
    cfg = cfg.get("vision_config", cfg)
    act = cfg.get("hidden_act", "quick_gelu")
    if act not in ("gelu", "quick_gelu"):
        raise SdxlError(f"vision config: hidden_act {act!r} is not supported (gelu, quick_gelu)")
    return ClipVisionConfig(n_state=int(cfg["hidden_size"]), n_head=int(cfg["num_attention_heads"]), n_layer=int(cfg["num_hidden_layers"]),
                            mlp_dim=int(cfg["intermediate_size"]), proj_dim=int(cfg["projection_dim"]),
                            image_size=int(cfg.get("image_size", 224)), patch_size=int(cfg.get("patch_size", 14)), quick_gelu=act == "quick_gelu")


def from_hf(state_dict: Dict[str, torch.Tensor], config) -> Tuple[ClipVisionConfig, Dict[str, torch.Tensor]]:
    """(config, pack-named f16 tensors) of a CLIPVisionModelWithProjection state dict; `vision_model.embeddings.position_ids`
    is a buffer and is skipped, any other unknown key is rejected by name."""
    cfg = config_from_hf(config) if not isinstance(config, ClipVisionConfig) else config
    m = hf_name_map(cfg)
    out = {}
    for k, t in state_dict.items():
        if k.endswith("position_ids"):
            continue
        if k not in m:
            raise SdxlError(f"vision encoder: unexpected key '{k}'")
        name, tr = m[k]
        out[name] = (t.t() if tr else t).contiguous().to(torch.float16)
    missing = [k for k, (n, _) in m.items() if n not in out]
    if missing:
        raise SdxlError(f"vision encoder: key '{missing[0]}' is missing ({len(missing)} missing)")
    return cfg, out


def to_hf(weights: Dict[str, torch.Tensor], cfg: ClipVisionConfig) -> Dict[str, torch.Tensor]:
    """Inverse of from_hf (f32): pack names -> HF keys."""
    return {k: (weights[n].t() if tr else weights[n]).float().contiguous() for k, (n, tr) in hf_name_map(cfg).items()}


def clip_preprocess(rgb: torch.Tensor, size: int = 224) -> torch.Tensor:
    """CLIPImageProcessor in torch: u8 [N, H, W, 3] or [H, W, 3] -> f32 [N, 3, size, size]. Shortest side to `size` (bicubic,
    antialiased), centre crop, / 255, CLIP mean / std. PIL's bicubic filter and torch's differ by a few u8 levels at edges."""
    if rgb.dim() == 3:
        rgb = rgb.unsqueeze(0)
    if rgb.dim() != 4 or rgb.shape[3] != 3 or rgb.dtype != torch.uint8:
        raise SdxlError(f"clip_preprocess: expected u8 [N, H, W, 3], got {rgb.dtype} {tuple(rgb.shape)}")
    x = rgb.permute(0, 3, 1, 2).float()
    h, w = x.shape[2], x.shape[3]
    s = size / min(h, w)
    nh, nw = (size, max(size, int(round(w * s)))) if h <= w else (max(size, int(round(h * s))), size)
    x = F.interpolate(x, size=(nh, nw), mode="bicubic", antialias=True, align_corners=False).round().clamp(0, 255)
    top, left = (nh - size) // 2, (nw - size) // 2
    x = x[:, :, top:top + size, left:left + size] / 255.0
    mean = torch.tensor(CLIP_MEAN).view(1, 3, 1, 1)
    std = torch.tensor(CLIP_STD).view(1, 3, 1, 1)
    return (x - mean) / std


def cfg_struct(cfg: ClipVisionConfig) -> _lib.ClipVisionCfg:
    s = _lib.ClipVisionCfg()
    s.n_state, s.n_head, s.n_layer, s.mlp_dim = cfg.n_state, cfg.n_head, cfg.n_layer, cfg.mlp_dim
    s.image_size, s.patch_size, s.proj_dim, s.quick_gelu = cfg.image_size, cfg.patch_size, cfg.proj_dim, int(cfg.quick_gelu)
    return s


class ClipVisionEncoder:
    """A device-resident CLIP vision encoder (sdxl_clip_vision_load). weights: pack-named tensor dict or a built pack."""

    def __init__(self, ctx, cfg: ClipVisionConfig, weights):
        self.ctx, self.cfg = ctx, cfg
        pack = weights if isinstance(weights, torch.Tensor) else build_pack(weights)
        ctx.enter()
        if pack.is_cuda:
            torch.cuda.current_stream(ctx.device).synchronize()
        cs = cfg_struct(cfg)
        h = C.c_void_p()
        ctx.check(ctx.lib.sdxl_clip_vision_load(ctx.h, C.byref(cs), pack.data_ptr(), pack.numel(), int(pack.is_cuda), C.byref(h)),
                  "sdxl_clip_vision_load")
        self.h = h

    @classmethod
    def from_hf(cls, ctx, state_dict: Dict[str, torch.Tensor], config_json) -> "ClipVisionEncoder":
        cfg, w = from_hf(state_dict, config_json)
        return cls(ctx, cfg, w)

    def encode(self, pixels: torch.Tensor) -> torch.Tensor:
        """image_embeds f32 [N, proj_dim] of preprocessed pixels f32 [N, 3, S, S] (clip_preprocess)."""
        ctx, g = self.ctx, self.cfg
        if pixels.dim() != 4 or tuple(pixels.shape[1:]) != (3, g.image_size, g.image_size):
            raise SdxlError(f"encode: pixels must be [N, 3, {g.image_size}, {g.image_size}], got {tuple(pixels.shape)}")
        px = pixels.to(ctx.device, torch.float32).contiguous()
        out = torch.empty(px.shape[0], g.proj_dim, device=ctx.device, dtype=torch.float32)
        ctx.enter()
        ctx.check(ctx.lib.sdxl_clip_vision_encode(self.h, px.shape[0], px.data_ptr(), 0, out.data_ptr()), "sdxl_clip_vision_encode")
        ctx.leave()
        return out

    def encode_images(self, rgb: torch.Tensor) -> torch.Tensor:
        """image_embeds of u8 images [N, H, W, 3]."""
        return self.encode(clip_preprocess(rgb, self.cfg.image_size))

    def encode_hidden(self, pixels: torch.Tensor, hidden_idx: Optional[int] = None) -> torch.Tensor:
        """HF hidden_states[hidden_idx] f32 [N, T, n_state] of preprocessed pixels f32 [N, 3, S, S]; hidden_idx in [0, n_layer],
        default n_layer - 1 (hidden_states[-2], the image features of IP-Adapter Plus)."""
        ctx, g = self.ctx, self.cfg
        idx = g.n_layer - 1 if hidden_idx is None else int(hidden_idx)
        if pixels.dim() != 4 or tuple(pixels.shape[1:]) != (3, g.image_size, g.image_size):
            raise SdxlError(f"encode_hidden: pixels must be [N, 3, {g.image_size}, {g.image_size}], got {tuple(pixels.shape)}")
        if not 0 <= idx <= g.n_layer:
            raise SdxlError(f"encode_hidden: hidden_idx {idx} outside [0, {g.n_layer}]")
        px = pixels.to(ctx.device, torch.float32).contiguous()
        out = torch.empty(px.shape[0], g.n_tokens, g.n_state, device=ctx.device, dtype=torch.float32)
        ctx.enter()
        ctx.check(ctx.lib.sdxl_clip_vision_encode_hidden(self.h, px.shape[0], px.data_ptr(), 0, idx, out.data_ptr()),
                  "sdxl_clip_vision_encode_hidden")
        ctx.leave()
        return out

    def encode_images_hidden(self, rgb: torch.Tensor) -> torch.Tensor:
        """hidden_states[-2] of u8 images [N, H, W, 3]."""
        return self.encode_hidden(clip_preprocess(rgb, self.cfg.image_size))

    def close(self) -> None:
        if getattr(self, "h", None):
            self.ctx.lib.sdxl_clip_vision_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
