"""IP-Adapter image prompts (DESIGN.md §9): h94 IP-Adapter files -> pack names, the device-resident adapter of
sdxl_ip_adapter_load, and its attachment to a UNet (Diffuser.set_image_prompt, sample(..., image_prompt=...)).

The base IP-Adapter for SDXL (h94/IP-Adapter `ip-adapter_sdxl*`; diffusers ImageProjection + IPAdapterAttnProcessor2_0): an
image embedding becomes 4 tokens, LayerNorm(e @ proj + b).reshape(4, 2048), and every cross-attention adds
s * softmax(q K_ip^T / 8) V_ip to its text attention before the out projection."""
from __future__ import annotations

import ctypes as C
import re
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch

from . import _lib
from ._lib import SdxlError
from .config import UNetConfig, block_program
from .engine import _cfg_struct
from .lora import read_safetensors
from .weights import build_pack

TOKENS_PER_IMAGE = 4
# IP-Adapter variants this loader does not implement, recognised by a key substring
_FOREIGN = [("image_proj.latents", "an IP-Adapter Plus (Resampler) file"), ("image_proj.layers.", "an IP-Adapter Plus (Resampler) file"),
            ("image_proj.proj_in", "an IP-Adapter Plus (Resampler) file"), ("image_proj.proj.0.", "an IP-Adapter FaceID file"),
            ("perceiver_resampler", "an IP-Adapter FaceID Plus file"), ("lora", "an IP-Adapter FaceID file (LoRA layers)")]


def transformer_block_paths(cfg: UNetConfig) -> List[str]:
    """Reference paths of the UNet's transformer blocks in execution order (input blocks, middle, output blocks): the order of
    sdxl_image_prompt.block_scales_host."""
    ins, mid, outs = block_program(cfg)
    paths = []
    for b in ins + [mid] + outs:
        if b.depth:
            paths += [f"{b.path}/transformer/transformer_{k}" for k in range(b.depth)]
    return paths


def ip_index_map(cfg: UNetConfig) -> Dict[int, str]:
    """h94 `ip_adapter.<i>` index -> reference transformer block path.

    IP-Adapter numbers diffusers' attn_processors in module registration order (down_blocks, then up_blocks, then mid_block;
    attentions.j, then transformer_blocks.k), attn1 at 2n and attn2 at 2n + 1; only the attn2 (odd) indices carry weights.
    down_blocks.{level}.attentions.{j} is input block j of that level, up_blocks.{u}.attentions.{j} is
    output_blocks/{3u + j} and mid_block.attentions.0 is middle_block."""
    ins, mid, outs = block_program(cfg)
    down = [f"{b.path}/transformer/transformer_{k}" for b in ins if b.depth for k in range(b.depth)]   # by level, then j
    up = [f"{b.path}/transformer/transformer_{k}" for b in outs if b.depth for k in range(b.depth)]   # output_blocks in order
    mids = [f"{mid.path}/transformer/transformer_{k}" for k in range(mid.depth)]
    return {2 * n + 1: p for n, p in enumerate(down + up + mids)}


def ip_tensor_specs(cfg: UNetConfig, image_embed_dim: int, tokens: int = TOKENS_PER_IMAGE) -> List[Tuple[str, Tuple[int, ...]]]:
    """Pack names and shapes of an adapter for `cfg` (Linear weights [in, out])."""
    ctx = cfg.context_dim
    specs = [("image_proj/proj/weight", (image_embed_dim, tokens * ctx)), ("image_proj/proj/bias", (tokens * ctx,)),
             ("image_proj/norm/weight", (ctx,)), ("image_proj/norm/bias", (ctx,))]
    ins, mid, outs = block_program(cfg)
    widths = {b.path: b.c_out for b in ins + [mid] + outs}
    for p in transformer_block_paths(cfg):
        c = widths[p.split("/transformer/")[0]]
        specs += [(f"{p}/attn2/ip_key/weight", (ctx, c)), (f"{p}/attn2/ip_value/weight", (ctx, c))]
    return specs


def synth_ip_adapter(cfg: UNetConfig, image_embed_dim: int, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Deterministic synthetic f16 adapter weights (pack names) for tests and benchmarks."""
    gen = torch.Generator().manual_seed(seed)
    out = {}
    for name, shape in ip_tensor_specs(cfg, image_embed_dim):
        if name.endswith("norm/weight"):
            t = 1.0 + 0.05 * torch.randn(shape, generator=gen)
        elif name.endswith("bias"):
            t = 0.05 * torch.randn(shape, generator=gen)
        else:
            t = torch.randn(shape, generator=gen) / shape[0] ** 0.5
        out[name] = t.to(torch.float16)
    return out


def _flatten(sd: Dict) -> Dict[str, torch.Tensor]:
    """h94 `.bin` files nest {"image_proj": {...}, "ip_adapter": {...}}; `.safetensors` files are flat."""
    flat: Dict[str, torch.Tensor] = {}
    for k, v in sd.items():
        if isinstance(v, dict):
            for k2, v2 in v.items():
                flat[f"{k}.{k2}"] = v2
        else:
            flat[k] = v
    return flat


def from_h94(state_dict: Dict, cfg: UNetConfig) -> Tuple[int, Dict[str, torch.Tensor]]:
    """(image_embed_dim, pack-named f16 tensors) of an h94 IP-Adapter state dict (flat or nested). Anything that is not a base
    IP-Adapter with 4 tokens per image for `cfg` is rejected by name."""
    sd = _flatten(state_dict)
    for k in sd:
        for pat, what in _FOREIGN:
            if pat in k:
                raise SdxlError(f"IP-Adapter: key '{k}' marks {what}; only the base IP-Adapter is supported")
    if cfg.is_refiner:
        raise SdxlError("IP-Adapter: the refiner is not supported")
    ctx = cfg.context_dim
    w = sd.get("image_proj.proj.weight")
    if w is None:
        raise SdxlError("IP-Adapter: key 'image_proj.proj.weight' is missing")
    if w.dim() != 2 or w.shape[0] % ctx:
        raise SdxlError(f"IP-Adapter: 'image_proj.proj.weight' has shape {tuple(w.shape)}, not [tokens * {ctx}, D]")
    if w.shape[0] // ctx != TOKENS_PER_IMAGE:
        raise SdxlError(f"IP-Adapter: 'image_proj.proj.weight' gives {w.shape[0] // ctx} tokens per image; only "
                        f"{TOKENS_PER_IMAGE} (the base IP-Adapter) is supported")
    out = {"image_proj/proj/weight": w.t().contiguous()}
    for src, dst in (("image_proj.proj.bias", "image_proj/proj/bias"), ("image_proj.norm.weight", "image_proj/norm/weight"),
                     ("image_proj.norm.bias", "image_proj/norm/bias")):
        if src not in sd:
            raise SdxlError(f"IP-Adapter: key '{src}' is missing")
        out[dst] = sd[src]
    index = ip_index_map(cfg)
    pat = re.compile(r"^ip_adapter\.(\d+)\.to_([kv])_ip\.weight$")
    for k, t in sd.items():
        if k.startswith("image_proj."):
            if k not in ("image_proj.proj.weight", "image_proj.proj.bias", "image_proj.norm.weight", "image_proj.norm.bias"):
                raise SdxlError(f"IP-Adapter: unexpected key '{k}'")
            continue
        m = pat.match(k)
        if not m:
            raise SdxlError(f"IP-Adapter: unexpected key '{k}'")
        i = int(m.group(1))
        if i not in index:
            raise SdxlError(f"IP-Adapter: key '{k}' has no cross-attention of this UNet (expected odd indices 1..{max(index)})")
        out[f"{index[i]}/attn2/ip_{'key' if m.group(2) == 'k' else 'value'}/weight"] = t.t().contiguous()
    missing = [f"ip_adapter.{i}.to_{kv}_ip.weight" for i in index for kv in "kv"
               if f"{index[i]}/attn2/ip_{'key' if kv == 'k' else 'value'}/weight" not in out]
    if missing:
        raise SdxlError(f"IP-Adapter: key '{missing[0]}' is missing ({len(missing)} missing)")
    return int(w.shape[1]), {k: v.to(torch.float16) for k, v in out.items()}


def read_h94(path: str) -> Dict:
    """An h94 IP-Adapter file: `.safetensors` (flat keys) or `.bin` (torch.load(weights_only=True), flat or nested)."""
    if path.endswith(".safetensors"):
        return read_safetensors(path)
    return torch.load(path, map_location="cpu", weights_only=True)


def cfg_struct(cfg: UNetConfig, image_embed_dim: int) -> _lib.IpAdapterCfg:
    s = _lib.IpAdapterCfg()
    s.unet = _cfg_struct(cfg)
    s.image_embed_dim = image_embed_dim
    s.tokens_per_image = TOKENS_PER_IMAGE
    return s


class IPAdapter:
    """A device-resident IP-Adapter (sdxl_ip_adapter_load). weights: pack-named tensor dict or a built pack."""

    def __init__(self, ctx, cfg: UNetConfig, image_embed_dim: int, weights):
        self.ctx, self.cfg, self.image_embed_dim = ctx, cfg, int(image_embed_dim)
        pack = weights if isinstance(weights, torch.Tensor) else build_pack(weights)
        ctx.enter()
        if pack.is_cuda:
            torch.cuda.current_stream(ctx.device).synchronize()
        cs = cfg_struct(cfg, self.image_embed_dim)
        h = C.c_void_p()
        ctx.check(ctx.lib.sdxl_ip_adapter_load(ctx.h, C.byref(cs), pack.data_ptr(), pack.numel(), int(pack.is_cuda), C.byref(h)),
                  "sdxl_ip_adapter_load")
        self.h = h
        self.attached = 0   # attachments to UNets; close() refuses while > 0

    @classmethod
    def from_file(cls, ctx, path: str, cfg: UNetConfig) -> "IPAdapter":
        """An h94 file, e.g. `sdxl_models/ip-adapter_sdxl_vit-h.safetensors` or `ip-adapter_sdxl.bin`."""
        dim, w = from_h94(read_h94(path), cfg)
        return cls(ctx, cfg, dim, w)

    def handle(self) -> int:
        if not getattr(self, "h", None):
            raise SdxlError("IPAdapter is closed")
        return self.h.value

    def project(self, embeds: torch.Tensor) -> torch.Tensor:
        """Image tokens f16 [n * 4, context_dim] of embeddings f32 [n, D] (test aid)."""
        ctx = self.ctx
        h = self.handle()
        e = _embeds(embeds, self.image_embed_dim).reshape(-1, self.image_embed_dim).to(ctx.device).contiguous()
        out = torch.empty(e.shape[0] * TOKENS_PER_IMAGE, self.cfg.context_dim, device=ctx.device, dtype=torch.float16)
        ctx.enter()
        ctx.check(ctx.lib.sdxl_ip_adapter_project(h, e.shape[0], e.data_ptr(), 0, out.data_ptr()), "sdxl_ip_adapter_project")
        ctx.leave()
        return out

    def close(self) -> None:
        """Frees the device weights. Refused while the adapter is attached to a UNet: detach it first."""
        if getattr(self, "attached", 0) > 0:
            raise SdxlError("IPAdapter.close: the adapter is still attached to a UNet (detach it with set_image_prompt(None) first)")
        if getattr(self, "h", None):
            self.ctx.lib.sdxl_ip_adapter_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _embeds(e: torch.Tensor, dim: int) -> torch.Tensor:
    """Image embeddings as [n_batch, n_images, D] f32; [n_batch, D] is one image per prompt. The engine reads
    n_batch * n_images * D floats, so any other shape is refused here."""
    e = torch.as_tensor(e)
    if e.dim() == 2:
        e = e.unsqueeze(1)
    if e.dim() != 3 or e.shape[2] != dim or e.shape[0] < 1 or e.shape[1] < 1:
        raise SdxlError(f"image embeddings must be [n_batch, D] or [n_batch, n_images, D] with D = {dim}, got {tuple(e.shape)}")
    return e.to(torch.float32)


def set_image_prompt(diffuser, adapter: Optional[IPAdapter], embeds: Optional[torch.Tensor] = None,
                     scale: Union[float, Sequence[float]] = 1.0, negative: Optional[torch.Tensor] = None) -> None:
    """sdxl_unet_set_image_prompt; adapter None detaches. scale: one float, or one per UNet transformer block in execution order
    (transformer_block_paths). negative: embeddings of the unconditional CFG rows (default: zeros)."""
    ctx = diffuser.ctx
    if adapter is None:
        ctx.enter()
        ctx.check(ctx.lib.sdxl_unet_set_image_prompt(diffuser.h, None), "sdxl_unet_set_image_prompt")
        ctx.leave()
        release_image_prompt(diffuser)
        return
    h = adapter.handle()
    e = _embeds(embeds, adapter.image_embed_dim)
    neg = None
    if negative is not None:
        neg = _embeds(negative, adapter.image_embed_dim)
        if neg.shape != e.shape:
            raise SdxlError(f"negative image embeddings {tuple(neg.shape)} must match the embeddings {tuple(e.shape)}")
    n_tb = len(transformer_block_paths(diffuser.cfg))
    block = None
    if isinstance(scale, (int, float)):
        s0 = float(scale)
    else:
        if len(scale) != n_tb:
            raise SdxlError(f"per-block scales: {len(scale)} given, the UNet has {n_tb} transformer blocks")
        block = (C.c_float * n_tb)(*[float(v) for v in scale])
        s0 = 0.0
    e = e.to(ctx.device).contiguous()
    neg = None if neg is None else neg.to(ctx.device).contiguous()
    p = _lib.ImagePrompt()
    p.adapter, p.embeds, p.negative_embeds, p.on_host = h, e.data_ptr(), None if neg is None else neg.data_ptr(), 0
    p.n_batch, p.n_images, p.scale = e.shape[0], e.shape[1], s0
    p.block_scales_host = C.cast(block, C.c_void_p) if block is not None else None
    ctx.enter()
    ctx.check(ctx.lib.sdxl_unet_set_image_prompt(diffuser.h, C.byref(p)), "sdxl_unet_set_image_prompt")
    ctx.leave()
    release_image_prompt(diffuser)
    diffuser._image_prompt = adapter   # the adapter stays alive, and cannot be closed, while attached
    adapter.attached += 1


def release_image_prompt(diffuser) -> None:
    """Forgets the diffuser's attached adapter (after a detach, or when the UNet is destroyed)."""
    a = getattr(diffuser, "_image_prompt", None)
    if a is not None:
        a.attached -= 1
    diffuser._image_prompt = None
