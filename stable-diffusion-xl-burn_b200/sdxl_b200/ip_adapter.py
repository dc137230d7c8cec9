"""IP-Adapter image prompts (DESIGN.md §9): h94 IP-Adapter files -> pack names, the device-resident adapter of
sdxl_ip_adapter_load, and its attachment to a UNet (Diffuser.set_image_prompt, sample(..., image_prompt=...)).

The base IP-Adapter for SDXL (h94/IP-Adapter `ip-adapter_sdxl*`; diffusers ImageProjection + IPAdapterAttnProcessor2_0): an
image embedding becomes 4 tokens, LayerNorm(e @ proj + b).reshape(4, 2048), and every cross-attention adds
s * softmax(q K_ip^T / 8) V_ip to its text attention before the out projection.

IP-Adapter Plus (h94 `ip-adapter-plus*_sdxl_vit-h`; diffusers IPAdapterPlusImageProjection): the image features are the vision
encoder's penultimate hidden states [257, 1280], and a perceiver Resampler (ResamplerConfig) turns them into 16 tokens; the negative
is the Resampler of the hidden states of an all-zero pixel tensor. The UNet side is the same as for the base adapter."""
from __future__ import annotations

import ctypes as C
import re
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch

from . import _lib
from ._lib import SdxlError
from .config import UNetConfig, block_program
from .engine import AttachableModel, _cfg_struct
from .lora import read_safetensors

TOKENS_PER_IMAGE = 4
# keys of an IP-Adapter Plus (Resampler) image projection; in a file that also has the base projection they are refused
_PLUS_MARKS = [("image_proj.latents", "an IP-Adapter Plus (Resampler) file"), ("image_proj.layers.", "an IP-Adapter Plus (Resampler) file"),
               ("image_proj.proj_in", "an IP-Adapter Plus (Resampler) file")]
# IP-Adapter variants this loader does not implement, recognised by a key substring
_FACEID = [("image_proj.proj.0.", "an IP-Adapter FaceID file"), ("perceiver_resampler", "an IP-Adapter FaceID Plus file"),
           ("lora", "an IP-Adapter FaceID file (LoRA layers)")]
# Resampler options h94's SDXL Plus files do not use and the engine does not implement
_PLUS_UNSUPPORTED = [("pos_emb", "a positional embedding of the image features"),
                     ("to_latents_from_mean_pooled_seq", "latents from the mean-pooled image features")]


@dataclass(frozen=True)
class ResamplerConfig:
    """The perceiver Resampler of IP-Adapter Plus (h94 resampler.py, diffusers IPAdapterPlusImageProjection): `depth` layers of
    `heads` heads of width 64 (the width is 64 * heads), `tokens` learned latent queries, feed-forward width 4 * width."""
    depth: int
    heads: int
    tokens: int = 16

    @property
    def width(self) -> int:
        return 64 * self.heads


# h94 `ip-adapter-plus_sdxl_vit-h` and `ip-adapter-plus-face_sdxl_vit-h` (image features: ViT-H/14 hidden_states[-2], D = 1280)
SDXL_PLUS = ResamplerConfig(depth=4, heads=20, tokens=16)


def resampler_specs(context_dim: int, image_embed_dim: int, r: ResamplerConfig) -> List[Tuple[str, Tuple[int, ...]]]:
    """Pack names and shapes of a Resampler's tensors (Linear weights [in, out])."""
    W = r.width
    specs = [("image_proj/latents", (r.tokens, W)), ("image_proj/proj_in/weight", (image_embed_dim, W)), ("image_proj/proj_in/bias", (W,))]
    for i in range(r.depth):
        p = f"image_proj/layers/{i}"
        for n in ("attn/norm1", "attn/norm2"):
            specs += [(f"{p}/{n}/weight", (W,)), (f"{p}/{n}/bias", (W,))]
        specs += [(f"{p}/attn/to_q/weight", (W, W)), (f"{p}/attn/to_kv/weight", (W, 2 * W)), (f"{p}/attn/to_out/weight", (W, W)),
                  (f"{p}/ff/norm/weight", (W,)), (f"{p}/ff/norm/bias", (W,)), (f"{p}/ff/fc1/weight", (W, 4 * W)),
                  (f"{p}/ff/fc2/weight", (4 * W, W))]
    return specs + [("image_proj/proj_out/weight", (W, context_dim)), ("image_proj/proj_out/bias", (context_dim,)),
                    ("image_proj/norm_out/weight", (context_dim,)), ("image_proj/norm_out/bias", (context_dim,))]


def resampler_of(weights: Dict[str, torch.Tensor]) -> Optional[ResamplerConfig]:
    """The ResamplerConfig of pack-named adapter weights, or None for a base adapter."""
    lat = weights.get("image_proj/latents")
    if lat is None:
        return None
    depth = len({k.split("/")[2] for k in weights if k.startswith("image_proj/layers/")})
    return ResamplerConfig(depth=depth, heads=int(lat.shape[1]) // 64, tokens=int(lat.shape[0]))


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


def ip_tensor_specs(cfg: UNetConfig, image_embed_dim: int, tokens: int = TOKENS_PER_IMAGE,
                    resampler: Optional[ResamplerConfig] = None) -> List[Tuple[str, Tuple[int, ...]]]:
    """Pack names and shapes of an adapter for `cfg` (Linear weights [in, out]); with `resampler` an IP-Adapter Plus (`tokens` is
    then resampler.tokens)."""
    ctx = cfg.context_dim
    if resampler is not None:
        specs = resampler_specs(ctx, image_embed_dim, resampler)
    else:
        specs = [("image_proj/proj/weight", (image_embed_dim, tokens * ctx)), ("image_proj/proj/bias", (tokens * ctx,)),
                 ("image_proj/norm/weight", (ctx,)), ("image_proj/norm/bias", (ctx,))]
    ins, mid, outs = block_program(cfg)
    widths = {b.path: b.c_out for b in ins + [mid] + outs}
    for p in transformer_block_paths(cfg):
        c = widths[p.split("/transformer/")[0]]
        specs += [(f"{p}/attn2/ip_key/weight", (ctx, c)), (f"{p}/attn2/ip_value/weight", (ctx, c))]
    return specs


def synth_ip_adapter(cfg: UNetConfig, image_embed_dim: int, seed: int = 0, resampler: Optional[ResamplerConfig] = None) -> Dict[str, torch.Tensor]:
    """Deterministic synthetic f16 adapter weights (pack names) for tests and benchmarks; with `resampler` an IP-Adapter Plus."""
    gen = torch.Generator().manual_seed(seed)
    out = {}
    for name, shape in ip_tensor_specs(cfg, image_embed_dim, resampler=resampler):
        if name.endswith("/weight") and name.split("/")[-2].startswith("norm"):   # LayerNorm gains
            t = 1.0 + 0.05 * torch.randn(shape, generator=gen)
        elif name.endswith("bias"):
            t = 0.05 * torch.randn(shape, generator=gen)
        elif name.endswith("latents"):   # h94's initialisation
            t = torch.randn(shape, generator=gen) / shape[1] ** 0.5
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


def _ip_layers(sd: Dict[str, torch.Tensor], cfg: UNetConfig, out: Dict[str, torch.Tensor]) -> None:
    """Maps the `ip_adapter.<i>.to_{k,v}_ip.weight` keys into `out`; any other key outside image_proj is rejected by name."""
    index = ip_index_map(cfg)
    pat = re.compile(r"^ip_adapter\.(\d+)\.to_([kv])_ip\.weight$")
    for k, t in sd.items():
        if k.startswith("image_proj."):
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


def _plus_key_map(depth: int) -> Dict[str, Tuple[str, bool]]:
    """h94 Resampler key -> (pack name, transpose). h94 layer i is ModuleList([PerceiverAttention, FeedForward]) and FeedForward is
    Sequential(LayerNorm, Linear, GELU, Linear), hence `.0.` / `.1.{0,1,3}`."""
    m = {"image_proj.latents": ("image_proj/latents", False)}
    for n in ("proj_in", "proj_out"):
        m[f"image_proj.{n}.weight"] = (f"image_proj/{n}/weight", True)
        m[f"image_proj.{n}.bias"] = (f"image_proj/{n}/bias", False)
    m["image_proj.norm_out.weight"] = ("image_proj/norm_out/weight", False)
    m["image_proj.norm_out.bias"] = ("image_proj/norm_out/bias", False)
    for i in range(depth):
        s, d = f"image_proj.layers.{i}", f"image_proj/layers/{i}"
        for n in ("norm1", "norm2"):
            m[f"{s}.0.{n}.weight"] = (f"{d}/attn/{n}/weight", False)
            m[f"{s}.0.{n}.bias"] = (f"{d}/attn/{n}/bias", False)
        for n in ("to_q", "to_kv", "to_out"):
            m[f"{s}.0.{n}.weight"] = (f"{d}/attn/{n}/weight", True)
        m[f"{s}.1.0.weight"] = (f"{d}/ff/norm/weight", False)
        m[f"{s}.1.0.bias"] = (f"{d}/ff/norm/bias", False)
        m[f"{s}.1.1.weight"] = (f"{d}/ff/fc1/weight", True)
        m[f"{s}.1.3.weight"] = (f"{d}/ff/fc2/weight", True)
    return m


def _from_h94_plus(sd: Dict[str, torch.Tensor], cfg: UNetConfig) -> Tuple[int, Dict[str, torch.Tensor]]:
    for k in sd:
        for pat, what in _PLUS_UNSUPPORTED:
            if pat in k:
                raise SdxlError(f"IP-Adapter Plus: key '{k}' marks a Resampler with {what}, which is not supported")
    ctx = cfg.context_dim
    lat = sd["image_proj.latents"]
    if lat.dim() == 3 and lat.shape[0] == 1:
        lat = lat[0]
    if lat.dim() != 2 or lat.shape[1] % 64 or not 1 <= lat.shape[0] <= 64:
        raise SdxlError(f"IP-Adapter Plus: 'image_proj.latents' has shape {tuple(sd['image_proj.latents'].shape)}, not [1, Q, 64 * heads] "
                        "with Q <= 64")
    layers = {int(k.split(".")[2]) for k in sd if re.match(r"^image_proj\.layers\.\d+\.", k)}
    depth = max(layers) + 1 if layers else 0
    if depth == 0:
        raise SdxlError("IP-Adapter Plus: key 'image_proj.layers.0.0.to_q.weight' is missing")
    q = sd.get("image_proj.layers.0.0.to_q.weight")
    if q is None:
        raise SdxlError("IP-Adapter Plus: key 'image_proj.layers.0.0.to_q.weight' is missing")
    r = ResamplerConfig(depth=depth, heads=int(q.shape[0]) // 64, tokens=int(lat.shape[0]))
    if q.dim() != 2 or q.shape[0] != lat.shape[1]:
        raise SdxlError(f"IP-Adapter Plus: 'image_proj.layers.0.0.to_q.weight' has shape {tuple(q.shape)}: the engine needs an "
                        f"attention width (64 * heads) equal to the latent width {lat.shape[1]}")
    w_in = sd.get("image_proj.proj_in.weight")
    if w_in is None:
        raise SdxlError("IP-Adapter Plus: key 'image_proj.proj_in.weight' is missing")
    D = int(w_in.shape[1])
    w_out = sd.get("image_proj.proj_out.weight")
    if w_out is not None and w_out.shape[0] != ctx:
        raise SdxlError(f"IP-Adapter Plus: 'image_proj.proj_out.weight' has {w_out.shape[0]} output features; this UNet's context_dim "
                        f"is {ctx}")
    keymap = _plus_key_map(depth)
    out = {}
    for k, t in sd.items():
        if not k.startswith("image_proj."):
            continue
        if k not in keymap:
            raise SdxlError(f"IP-Adapter Plus: unexpected key '{k}'")
        name, tr = keymap[k]
        out[name] = (lat if k == "image_proj.latents" else (t.t() if tr else t)).contiguous()
    missing = [k for k, (n, _) in keymap.items() if n not in out]
    if missing:
        raise SdxlError(f"IP-Adapter Plus: key '{missing[0]}' is missing ({len(missing)} missing)")
    src = {n: k for k, (n, _) in keymap.items()}
    for name, shape in resampler_specs(ctx, D, r):
        if tuple(out[name].shape) != shape:
            raise SdxlError(f"IP-Adapter Plus: key '{src[name]}' has shape {tuple(sd[src[name]].shape)}; a Resampler of width "
                            f"{r.width}, depth {depth}, {r.tokens} tokens and input width {D} needs {shape} ([in, out] here)")
    _ip_layers(sd, cfg, out)
    return D, {k: v.to(torch.float16) for k, v in out.items()}


def from_h94(state_dict: Dict, cfg: UNetConfig) -> Tuple[int, Dict[str, torch.Tensor]]:
    """(image_embed_dim, pack-named f16 tensors) of an h94 IP-Adapter state dict (flat or nested): the base IP-Adapter with 4
    tokens per image, or IP-Adapter Plus (recognised by `image_proj.latents` without `image_proj.proj.weight`; image_embed_dim is
    then the width of the image features, and resampler_of(weights) describes the Resampler). Anything else is rejected by name."""
    sd = _flatten(state_dict)
    plus = "image_proj.latents" in sd and "image_proj.proj.weight" not in sd
    for k in sd:
        for pat, what in _FACEID:
            if pat in k:
                raise SdxlError(f"IP-Adapter: key '{k}' marks {what}; only the base IP-Adapter and IP-Adapter Plus are supported")
        for pat, what in ([] if plus else _PLUS_MARKS):
            if pat in k:
                raise SdxlError(f"IP-Adapter: key '{k}' marks {what}, but the file is not one: a Plus file has 'image_proj.latents' "
                                "and no 'image_proj.proj.weight'")
    if cfg.is_refiner:
        raise SdxlError("IP-Adapter: the refiner is not supported")
    if plus:
        return _from_h94_plus(sd, cfg)
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
    for k in sd:
        if k.startswith("image_proj.") and k not in ("image_proj.proj.weight", "image_proj.proj.bias", "image_proj.norm.weight",
                                                     "image_proj.norm.bias"):
            raise SdxlError(f"IP-Adapter: unexpected key '{k}'")
    _ip_layers(sd, cfg, out)
    return int(w.shape[1]), {k: v.to(torch.float16) for k, v in out.items()}


def read_h94(path: str) -> Dict:
    """An h94 IP-Adapter file: `.safetensors` (flat keys) or `.bin` (torch.load(weights_only=True), flat or nested)."""
    if path.endswith(".safetensors"):
        return read_safetensors(path)
    return torch.load(path, map_location="cpu", weights_only=True)


def cfg_struct(cfg: UNetConfig, image_embed_dim: int, resampler: Optional[ResamplerConfig] = None) -> _lib.IpAdapterCfg:
    s = _lib.IpAdapterCfg()
    s.unet = _cfg_struct(cfg)
    s.image_embed_dim = image_embed_dim
    s.tokens_per_image = TOKENS_PER_IMAGE if resampler is None else resampler.tokens
    if resampler is not None:
        s.resampler_depth, s.resampler_heads = resampler.depth, resampler.heads
    return s


class IPAdapter(AttachableModel):
    """A device-resident IP-Adapter (sdxl_ip_adapter_load). weights: pack-named tensor dict or a built pack. The kind is read from
    the weights: `image_proj/latents` makes an IP-Adapter Plus (resampler_of); a built pack is a base adapter unless `resampler`
    describes it. image_embed_dim: D of the image embeddings (base) or of the image features (Plus)."""
    _load_fn, _destroy_fn, _detach_call = "sdxl_ip_adapter_load", "sdxl_ip_adapter_destroy", "set_image_prompt(None)"

    resampler: Optional[ResamplerConfig] = None   # None: the base adapter

    def __init__(self, ctx, cfg: UNetConfig, image_embed_dim: int, weights, resampler: Optional[ResamplerConfig] = None):
        self.cfg, self.image_embed_dim = cfg, int(image_embed_dim)
        self.resampler = resampler if isinstance(weights, torch.Tensor) else resampler_of(weights)
        self._load(ctx, cfg_struct(cfg, self.image_embed_dim, self.resampler), weights)

    @classmethod
    def from_file(cls, ctx, path: str, cfg: UNetConfig) -> "IPAdapter":
        """An h94 file, e.g. `sdxl_models/ip-adapter_sdxl_vit-h.safetensors` or `ip-adapter_sdxl.bin`."""
        dim, w = from_h94(read_h94(path), cfg)
        return cls(ctx, cfg, dim, w)

    @property
    def tokens_per_image(self) -> int:
        return TOKENS_PER_IMAGE if self.resampler is None else self.resampler.tokens

    def image_embeds(self, encoder, rgb: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """(embeds, negative) of u8 images [n, H, W, 3] for set_image_prompt, as diffusers / h94 compute them. Base: image_embeds
        [n, D] and zeros. Plus: hidden_states[-2] [n, T, D] of the images and of an all-zero pixel tensor (the preprocessed, i.e.
        already normalised, pixels set to zero)."""
        if self.resampler is None:
            e = encoder.encode_images(rgb)
            return e, torch.zeros_like(e)
        from .clip_vision import clip_preprocess
        px = clip_preprocess(rgb, encoder.cfg.image_size)
        return encoder.encode_hidden(px), encoder.encode_hidden(torch.zeros_like(px))

    def resample(self, hidden: torch.Tensor) -> torch.Tensor:
        """Plus: image tokens f16 [n * Q, context_dim] of image features f32 [n, L, D] (test aid)."""
        ctx = self.ctx
        h = self.handle()
        x = torch.as_tensor(hidden)
        if self.resampler is None or x.dim() != 3 or x.shape[2] != self.image_embed_dim:
            raise SdxlError(f"resample: needs an IP-Adapter Plus and features [n, L, {self.image_embed_dim}], got {tuple(x.shape)}")
        x = x.to(ctx.device, torch.float32).contiguous()
        out = torch.empty(x.shape[0] * self.resampler.tokens, self.cfg.context_dim, device=ctx.device, dtype=torch.float16)
        ctx.call("sdxl_ip_adapter_resample", ctx.lib.sdxl_ip_adapter_resample, h, x.shape[0], x.shape[1], x.data_ptr(), 0, out.data_ptr())
        return out

    def project(self, embeds: torch.Tensor) -> torch.Tensor:
        """Image tokens f16 [n * 4, context_dim] of embeddings f32 [n, D] (test aid)."""
        ctx = self.ctx
        h = self.handle()
        e = _embeds(embeds, self.image_embed_dim).reshape(-1, self.image_embed_dim).to(ctx.device).contiguous()
        out = torch.empty(e.shape[0] * TOKENS_PER_IMAGE, self.cfg.context_dim, device=ctx.device, dtype=torch.float16)
        ctx.call("sdxl_ip_adapter_project", ctx.lib.sdxl_ip_adapter_project, h, e.shape[0], e.data_ptr(), 0, out.data_ptr())
        return out


def _embeds(e: torch.Tensor, dim: int) -> torch.Tensor:
    """Image embeddings as [n_batch, n_images, D] f32; [n_batch, D] is one image per prompt. The engine reads
    n_batch * n_images * D floats, so any other shape is refused here."""
    e = torch.as_tensor(e)
    if e.dim() == 2:
        e = e.unsqueeze(1)
    if e.dim() != 3 or e.shape[2] != dim or e.shape[0] < 1 or e.shape[1] < 1:
        raise SdxlError(f"image embeddings must be [n_batch, D] or [n_batch, n_images, D] with D = {dim}, got {tuple(e.shape)}")
    return e.to(torch.float32)


def _features(x: torch.Tensor, dim: int, what: str) -> torch.Tensor:
    """IP-Adapter Plus image features as [n_batch, n_images, L, D] f32; [n_batch, L, D] is one image per prompt. The engine reads
    n_batch * n_images * L * D floats, so any other shape is refused here."""
    x = torch.as_tensor(x)
    if x.dim() == 3:
        x = x.unsqueeze(1)
    if x.dim() != 4 or x.shape[3] != dim or min(x.shape[:3]) < 1:
        raise SdxlError(f"IP-Adapter Plus {what} must be [n_batch, L, D] or [n_batch, n_images, L, D] with D = {dim} (vision encoder "
                        f"hidden states), got {tuple(x.shape)}")
    return x.to(torch.float32)


MAX_IMAGE_PROMPTS = 4   # SDXL_MAX_IMAGE_PROMPTS
MAX_IP_SOURCES = 8      # SDXL_MAX_IP_SOURCES: one per unmasked prompt, one per image of a masked prompt


def _prompt_struct(diffuser, adapter: IPAdapter, embeds, scale, negative) -> Tuple[_lib.ImagePrompt, list]:
    """The sdxl_image_prompt of one prompt and the objects its pointers borrow; every shape is checked here."""
    ctx = diffuser.ctx
    h = adapter.handle()
    plus = getattr(adapter, "resampler", None) is not None
    if plus:
        e = _features(embeds, adapter.image_embed_dim, "image features")
        if negative is None:
            raise SdxlError("IP-Adapter Plus: negative image features are required (IPAdapter.image_embeds computes them from an "
                            "all-zero image)")
    else:
        e = _embeds(embeds, adapter.image_embed_dim)
    neg = None
    if negative is not None:
        neg = _features(negative, adapter.image_embed_dim, "negative image features") if plus else _embeds(negative, adapter.image_embed_dim)
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
    p.seq_len = e.shape[2] if plus else 0
    p.block_scales_host = C.cast(block, C.c_void_p) if block is not None else None
    return p, [e, neg, block]


def _mask(mask, n_images: int) -> torch.Tensor:
    """A prompt's regional mask as f32 [n_images, H, W] of 0 / 1: bool, u8 or float, binarised at 0.5 as diffusers'
    IPAdapterMaskProcessor does. The engine reads n_images * H * W values of a multiple-of-8 extent, so anything else is refused here."""
    m = torch.as_tensor(mask)
    if m.dim() != 3 or m.shape[0] != n_images or m.shape[1] < 8 or m.shape[2] < 8 or m.shape[1] % 8 or m.shape[2] % 8:
        raise SdxlError(f"image-prompt mask must be [n_images = {n_images}, H, W] with H and W positive multiples of 8, got {tuple(m.shape)}")
    if m.dtype == torch.uint8:
        m = m.float() / 255.0
    m = m.float()
    if not bool(torch.isfinite(m).all()):
        raise SdxlError("image-prompt mask has non-finite values")
    return (m >= 0.5).float().contiguous()


def set_image_prompt(diffuser, adapter: Optional[IPAdapter], embeds: Optional[torch.Tensor] = None,
                     scale: Union[float, Sequence[float]] = 1.0, negative: Optional[torch.Tensor] = None) -> None:
    """sdxl_unet_set_image_prompt; adapter None detaches. scale: one float, or one per UNet transformer block in execution order
    (transformer_block_paths). negative: embeddings of the unconditional CFG rows (default: zeros). For an IP-Adapter Plus, embeds
    and negative are image features [n_batch, n_images, L, D] (IPAdapter.image_embeds) and negative is required."""
    ctx = diffuser.ctx
    p, _keep = (None, None) if adapter is None else _prompt_struct(diffuser, adapter, embeds, scale, negative)
    ctx.call("sdxl_unet_set_image_prompt", ctx.lib.sdxl_unet_set_image_prompt, diffuser.h, None if p is None else C.byref(p))
    diffuser._attach("image_prompts", [] if adapter is None else [adapter])


def set_image_prompts(diffuser, prompts: Sequence) -> None:
    """sdxl_unet_set_image_prompts: replaces the attached image prompts with [(adapter, embeds, scale, negative, mask), ...] (DESIGN.md
    §13); [] detaches. Each of the first four items is as for set_image_prompt. mask: None, or [n_images, H, W] (bool, u8 or float,
    binarised at 0.5) limiting each image of the prompt to its region of an (H / 8) x (W / 8) latent. At most MAX_IMAGE_PROMPTS
    prompts and MAX_IP_SOURCES sources (one per unmasked prompt, one per image of a masked prompt)."""
    ctx = diffuser.ctx
    prompts = list(prompts)
    if len(prompts) > MAX_IMAGE_PROMPTS:
        raise SdxlError(f"set_image_prompts: {len(prompts)} prompts given, at most {MAX_IMAGE_PROMPTS}")
    structs, masks, keep = [], [], []
    n_src = 0
    for item in prompts:
        if len(item) != 5:
            raise SdxlError("set_image_prompts: each prompt is (adapter, embeds, scale, negative, mask)")
        adapter, embeds, scale, negative, mask = item
        p, k = _prompt_struct(diffuser, adapter, embeds, scale, negative)
        m = _lib.IpMask()
        if mask is not None:
            mt = _mask(mask, p.n_images).to(ctx.device)
            m.mask, m.on_host, m.height, m.width = mt.data_ptr(), 0, mt.shape[1], mt.shape[2]
            k.append(mt)
        n_src += p.n_images if mask is not None else 1
        structs.append(p)
        masks.append(m)
        keep.append(k)
    if n_src > MAX_IP_SOURCES:
        raise SdxlError(f"set_image_prompts: {n_src} image sources (one per unmasked prompt, one per image of a masked prompt), at "
                        f"most {MAX_IP_SOURCES}")
    n = len(structs)
    arr = (_lib.ImagePrompt * max(n, 1))(*structs)
    marr = (_lib.IpMask * max(n, 1))(*masks)
    ctx.call("sdxl_unet_set_image_prompts", ctx.lib.sdxl_unet_set_image_prompts, diffuser.h, n, arr, marr)
    diffuser._attach("image_prompts", [item[0] for item in prompts])
