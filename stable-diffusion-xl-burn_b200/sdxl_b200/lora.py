"""LoRA adapters: `.safetensors` reader, kohya -> reference layer-name map and the host-side merge formula.

An adapter here is a mapping in the reference's npy-tree naming (include/sdxl_b200.h, "LoRA adapters"):
  <layer path>/lora_down  f16 [r, in] (Linear) or [r, I, kh, kw] (conv)
  <layer path>/lora_up    f16 [out, r] (Linear) or [O, r, 1, 1] (conv)
  <layer path>/alpha      optional scalar (f32); missing => alpha = r
`Diffuser.set_adapters` / `ClipTextEncoder.set_adapters` merge such adapters on the device; `merge_into` is the same formula
on host weights (tests, and baking an adapter into a pack).

kohya's SDXL files name modules by the SGM / HF module tree with dots replaced by underscores (`lora_unet_input_blocks_4_1_
transformer_blocks_0_attn1_to_q`, `lora_te1_text_model_encoder_layers_0_self_attn_q_proj`). Those names contain underscores of
their own, so they are never parsed: the map is built by enumerating every LoRA-able module of a config under both names
(the reference's dump scripts python/unet.py and python/clip.py give the correspondence).
"""
from __future__ import annotations

import json
import struct
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from .config import ClipConfig, UNetConfig, block_program

Adapter = Dict[str, torch.Tensor]

# ------------------------------------------------------------------------------------------------
# safetensors
# ------------------------------------------------------------------------------------------------
_ST_DTYPES = {"F16": torch.float16, "F32": torch.float32, "BF16": torch.bfloat16}


def read_safetensors(src: Union[str, bytes]) -> Dict[str, torch.Tensor]:
    """Reads a `.safetensors` file (path or bytes): u64 header length, JSON header {name: {dtype, shape, data_offsets}},
    then the data. F16 / F32 / BF16 tensors; anything else raises."""
    if isinstance(src, (bytes, bytearray)):
        buf = bytes(src)
    else:
        with open(src, "rb") as f:
            buf = f.read()
    if len(buf) < 8:
        raise ValueError("safetensors: file too small")
    (n,) = struct.unpack_from("<Q", buf, 0)
    if 8 + n > len(buf):
        raise ValueError("safetensors: truncated header")
    header = json.loads(buf[8:8 + n].decode("utf-8"))
    data = memoryview(buf)[8 + n:]
    out: Dict[str, torch.Tensor] = {}
    for name, info in header.items():
        if name == "__metadata__":
            continue
        dt = _ST_DTYPES.get(info.get("dtype"))
        if dt is None:
            raise ValueError(f"safetensors: tensor '{name}' has unsupported dtype {info.get('dtype')!r} (F16, F32, BF16 only)")
        shape = [int(d) for d in info["shape"]]
        b0, b1 = (int(v) for v in info["data_offsets"])
        count = int(np.prod(shape)) if shape else 1
        if not (0 <= b0 <= b1 <= len(data)) or b1 - b0 != count * torch.empty(0, dtype=dt).element_size():
            raise ValueError(f"safetensors: tensor '{name}' has bad data_offsets {info['data_offsets']}")
        t = torch.frombuffer(bytearray(data[b0:b1]), dtype=dt) if b1 > b0 else torch.empty(0, dtype=dt)
        out[name] = t.reshape(shape)
    return out


# ------------------------------------------------------------------------------------------------
# kohya name map
# ------------------------------------------------------------------------------------------------
Module = Tuple[str, str, str]   # (kohya module name, reference layer path, "linear" | "conv")


def _res_modules(sgm: str, ref: str, has_skip: bool) -> List[Module]:
    m = [(f"{sgm}.in_layers.2", f"{ref}/conv_in", "conv"), (f"{sgm}.emb_layers.1", f"{ref}/lin_embed", "linear"),
         (f"{sgm}.out_layers.3", f"{ref}/conv_out", "conv")]
    if has_skip:
        m.append((f"{sgm}.skip_connection", f"{ref}/skip_connection", "conv"))
    return m


def _st_modules(sgm: str, ref: str, depth: int) -> List[Module]:
    m = [(f"{sgm}.proj_in", f"{ref}/proj_in", "linear"), (f"{sgm}.proj_out", f"{ref}/proj_out", "linear")]
    for j in range(depth):
        s, r = f"{sgm}.transformer_blocks.{j}", f"{ref}/transformer_{j}"
        for a in ("attn1", "attn2"):
            m += [(f"{s}.{a}.to_q", f"{r}/{a}/query", "linear"), (f"{s}.{a}.to_k", f"{r}/{a}/key", "linear"),
                  (f"{s}.{a}.to_v", f"{r}/{a}/value", "linear"), (f"{s}.{a}.to_out.0", f"{r}/{a}/out", "linear")]
        m += [(f"{s}.ff.net.0.proj", f"{r}/mlp/geglu/proj", "linear"), (f"{s}.ff.net.2", f"{r}/mlp/lin", "linear")]
    return m


def unet_lora_modules(cfg: UNetConfig) -> List[Module]:
    """Every LoRA-able module of the UNet (all Linears and convs) as (kohya name, reference path, kind)."""
    sgm: List[Tuple[str, str, str]] = [("time_embed.0", "lin1_time_embed", "linear"), ("time_embed.2", "lin2_time_embed", "linear"),
                                       ("label_emb.0.0", "lin1_label_embed", "linear"), ("label_emb.0.2", "lin2_label_embed", "linear")]
    ins, mid, outs = block_program(cfg)
    for b in ins + outs:
        s = b.path.replace("/", ".")
        if b.kind == "conv":
            sgm.append((f"{s}.0", b.path, "conv"))
        elif b.kind == "downsample":
            sgm.append((f"{s}.0.op", b.path, "conv"))
        elif b.kind == "resnet":
            sgm += _res_modules(f"{s}.0", b.path, b.c_in != b.c_out)
        else:
            sgm += _res_modules(f"{s}.0", f"{b.path}/res", b.c_in != b.c_out)
            if "transformer" in b.kind:
                sgm += _st_modules(f"{s}.1", f"{b.path}/transformer", b.depth)
            if b.kind.endswith("upsample"):
                sgm.append((f"{s}.{2 if 'transformer' in b.kind else 1}.conv", f"{b.path}/upsample/conv", "conv"))
    sgm += _res_modules("middle_block.0", "middle_block/res1", False)
    sgm += _st_modules("middle_block.1", "middle_block/transformer", mid.depth)
    sgm += _res_modules("middle_block.2", "middle_block/res2", False)
    sgm.append(("out.2", "conv_out", "conv"))
    return [("lora_unet_" + k.replace(".", "_"), r, kind) for k, r, kind in sgm]


def clip_lora_modules(cfg: ClipConfig, prefix: str) -> List[Module]:
    """Every LoRA-able Linear of a text encoder under kohya's HF names; prefix 'lora_te1' (CLIP-L) or 'lora_te2' (bigG)."""
    m: List[Module] = []
    for i in range(cfg.n_layer):
        hf, ref = f"{prefix}_text_model_encoder_layers_{i}", f"blocks/{i}"
        for h, r in (("q_proj", "query"), ("k_proj", "key"), ("v_proj", "value"), ("out_proj", "out")):
            m.append((f"{hf}_self_attn_{h}", f"{ref}/attn/{r}", "linear"))
        m += [(f"{hf}_mlp_fc1", f"{ref}/mlp/fc1", "linear"), (f"{hf}_mlp_fc2", f"{ref}/mlp/fc2", "linear")]
    return m


_LEAVES = {"lora_down.weight": "lora_down", "lora_up.weight": "lora_up", "alpha": "alpha"}


def _unsupported(key: str) -> str:
    if any(t in key for t in ("hada_", "lokr_")):
        return f"'{key}': LyCORIS (LoHa / LoKr) tensors are not supported"
    if "dora_scale" in key:
        return f"'{key}': DoRA is not supported"
    if key.endswith((".diff", ".diff_b", ".bias")) or ".norm" in key:
        return f"'{key}': norm or bias differences are not supported"
    if key.startswith(("unet.", "text_encoder", "lora_unet_down_blocks", "lora_unet_up_blocks", "lora_unet_mid_block")) or ".lora.down" in key \
            or ".lora_A" in key or ".lora_B" in key:
        return f"'{key}': diffusers-style LoRA names are not supported (kohya SGM names expected)"
    return f"'{key}': not a kohya LoRA tensor of a known module"


def from_kohya(tensors: Dict[str, torch.Tensor], unet_cfg: Optional[UNetConfig] = None, te1_cfg: Optional[ClipConfig] = None,
               te2_cfg: Optional[ClipConfig] = None) -> Dict[str, Adapter]:
    """kohya LoRA tensors -> {"unet": adapter, "te1": adapter, "te2": adapter} in reference naming (factors f16, alpha f32).
    Every key must belong to a module of the given configs; all offending keys are named in one ValueError."""
    table: Dict[str, Tuple[str, str]] = {}
    for part, mods in (("unet", unet_lora_modules(unet_cfg) if unet_cfg else []),
                       ("te1", clip_lora_modules(te1_cfg, "lora_te1") if te1_cfg else []),
                       ("te2", clip_lora_modules(te2_cfg, "lora_te2") if te2_cfg else [])):
        for k, ref, _ in mods:
            table[k] = (part, ref)
    out: Dict[str, Adapter] = {"unet": {}, "te1": {}, "te2": {}}
    bad: List[str] = []
    for key, t in tensors.items():
        mod, _, leaf = key.partition(".")
        if leaf not in _LEAVES or mod not in table:
            bad.append(_unsupported(key))
            continue
        part, ref = table[mod]
        name = f"{ref}/{_LEAVES[leaf]}"
        out[part][name] = t.to(torch.float32).reshape(()) if leaf == "alpha" else t.to(torch.float16).contiguous()
    if bad:
        more = f" (and {len(bad) - 8} more)" if len(bad) > 8 else ""
        raise ValueError("unsupported LoRA tensors: " + "; ".join(bad[:8]) + more)
    return out


def load_kohya(src: Union[str, bytes, Dict[str, torch.Tensor]], unet_cfg: Optional[UNetConfig] = None,
               te1_cfg: Optional[ClipConfig] = None, te2_cfg: Optional[ClipConfig] = None) -> Dict[str, Adapter]:
    """from_kohya over a `.safetensors` path / bytes (or an already-read tensor dict)."""
    tensors = src if isinstance(src, dict) else read_safetensors(src)
    return from_kohya(tensors, unet_cfg, te1_cfg, te2_cfg)


# ------------------------------------------------------------------------------------------------
# host-side merge
# ------------------------------------------------------------------------------------------------
def layer_delta(adapter: Adapter, path: str, scale: float) -> np.ndarray:
    """(scale * alpha / r) * (up @ down) of one layer in f32, shaped [out, in(, kh, kw)] like the factors."""
    down = adapter[f"{path}/lora_down"].to(torch.float32).numpy()
    up = adapter[f"{path}/lora_up"].to(torch.float32).numpy()
    r = down.shape[0]
    a = adapter.get(f"{path}/alpha")
    alpha = float(a.to(torch.float32).reshape(-1)[0]) if a is not None else float(r)
    coef = np.float32(float(np.float32(scale)) * alpha / r)
    inner = up.reshape(up.shape[0], r) @ down.reshape(r, -1)
    return (coef * inner).reshape((up.shape[0],) + down.shape[1:])


def merge_into(weights: Dict[str, torch.Tensor], adapter: Adapter, scale: float = 1.0) -> Dict[str, torch.Tensor]:
    """Returns a copy of `weights` (reference layouts, f16) with W' = f16(f32(W) + scale * alpha / r * up @ down) for every layer
    of `adapter` (the Linear delta transposed to the [in, out] layout). A zero delta element leaves W's bits unchanged."""
    out = dict(weights)
    layers = sorted({k.rsplit("/", 1)[0] for k in adapter})
    for path in layers:
        key = f"{path}/weight"
        if key not in weights:
            raise KeyError(f"merge_into: the weights have no '{key}'")
        w = weights[key].to(torch.float32).numpy()
        d = layer_delta(adapter, path, scale)
        if w.ndim == 2:
            d = d.T
        if d.shape != w.shape:
            raise ValueError(f"merge_into: delta of '{path}' is {d.shape}, weight is {w.shape}")
        merged = torch.from_numpy((w + d).astype(np.float32)).to(torch.float16)
        out[key] = torch.where(torch.from_numpy(d == 0), weights[key], merged)
    return out
