"""Synthetic LoRA adapters and a `.safetensors` writer shared by the LoRA tests."""
import json
import struct
from typing import Dict, Iterable, List, Optional

import numpy as np
import torch

from sdxl_b200 import clip_tensor_specs, unet_tensor_specs
from sdxl_b200.lora import clip_lora_modules, unet_lora_modules

_ST_NAMES = {torch.float16: "F16", torch.float32: "F32", torch.bfloat16: "BF16"}


def write_safetensors(path, tensors: Dict[str, torch.Tensor], metadata: Optional[Dict[str, str]] = None) -> None:
    header, blobs, off = {}, [], 0
    if metadata:
        header["__metadata__"] = metadata
    for name, t in tensors.items():
        raw = t.contiguous().reshape(-1).view(torch.uint8).numpy().tobytes() if t.numel() else b""
        header[name] = {"dtype": _ST_NAMES[t.dtype], "shape": list(t.shape), "data_offsets": [off, off + len(raw)]}
        blobs.append(raw)
        off += len(raw)
    h = json.dumps(header).encode()
    h += b" " * (-len(h) % 8)
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(h)) + h + b"".join(blobs))


def weight_shapes(cfg, clip: bool = False) -> Dict[str, tuple]:
    specs = clip_tensor_specs(cfg) if clip else unet_tensor_specs(cfg)
    return {n[: -len("/weight")]: s for n, s, _, _ in specs if n.endswith("/weight") and len(s) >= 2}


def layer_paths(cfg, clip: bool = False) -> List[str]:
    mods = clip_lora_modules(cfg, "lora_te1") if clip else unet_lora_modules(cfg)
    return [r for _, r, _ in mods]


def make_adapter(cfg, paths: Iterable[str], rank: int, seed: int, dyadic: bool = True, clip: bool = False,
                 alpha: Optional[float] = None, zero_up: bool = False) -> Dict[str, torch.Tensor]:
    """Factors for `paths`. dyadic: entries in {-1, 0, 1} / 16, so every f32 product and sum of the merge is exact (with an
    alpha / r and scale that are powers of two the merged weights are order-free); otherwise N(0, 0.02^2)."""
    shapes = weight_shapes(cfg, clip)
    g = torch.Generator().manual_seed(seed)
    out = {}
    for p in paths:
        s = shapes[p]
        if len(s) == 2:
            dshape, ushape = (rank, s[0]), (s[1], rank)
        else:
            dshape, ushape = (rank,) + tuple(s[1:]), (s[0], rank, 1, 1)
        if dyadic:
            down = torch.randint(-1, 2, dshape, generator=g).float() / 16
            up = torch.randint(-1, 2, ushape, generator=g).float() / 16
        else:
            down = torch.randn(dshape, generator=g) * 0.02
            up = torch.randn(ushape, generator=g) * 0.02
        if zero_up:
            up = torch.zeros_like(up)
        out[f"{p}/lora_down"] = down.half()
        out[f"{p}/lora_up"] = up.half()
        if alpha is not None:
            out[f"{p}/alpha"] = torch.tensor(float(alpha), dtype=torch.float32)
    return out


def to_kohya(adapter: Dict[str, torch.Tensor], modules) -> Dict[str, torch.Tensor]:
    by_ref = {r: k for k, r, _ in modules}
    leaf = {"lora_down": "lora_down.weight", "lora_up": "lora_up.weight", "alpha": "alpha"}
    out = {}
    for name, t in adapter.items():
        path, l = name.rsplit("/", 1)
        out[f"{by_ref[path]}.{leaf[l]}"] = t
    return out


def numpy_merge(w: np.ndarray, down: np.ndarray, up: np.ndarray, scale: float, alpha: float) -> np.ndarray:
    """The merge formula written directly: f16(f32(W) + scale * alpha / r * (up @ down)), Linear delta transposed to [in, out]."""
    r = down.shape[0]
    d = (np.float32(scale * alpha / r) * (up.reshape(up.shape[0], r).astype(np.float32) @ down.reshape(r, -1).astype(np.float32)))
    d = d.reshape((up.shape[0],) + down.shape[1:])
    if w.ndim == 2:
        d = d.T
    return np.where(d == 0, w, (w.astype(np.float32) + d).astype(np.float16))
