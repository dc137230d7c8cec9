"""Synthetic adapters of every family (LoRA, LoHa, LoKr, full delta, DoRA) and writers for every naming scheme that
sdxl_b200.lora.load_adapter reads, shared by the adapter-format tests."""
import math
from typing import Dict, Iterable, Optional

import numpy as np
import torch

from sdxl_b200.lora import _hf_dotted, clip_lora_modules, diffusers_unet_modules, family_product, unet_lora_modules
from lora_cases import make_adapter, weight_shapes

FAMILIES = ("lora", "loha", "lokr", "full")
SCHEMES = ("kohya", "kohya_diffusers", "diffusers", "peft")


def logical(shape):
    """(N, I, taps, conv) of a reference weight shape (Linear [in, out], conv OIHW)."""
    if len(shape) == 2:
        return shape[1], shape[0], 1, False
    return shape[0], shape[1], shape[2] * shape[3], True


def _t(g, shape, denom, dyadic):
    if dyadic:
        return torch.randint(-1, 2, shape, generator=g).float() / denom
    return torch.randn(shape, generator=g) * (0.5 / denom)


def _split(n: int) -> int:
    """A divisor of n near sqrt(n) (the w1 side of a LoKr factorisation)."""
    best = 1
    for a in range(1, int(math.isqrt(n)) + 1):
        if n % a == 0:
            best = a
    return best


def make_family(cfg, paths: Iterable[str], family: str, seed: int, dyadic: bool = True, clip: bool = False, rank: int = 2,
                lokr_mode: Optional[int] = None, alpha: Optional[float] = None) -> Dict[str, torch.Tensor]:
    """Pack-named adapter of one family on `paths`. Dyadic entries ({-1, 0, 1} / 16; / 4 for LoKr's w1), no alpha and a
    power-of-two scale make every f32 product and sum of the merge exact (LoHa's factors are in {-1, 0, 1} / 4, so that the
    product of its two rank sums is as large as a LoRA delta). lokr_mode (0..3; None: path index % 4) picks which of
    w1, w2 are given as products: bit 0 w1, bit 1 w2."""
    if family == "lora":
        return make_adapter(cfg, paths, rank, seed, dyadic=dyadic, clip=clip, alpha=alpha)
    shapes = weight_shapes(cfg, clip)
    g = torch.Generator().manual_seed(seed)
    out = {}
    for idx, p in enumerate(paths):
        N, I, taps, conv = logical(shapes[p])
        ks = int(round(math.sqrt(taps)))
        if family == "loha":
            r2 = rank + 1
            out[f"{p}/hada_w1_a"] = _t(g, (N, rank), 4, dyadic)
            out[f"{p}/hada_w1_b"] = _t(g, (rank, I, ks, ks) if conv else (rank, I), 4, dyadic)
            out[f"{p}/hada_w2_a"] = _t(g, (N, r2), 4, dyadic)
            out[f"{p}/hada_w2_b"] = _t(g, (r2, I * taps), 4, dyadic)   # the flat form of a conv factor
        elif family == "lokr":
            mode = idx % 4 if lokr_mode is None else lokr_mode
            a, b = _split(N), _split(I)
            c, d = N // a, I // b
            if mode & 1:
                out[f"{p}/lokr_w1_a"] = _t(g, (a, rank), 4, dyadic)
                out[f"{p}/lokr_w1_b"] = _t(g, (rank, b), 4, dyadic)
            else:
                out[f"{p}/lokr_w1"] = _t(g, (a, b), 4, dyadic)
            if mode & 2:
                out[f"{p}/lokr_w2_a"] = _t(g, (c, rank), 16, dyadic)
                out[f"{p}/lokr_w2_b"] = _t(g, (rank, d, ks, ks) if conv else (rank, d), 16, dyadic)
            else:
                out[f"{p}/lokr_w2"] = _t(g, (c, d, ks, ks) if conv else (c, d), 16, dyadic)
        elif family == "full":
            out[f"{p}/diff"] = _t(g, (N, I, ks, ks) if conv else (N, I), 64, dyadic)
        else:
            raise ValueError(family)
        if alpha is not None:
            out[f"{p}/alpha"] = torch.tensor(float(alpha), dtype=torch.float32)
    return {k: (v if k.endswith("/alpha") else v.half()) for k, v in out.items()}


def add_dora(cfg, adapter: Dict[str, torch.Tensor], weights: Dict[str, torch.Tensor], axis: int, seed: int, clip: bool = False,
             scale: float = 1.0) -> Dict[str, torch.Tensor]:
    """adapter + a dora_scale per layer: the norm of W + c * P along `axis` (0: per output row, shape [N]; 1: per input channel,
    shape [1, I] or [1, I, 1, 1]) times a factor in [0.9, 1.1], so the merged weight stays near W."""
    shapes = weight_shapes(cfg, clip)
    g = torch.Generator().manual_seed(seed)
    out = dict(adapter)
    for p in sorted({k.rsplit("/", 1)[0] for k in adapter}):
        N, I, taps, conv = logical(shapes[p])
        w = weights[f"{p}/weight"].double().numpy()
        W = w.T if w.ndim == 2 else w.reshape(N, -1)
        al, r, P = family_product(adapter, p, N, I, taps, np.float64)
        V = W + al / r * P
        if axis == 0:
            n = np.sqrt((V * V).sum(1))
            shape = (N,)
        else:
            n = np.sqrt((V * V).reshape(N, I, taps).sum((0, 2)))
            shape = (1, I, 1, 1) if conv else (1, I)
        f = 0.9 + 0.2 * torch.rand(n.shape, generator=g, dtype=torch.float64).numpy()
        out[f"{p}/dora_scale"] = torch.from_numpy(n * f).float().reshape(shape)
    return out


_FILE_LEAF = {
    "kohya": {"lora_down": "lora_down.weight", "lora_up": "lora_up.weight"},
    "kohya_diffusers": {"lora_down": "lora_down.weight", "lora_up": "lora_up.weight"},
    "diffusers": {"lora_down": "lora.down.weight", "lora_up": "lora.up.weight"},
    "peft": {"lora_down": "lora_A.weight", "lora_up": "lora_B.weight", "dora_scale": "lora_magnitude_vector"},
}


def module_names(scheme: str, part: str, cfg) -> Dict[str, str]:
    """reference layer path -> module name of `part` ("unet", "te1", "te2") under `scheme`."""
    if part == "unet":
        if scheme == "kohya":
            return {r: k for k, r, _ in unet_lora_modules(cfg)}
        dm = diffusers_unet_modules(cfg)
        if scheme == "kohya_diffusers":
            return {r: "lora_unet_" + m.replace(".", "_") for m, r in dm.items()}
        return {r: "unet." + m for m, r in dm.items()}
    kp = "lora_te1" if part == "te1" else "lora_te2"
    mods = clip_lora_modules(cfg, kp)
    if scheme.startswith("kohya"):
        return {r: k for k, r, _ in mods}
    dp = "text_encoder." if part == "te1" else "text_encoder_2."
    return {r: dp + _hf_dotted(k[len(kp) + 1:]) for k, r, _ in mods}


def to_file(scheme: str, parts) -> Dict[str, torch.Tensor]:
    """File tensors of [(part, cfg, adapter), ...] under `scheme` (module separator '.' for dotted schemes)."""
    out = {}
    for part, cfg, adapter in parts:
        names = module_names(scheme, part, cfg)
        for k, t in adapter.items():
            path, leaf = k.rsplit("/", 1)
            out[f"{names[path]}.{_FILE_LEAF[scheme].get(leaf, leaf)}"] = t
    return out
