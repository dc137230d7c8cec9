"""LoRA adapters: `.safetensors` reader, kohya -> reference layer-name map and the host-side merge formula.

An adapter here is a mapping in the reference's npy-tree naming (include/sdxl_b200.h, "LoRA adapters"):
  <layer path>/lora_down  f16 [r, in] (Linear) or [r, I, kh, kw] (conv)
  <layer path>/lora_up    f16 [out, r] (Linear) or [O, r, 1, 1] (conv)
  <layer path>/alpha      optional scalar (f32); missing => alpha = r
  <layer path>/hada_w1_a, hada_w1_b, hada_w2_a, hada_w2_b   LoHa factors (f16)
  <layer path>/lokr_w1 | lokr_w1_a + lokr_w1_b, lokr_w2 | lokr_w2_a + lokr_w2_b   LoKr factors (f16)
  <layer path>/diff       full delta (f16)
  <layer path>/dora_scale DoRA magnitude (f32)
(DESIGN.md §19 states each family's delta). `Diffuser.set_adapters` / `ClipTextEncoder.set_adapters` merge such adapters on the
device; `merge_into` is the same formula on host weights (tests, and baking an adapter into a pack).

kohya's SDXL files name modules by the SGM / HF module tree with dots replaced by underscores (`lora_unet_input_blocks_4_1_
transformer_blocks_0_attn1_to_q`, `lora_te1_text_model_encoder_layers_0_self_attn_q_proj`). Those names contain underscores of
their own, so they are never parsed: the map is built by enumerating every LoRA-able module of a config under both names
(the reference's dump scripts python/unet.py and python/clip.py give the correspondence). `load_adapter` also reads kohya names
of diffusers modules (`lora_unet_down_blocks_1_attentions_0_...`), diffusers / PEFT dotted names (`unet.down_blocks.1...lora_A.weight`,
`text_encoder.text_model.encoder.layers.0...`) and the LyCORIS LoHa, LoKr, full-delta and DoRA leaves.
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


# ------------------------------------------------------------------------------------------------
# every adapter format: kohya (SGM or diffusers module names), diffusers / PEFT dotted names, LoRA / LoHa / LoKr / full / DoRA
# ------------------------------------------------------------------------------------------------
# file leaf -> pack leaf. Longest first, so a dotted key's leaf is found by suffix.
_ADAPTER_LEAVES = {"lora_magnitude_vector.weight": "dora_scale", "lora_magnitude_vector": "dora_scale", "lora_down.weight": "lora_down",
                   "lora_up.weight": "lora_up", "lora.down.weight": "lora_down", "lora.up.weight": "lora_up", "lora_A.weight": "lora_down",
                   "lora_B.weight": "lora_up", "dora_scale": "dora_scale", "alpha": "alpha", "diff": "diff"}
_ADAPTER_LEAVES.update({k: k for k in ("hada_w1_a", "hada_w1_b", "hada_w2_a", "hada_w2_b", "lokr_w1", "lokr_w1_a", "lokr_w1_b", "lokr_w2",
                                       "lokr_w2_a", "lokr_w2_b")})
_F32_LEAVES = ("alpha", "dora_scale")


def diffusers_unet_modules(cfg: UNetConfig) -> Dict[str, str]:
    """diffusers UNet2DConditionModel module name (`down_blocks.1.attentions.0.transformer_blocks.0.attn1.to_q`) -> reference layer
    path, for every LoRA-able module (diffusers_unet.name_map, read backwards)."""
    from .diffusers_unet import name_map
    refs = {r for _, r, _ in unet_lora_modules(cfg)}
    out = {}
    for k, (dst, _) in name_map(cfg).items():
        if k.endswith(".weight") and dst[: -len("/weight")] in refs:
            out[k[: -len(".weight")]] = dst[: -len("/weight")]
    return out


def _hf_dotted(kohya_tail: str) -> str:
    # text_model_encoder_layers_3_self_attn_q_proj -> text_model.encoder.layers.3.self_attn.q_proj
    head = "text_model_encoder_layers_"
    i, rest = kohya_tail[len(head):].split("_", 1)
    return f"text_model.encoder.layers.{i}.{rest.replace('self_attn_', 'self_attn.').replace('mlp_', 'mlp.')}"


def adapter_module_table(unet_cfg: Optional[UNetConfig] = None, te1_cfg: Optional[ClipConfig] = None,
                         te2_cfg: Optional[ClipConfig] = None) -> Tuple[Dict[str, Tuple[str, str]], Dict[str, Tuple[str, str]]]:
    """(kohya module name -> (part, layer path), dotted module name -> (part, layer path)) under every naming scheme load_adapter reads:
    kohya SGM and kohya diffusers names (`lora_unet_...`, `lora_te1_...`, `lora_te2_...`), and diffusers / PEFT names under `unet.`,
    `text_encoder.` and `text_encoder_2.`."""
    under: Dict[str, Tuple[str, str]] = {}
    dotted: Dict[str, Tuple[str, str]] = {}
    if unet_cfg:
        for k, r, _ in unet_lora_modules(unet_cfg):
            under[k] = ("unet", r)
        for m, r in diffusers_unet_modules(unet_cfg).items():
            under["lora_unet_" + m.replace(".", "_")] = ("unet", r)
            dotted["unet." + m] = ("unet", r)
    for part, cfg, kp, dp in (("te1", te1_cfg, "lora_te1", "text_encoder."), ("te2", te2_cfg, "lora_te2", "text_encoder_2.")):
        if cfg:
            for k, r, _ in clip_lora_modules(cfg, kp):
                under[k] = (part, r)
                dotted[dp + _hf_dotted(k[len(kp) + 1:])] = (part, r)
    return under, dotted


def _adapter_refusal(key: str) -> str:
    leaf = key.rsplit(".", 1)[-1]
    if any(t in key for t in ("lora_mid", "hada_t1", "hada_t2", "lokr_t1", "lokr_t2")):
        return f"'{key}': Tucker-decomposed factors are not supported"
    if any(t in key for t in ("oft_", "boft_")) or leaf == "oft_blocks":
        return f"'{key}': OFT / BOFT tensors are not supported"
    if any(key.endswith(f".{g}.weight") for g in ("a1", "a2", "b1", "b2")):
        return f"'{key}': GLoRA tensors are not supported"
    if "ia3" in key or leaf == "on_input" or key.partition(".")[2] == "weight":
        return f"'{key}': IA3 tensors are not supported"
    if key.endswith((".diff_b", ".bias")) or (key.endswith(".diff") and "norm" in key):
        return f"'{key}': norm or bias differences are not supported"
    return f"'{key}': not an adapter tensor of a known module"


def from_adapter(tensors: Dict[str, torch.Tensor], unet_cfg: Optional[UNetConfig] = None, te1_cfg: Optional[ClipConfig] = None,
                 te2_cfg: Optional[ClipConfig] = None) -> Dict[str, Adapter]:
    """Adapter tensors under any naming scheme of adapter_module_table, with any leaf of DESIGN.md §19 -> {"unet", "te1", "te2"}
    adapters in reference naming (factors f16; alpha and dora_scale f32). All offending keys are named in one ValueError."""
    under, dotted = adapter_module_table(unet_cfg, te1_cfg, te2_cfg)
    out: Dict[str, Adapter] = {"unet": {}, "te1": {}, "te2": {}}
    bad: List[str] = []
    for key, t in tensors.items():
        hit = None
        mod, _, leaf = key.partition(".")
        if mod in under and leaf in _ADAPTER_LEAVES:
            hit = (under[mod], _ADAPTER_LEAVES[leaf])
        else:
            for fl in _ADAPTER_LEAVES:
                if key.endswith("." + fl) and key[: -len(fl) - 1] in dotted:
                    hit = (dotted[key[: -len(fl) - 1]], _ADAPTER_LEAVES[fl])
                    break
        if hit is None or (hit[1] == "diff" and "norm" in key):
            bad.append(_adapter_refusal(key))
            continue
        (part, ref), pl = hit
        name = f"{ref}/{pl}"
        if name in out[part]:
            bad.append(f"'{key}': a second tensor for '{name}'")
            continue
        if pl == "alpha":
            out[part][name] = t.to(torch.float32).reshape(())
        elif pl in _F32_LEAVES:
            out[part][name] = t.to(torch.float32).contiguous()
        else:
            out[part][name] = t.to(torch.float16).contiguous()
    if bad:
        more = f" (and {len(bad) - 8} more)" if len(bad) > 8 else ""
        raise ValueError("unsupported adapter tensors: " + "; ".join(bad[:8]) + more)
    return out


def load_adapter(src: Union[str, bytes, Dict[str, torch.Tensor]], unet_cfg: Optional[UNetConfig] = None,
                 te1_cfg: Optional[ClipConfig] = None, te2_cfg: Optional[ClipConfig] = None) -> Dict[str, Adapter]:
    """from_adapter over a `.safetensors` path / bytes (or an already-read tensor dict). On a kohya LoRA file it returns what
    load_kohya returns."""
    tensors = src if isinstance(src, dict) else read_safetensors(src)
    return from_adapter(tensors, unet_cfg, te1_cfg, te2_cfg)


def load_kohya(src: Union[str, bytes, Dict[str, torch.Tensor]], unet_cfg: Optional[UNetConfig] = None,
               te1_cfg: Optional[ClipConfig] = None, te2_cfg: Optional[ClipConfig] = None) -> Dict[str, Adapter]:
    """from_kohya over a `.safetensors` path / bytes (or an already-read tensor dict)."""
    tensors = src if isinstance(src, dict) else read_safetensors(src)
    return from_kohya(tensors, unet_cfg, te1_cfg, te2_cfg)


# ------------------------------------------------------------------------------------------------
# host-side merge
# ------------------------------------------------------------------------------------------------
def layer_delta(adapter: Adapter, path: str, scale: float) -> np.ndarray:
    """(scale * alpha / r) * (up @ down) of one LoRA layer in f32, shaped [out, in(, kh, kw)] like the factors."""
    down = adapter[f"{path}/lora_down"].to(torch.float32).numpy()
    up = adapter[f"{path}/lora_up"].to(torch.float32).numpy()
    r = down.shape[0]
    a = adapter.get(f"{path}/alpha")
    alpha = float(a.to(torch.float32).reshape(-1)[0]) if a is not None else float(r)
    coef = np.float32(float(np.float32(scale)) * alpha / r)
    inner = up.reshape(up.shape[0], r) @ down.reshape(r, -1)
    return (coef * inner).reshape((up.shape[0],) + down.shape[1:])


def family_product(adapter: Adapter, path: str, N: int, I: int, taps: int, dtype=np.float32) -> Tuple[float, float, np.ndarray]:
    """(alpha, r, P) of one layer of any family (DESIGN.md §19): P [N, I * taps] in `dtype` (f32: the device's arithmetic; f64: the
    exact statement) and the coefficient c = alpha / r (1 / 1 where the family takes no alpha). A missing alpha is r; a negative
    one is used as given."""
    def f(leaf):
        t = adapter.get(f"{path}/{leaf}")
        return None if t is None else t.to(torch.float64).numpy().astype(dtype)

    def alpha_r(r):
        a = adapter.get(f"{path}/alpha")
        return (float(a.to(torch.float32).reshape(-1)[0]) if a is not None else float(r)), float(r)

    if f"{path}/lora_down" in adapter:
        down, up = f("lora_down"), f("lora_up")
        r = down.shape[0]
        return (*alpha_r(r), up.reshape(N, r) @ down.reshape(r, -1))
    if f"{path}/hada_w1_a" in adapter:
        w1a, w1b, w2a, w2b = (f(x) for x in ("hada_w1_a", "hada_w1_b", "hada_w2_a", "hada_w2_b"))
        r = w1b.shape[0]
        return (*alpha_r(r), (w1a @ w1b.reshape(r, -1)) * (w2a @ w2b.reshape(w2b.shape[0], -1)))
    if any(k.startswith(f"{path}/lokr_") for k in adapter):
        rank = 0
        ws = []
        for w in ("lokr_w1", "lokr_w2"):
            full = f(w)
            if full is not None:
                ws.append(full.reshape(full.shape[0], -1))
            else:
                a, b = f(w + "_a"), f(w + "_b")
                rank = rank or a.shape[1]
                ws.append(a @ b.reshape(b.shape[0], -1))
        w1, w2 = ws
        a_, b_ = w1.shape
        c_ = w2.shape[0]
        d_ = w2.shape[1] // taps
        P = np.einsum("ip,jqt->ijpqt", w1, w2.reshape(c_, d_, taps)).reshape(a_ * c_, b_ * d_ * taps)
        return (*(alpha_r(rank) if rank else (1.0, 1.0)), P)
    return 1.0, 1.0, f("diff").reshape(N, -1)


def _as_rows(w: np.ndarray) -> np.ndarray:
    """A reference weight as the logical [N, I * taps] matrix (Linear [in, out] transposed; conv OIHW flattened)."""
    return w.T if w.ndim == 2 else w.reshape(w.shape[0], -1)


def merge_into(weights: Dict[str, torch.Tensor], adapter, scale: float = 1.0) -> Dict[str, torch.Tensor]:
    """Returns a copy of `weights` (reference layouts, f16) with every layer of the adapters merged as the device merges them
    (DESIGN.md §7, §19). `adapter` is one adapter (with `scale`) or a list of (adapter, scale), stacked in order. A layer without
    dora_scale gets W' = f16(f32(W) + sum of f32(s * c) * P in f32) (one LoRA: f16(f32(W) + scale * alpha / r * up @ down), the Linear
    delta transposed to the [in, out] layout). A layer with dora_scale is merged in float64: W' = f16(W + sum of the non-DoRA
    terms s * c * P + sum of the DoRA terms s * (m * V / n - W)), V = W + c * P, n the norm of V per row or input channel. A zero
    delta element leaves W's bits unchanged."""
    sets = [(adapter, scale)] if isinstance(adapter, dict) else list(adapter)
    out = dict(weights)
    layers = sorted({k.rsplit("/", 1)[0] for a, _ in sets for k in a})
    for path in layers:
        key = f"{path}/weight"
        if key not in weights:
            raise KeyError(f"merge_into: the weights have no '{key}'")
        w16 = weights[key]
        w = w16.to(torch.float32).numpy()
        here = [(a, s) for a, s in sets if any(k.rsplit("/", 1)[0] == path for k in a)]
        N = w.shape[1] if w.ndim == 2 else w.shape[0]
        I = w.shape[0] if w.ndim == 2 else w.shape[1]
        taps = 1 if w.ndim == 2 else w.shape[2] * w.shape[3]
        if not any(f"{path}/dora_scale" in a for a, _ in here):
            if len(here) == 1 and f"{path}/lora_down" in here[0][0]:   # the original LoRA formula
                d = layer_delta(here[0][0], path, here[0][1])
                d = d.T if w.ndim == 2 else d
            else:
                t = np.zeros((N, I * taps), np.float32)
                for a, s in here:
                    al, r, P = family_product(a, path, N, I, taps)
                    t = t + np.float32(float(np.float32(s)) * al / r) * P.astype(np.float32)
                d = t.T if w.ndim == 2 else t.reshape(w.shape)
            if d.shape != w.shape:
                raise ValueError(f"merge_into: delta of '{path}' is {d.shape}, weight is {w.shape}")
            merged = torch.from_numpy((w + d).astype(np.float32)).to(torch.float16)
            out[key] = torch.where(torch.from_numpy(d == 0), w16, merged)
            continue
        W = _as_rows(w.astype(np.float64))
        t = np.zeros_like(W)
        for a, s in sorted(here, key=lambda x: f"{path}/dora_scale" in x[0]):   # non-DoRA terms first (a stable sort)
            al, r, P = family_product(a, path, N, I, taps, np.float64)
            c = al / r
            ds = a.get(f"{path}/dora_scale")
            if ds is None:
                t += float(np.float32(s)) * c * P
                continue
            m = ds.to(torch.float64).numpy().reshape(-1)
            V = W + c * P
            if m.size == N and ds.shape[0] == N:
                n = np.sqrt((V * V).sum(1))[:, None]
                m = m[:, None]
            else:
                n = np.sqrt((V * V).reshape(N, I, taps).sum((0, 2))).repeat(taps)[None, :]
                m = m.repeat(taps)[None, :]
            with np.errstate(divide="ignore", invalid="ignore"):
                t += np.where(n == 0, 0.0, float(np.float32(s)) * (m * V / n - W))
        merged = _as_rows(w.astype(np.float64)) + t
        merged = merged.T if w.ndim == 2 else merged.reshape(w.shape)
        d = t.T if w.ndim == 2 else t.reshape(w.shape)
        out[key] = torch.where(torch.from_numpy(d == 0), w16, torch.from_numpy(merged).to(torch.float16))
    return out
