"""Reader / writer for the reference's shipped model files: burn 0.13 `NamedMpkFileRecorder<HalfPrecisionSettings>` records
(`<name>.mpk`, written by src/bin/convert/main.rs:65-70, read by src/bin/sample/main.rs:28-51) and their `<name>.cfg` JSON
(burn `Config::load`, sample/main.rs:29,36,47). With these a real `Gadersd/stable-diffusion-xl-burn` download drops in:

    cfg, weights = load_diffuser("SDXL/diffuser")          # -> UNetConfig, {dump-tree name: f16 tensor}
    Diffuser(ctx, cfg, weights)

Format (burn 0.13 / rmp-serde "named", restated from knowledge of those crates: neither is available offline, no sample file
exists in this environment, so the reader is validated against this module's own writer + the `msgpack` package, i.e. the
container and the field tree, not against a file written by burn itself):

  * file = MessagePack map {"metadata": {"float": "f16", "int": "i16", "format": ..., "version": "0.13.0", "settings": ...},
                            "item": <record>}
  * a Module struct is a map keyed by FIELD NAME (the Rust field names of src/model/**): Param<Tensor> fields are
    {"id": "<uuid>", "param": {"value": [...], "shape": [...]}}; `value` holds the f16 BIT PATTERNS as MessagePack unsigned
    integers (half::f16 serialises as a newtype over u16), row-major; constants (usize / f64 / bool / String fields) are nil —
    they are rebuilt from the .cfg; Vec<T> is an array; Option<T> is nil or T; an enum (UNetBlocks) is a one-entry map
    {"<Variant>": <record>}.
  * Linear weight is [d_input, d_output] and conv weight OIHW — the layouts of the npy dump tree (python/save.py) and of our pack.

The value arrays (2.6 G integers for the base UNet) are decoded by the native `sdxl_mpk_decode_u16`; everything else is a few
thousand small MessagePack objects walked here.
"""
from __future__ import annotations

import ctypes as C
import json
import mmap
import struct
import uuid
from typing import Any, Dict, List, Optional, Tuple

import numpy as np
import torch

from . import _lib
from .config import ClipConfig, UNetConfig, VaeConfig

Tree = Any


class BurnRecordError(ValueError):
    pass


# ---------------------------------------------------------------------------------------------------
# minimal MessagePack walker (maps / arrays / str / nil / bool / ints / floats) with a fast path for tensor value arrays
# ---------------------------------------------------------------------------------------------------
class _Reader:
    def __init__(self, buf):
        self.b = buf
        self.p = 0
        self.n = len(buf)
        self.lib = _lib.load()
        self.base = np.frombuffer(buf, dtype=np.uint8)

    def _need(self, k):
        if self.p + k > self.n:
            raise BurnRecordError("truncated record")

    def _u(self, fmt, k):
        self._need(k)
        v = struct.unpack_from(fmt, self.b, self.p)[0]
        self.p += k
        return v

    def _len(self, t, fix_lo, fix_mask, t16, t32):
        if fix_lo <= t <= fix_lo + fix_mask:
            return t - fix_lo
        if t == t16:
            return self._u(">H", 2)
        if t == t32:
            return self._u(">I", 4)
        return None

    def u16_array(self, count: int) -> np.ndarray:
        out = np.empty(count, dtype=np.uint16)
        used = C.c_size_t(0)
        src = self.base[self.p:]
        rc = self.lib.sdxl_mpk_decode_u16(src.ctypes.data, src.size, count, out.ctypes.data, C.byref(used))
        if rc != 0:
            raise BurnRecordError(f"tensor value array is not {count} unsigned 16-bit integers (code {rc})")
        self.p += used.value
        return out

    def value(self, key: Optional[str] = None) -> Tree:
        self._need(1)
        t = self.b[self.p]
        self.p += 1
        if t <= 0x7F:
            return t
        if t >= 0xE0:
            return t - 0x100
        if t == 0xC0:
            return None
        if t == 0xC2:
            return False
        if t == 0xC3:
            return True
        n = self._len(t, 0xA0, 0x1F, 0xDA, 0xDB)       # str (str8 below)
        if n is None and t == 0xD9:
            n = self._u(">B", 1)
        if n is not None:
            self._need(n)
            s = bytes(self.b[self.p:self.p + n]).decode("utf-8")
            self.p += n
            return s
        n = self._len(t, 0x90, 0x0F, 0xDC, 0xDD)       # array
        if n is not None:
            if key == "value":                          # tensor payload: f16 bit patterns
                return self.u16_array(n)
            return [self.value() for _ in range(n)]
        n = self._len(t, 0x80, 0x0F, 0xDE, 0xDF)       # map
        if n is not None:
            out = {}
            for _ in range(n):
                k = self.value()
                if not isinstance(k, str):
                    raise BurnRecordError("non-string map key")
                out[k] = self.value(k)
            return out
        fixed = {0xCC: (">B", 1), 0xCD: (">H", 2), 0xCE: (">I", 4), 0xCF: (">Q", 8), 0xD0: (">b", 1), 0xD1: (">h", 2), 0xD2: (">i", 4),
                 0xD3: (">q", 8), 0xCA: (">f", 4), 0xCB: (">d", 8)}
        if t in fixed:
            return self._u(*fixed[t])
        if t in (0xC4, 0xC5, 0xC6):                     # bin
            n = self._u({0xC4: ">B", 0xC5: ">H", 0xC6: ">I"}[t], {0xC4: 1, 0xC5: 2, 0xC6: 4}[t])
            self._need(n)
            v = bytes(self.b[self.p:self.p + n])
            self.p += n
            return v
        raise BurnRecordError(f"unsupported MessagePack type byte 0x{t:02x}")


def read_mpk(path: str) -> Tuple[dict, Tree]:
    """-> (metadata, item). Tensor leaves are {"id": str, "param": {"value": np.uint16[...], "shape": [...]}}."""
    with open(path, "rb") as fh:
        try:
            buf = mmap.mmap(fh.fileno(), 0, access=mmap.ACCESS_READ)
        except ValueError:
            buf = fh.read()
        top = _Reader(buf).value()
    if not isinstance(top, dict) or "item" not in top:
        raise BurnRecordError("not a burn record: top-level map with 'metadata' and 'item' expected")
    meta = top.get("metadata") or {}
    if meta.get("float") not in (None, "f16"):
        raise BurnRecordError(f"record float type is {meta.get('float')!r}: only HalfPrecisionSettings (f16) files are supported")
    return meta, top["item"]


# ---------------------------------------------------------------------------------------------------
# writer (fixtures, and the inverse of the reader: `convert`)
# ---------------------------------------------------------------------------------------------------
def _pack_len(n, fix_lo, fix_max, t16, t32) -> bytes:
    if n <= fix_max:
        return bytes([fix_lo + n])
    if n < 65536:
        return bytes([t16]) + struct.pack(">H", n)
    return bytes([t32]) + struct.pack(">I", n)


def _pack(obj, out: List[bytes]) -> None:
    lib = _lib.load()
    if obj is None:
        out.append(b"\xc0")
    elif obj is True:
        out.append(b"\xc3")
    elif obj is False:
        out.append(b"\xc2")
    elif isinstance(obj, int):
        if 0 <= obj < 128:
            out.append(bytes([obj]))
        elif 0 <= obj < 256:
            out.append(b"\xcc" + bytes([obj]))
        elif 0 <= obj < 65536:
            out.append(b"\xcd" + struct.pack(">H", obj))
        elif 0 <= obj < 2 ** 32:
            out.append(b"\xce" + struct.pack(">I", obj))
        elif obj >= 0:
            out.append(b"\xcf" + struct.pack(">Q", obj))
        else:
            out.append(b"\xd3" + struct.pack(">q", obj))
    elif isinstance(obj, float):
        out.append(b"\xcb" + struct.pack(">d", obj))
    elif isinstance(obj, str):
        b = obj.encode("utf-8")
        out.append((bytes([0xA0 + len(b)]) if len(b) < 32 else (b"\xd9" + bytes([len(b)]) if len(b) < 256 else b"\xda" + struct.pack(">H", len(b)))) + b)
    elif isinstance(obj, np.ndarray):                   # tensor payload
        a = np.ascontiguousarray(obj, dtype=np.uint16).reshape(-1)
        out.append(_pack_len(a.size, 0x90, 15, 0xDC, 0xDD))
        buf = np.empty(3 * a.size, dtype=np.uint8)
        n = lib.sdxl_mpk_encode_u16(a.ctypes.data, a.size, buf.ctypes.data)
        out.append(buf[:n].tobytes())
    elif isinstance(obj, (list, tuple)):
        out.append(_pack_len(len(obj), 0x90, 15, 0xDC, 0xDD))
        for v in obj:
            _pack(v, out)
    elif isinstance(obj, dict):
        out.append(_pack_len(len(obj), 0x80, 15, 0xDE, 0xDF))
        for k, v in obj.items():
            _pack(str(k), out)
            _pack(v, out)
    else:
        raise TypeError(type(obj))


def write_mpk(path: str, item: Tree) -> None:
    meta = {"float": "f16", "int": "i16", "format": "burn_core::record::file::NamedMpkFileRecorder<burn_core::record::settings::HalfPrecisionSettings>",
            "version": "0.13.0", "settings": "HalfPrecisionSettings"}
    out: List[bytes] = []
    _pack({"metadata": meta, "item": item}, out)
    with open(path, "wb") as fh:
        for b in out:
            fh.write(b)


# ---------------------------------------------------------------------------------------------------
# tensor leaves
# ---------------------------------------------------------------------------------------------------
def _tensor(leaf, where: str) -> torch.Tensor:
    if not isinstance(leaf, dict) or "param" not in leaf:
        raise BurnRecordError(f"{where}: expected a Param record {{id, param}}")
    d = leaf["param"]
    if not isinstance(d, dict) or "value" not in d or "shape" not in d:
        raise BurnRecordError(f"{where}: expected {{value, shape}}")
    shape = [int(x) for x in d["shape"]]
    v = d["value"]
    if int(np.prod(shape)) != v.size:
        raise BurnRecordError(f"{where}: {v.size} values for shape {shape}")
    return torch.from_numpy(v.view(np.float16).reshape(shape).copy())


def _param(t: torch.Tensor) -> dict:
    a = t.detach().to("cpu", torch.float16).contiguous().numpy()
    return {"id": str(uuid.uuid4()), "param": {"value": a.view(np.uint16).reshape(-1), "shape": [int(s) for s in a.shape]}}


# ---------------------------------------------------------------------------------------------------
# Diffuser record <-> dump-tree names (what the weight pack and sdxl_unet_load use; SURVEY Appendix B)
# ---------------------------------------------------------------------------------------------------
def _get_linear(rec, out: Dict[str, torch.Tensor], path: str, bias: bool = True) -> None:
    out[f"{path}/weight"] = _tensor(rec["weight"], path + ".weight")
    if rec.get("bias") is not None:
        out[f"{path}/bias"] = _tensor(rec["bias"], path + ".bias")
    elif bias:
        raise BurnRecordError(f"{path}: bias missing")


def _get_norm(rec, out, path):      # GroupNorm / LayerNorm of the reference: fields gamma, beta
    out[f"{path}/weight"] = _tensor(rec["gamma"], path + ".gamma")
    out[f"{path}/bias"] = _tensor(rec["beta"], path + ".beta")


def _get_res(rec, out, path):
    _get_norm(rec["norm_in"], out, f"{path}/norm_in")
    _get_linear(rec["conv_in"], out, f"{path}/conv_in")
    _get_linear(rec["lin_embed"], out, f"{path}/lin_embed")
    _get_norm(rec["norm_out"], out, f"{path}/norm_out")
    _get_linear(rec["conv_out"], out, f"{path}/conv_out")
    if rec.get("skip_connection") is not None:
        _get_linear(rec["skip_connection"], out, f"{path}/skip_connection")


def _get_attn(rec, out, path):
    for n in ("query", "key", "value"):
        _get_linear(rec[n], out, f"{path}/{n}", bias=False)
    _get_linear(rec["out"], out, f"{path}/out")


def _get_st(rec, out, path):
    _get_norm(rec["norm"], out, f"{path}/norm")
    _get_linear(rec["proj_in"], out, f"{path}/proj_in")
    _get_linear(rec["proj_out"], out, f"{path}/proj_out")
    for j, b in enumerate(rec["blocks"]):
        bp = f"{path}/transformer_{j}"
        for n in ("norm1", "norm2", "norm3"):
            _get_norm(b[n], out, f"{bp}/{n}")
        _get_attn(b["attn1"], out, f"{bp}/attn1")
        _get_attn(b["attn2"], out, f"{bp}/attn2")
        _get_linear(b["mlp"]["geglu"]["proj"], out, f"{bp}/mlp/geglu/proj")
        _get_linear(b["mlp"]["lin"], out, f"{bp}/mlp/lin")


def _get_block(rec, out, path):
    """UNetBlocks enum (src/model/unet/mod.rs:508-516): {"Conv"|"Res"|"Down"|"ResT"|"ResTU"|"ResU": record}."""
    if not isinstance(rec, dict) or len(rec) != 1:
        raise BurnRecordError(f"{path}: expected a one-entry enum map")
    (variant, body), = rec.items()
    if variant in ("Conv", "Down"):
        _get_linear(body, out, path)
    elif variant == "Res":
        _get_res(body, out, path)
    elif variant in ("ResT", "ResTU", "ResU"):
        _get_res(body["res"], out, f"{path}/res")
        if variant != "ResU":
            _get_st(body["transformer"], out, f"{path}/transformer")
        if variant != "ResT":
            _get_linear(body["upsample"]["conv"], out, f"{path}/upsample/conv")
    else:
        raise BurnRecordError(f"{path}: unknown UNetBlocks variant {variant!r}")


def diffuser_record_to_weights(item: Tree) -> Dict[str, torch.Tensor]:
    """Diffuser record (src/model/stablediffusion/mod.rs:308-314) -> {dump-tree name: f16 tensor}."""
    out: Dict[str, torch.Tensor] = {}
    u = item["diffusion"]
    for n in ("lin1_time_embed", "lin2_time_embed", "lin1_label_embed", "lin2_label_embed"):
        _get_linear(u[n], out, n)
    for i, b in enumerate(u["input_blocks"]):
        _get_block(b, out, f"input_blocks/{i}")
    m = u["middle_block"]
    _get_res(m["res1"], out, "middle_block/res1")
    _get_st(m["transformer"], out, "middle_block/transformer")
    _get_res(m["res2"], out, "middle_block/res2")
    for i, b in enumerate(u["output_blocks"]):
        _get_block(b, out, f"output_blocks/{i}")
    _get_norm(u["norm_out"], out, "norm_out")
    _get_linear(u["conv_out"], out, "conv_out")
    out["alphas_cumprod"] = _tensor(item["alpha_cumulative_products"], "alpha_cumulative_products")
    return out


# ---- inverse: weights -> record (writer side of the fixture / a `convert` replacement)
def _put_linear(w, path, conv: bool = False):
    rec = {"weight": _param(w[f"{path}/weight"]), "bias": _param(w[f"{path}/bias"]) if f"{path}/bias" in w else None}
    if conv:   # Conv2d record: the non-tensor fields are constants (nil)
        rec.update({"stride": None, "kernel_size": None, "dilation": None, "groups": None, "padding": None})
    return rec


def _put_norm(w, path, group: bool):
    rec = {"gamma": _param(w[f"{path}/weight"]), "beta": _param(w[f"{path}/bias"]), "eps": None}
    if group:
        rec = {"n_group": None, "n_channel": None, **rec}
    return rec


def _put_res(w, path):
    return {"norm_in": _put_norm(w, f"{path}/norm_in", True), "silu_in": None, "conv_in": _put_linear(w, f"{path}/conv_in", True), "silu_embed": None,
            "lin_embed": _put_linear(w, f"{path}/lin_embed"), "norm_out": _put_norm(w, f"{path}/norm_out", True), "silu_out": None,
            "conv_out": _put_linear(w, f"{path}/conv_out", True),
            "skip_connection": _put_linear(w, f"{path}/skip_connection", True) if f"{path}/skip_connection/weight" in w else None}


def _put_attn(w, path):
    return {"n_head": None, "query": _put_linear(w, f"{path}/query"), "key": _put_linear(w, f"{path}/key"), "value": _put_linear(w, f"{path}/value"),
            "out": _put_linear(w, f"{path}/out")}


def _put_st(w, path):
    blocks = []
    j = 0
    while f"{path}/transformer_{j}/norm1/weight" in w:
        bp = f"{path}/transformer_{j}"
        blocks.append({"norm1": _put_norm(w, f"{bp}/norm1", False), "attn1": _put_attn(w, f"{bp}/attn1"), "norm2": _put_norm(w, f"{bp}/norm2", False),
                       "attn2": _put_attn(w, f"{bp}/attn2"), "norm3": _put_norm(w, f"{bp}/norm3", False),
                       "mlp": {"geglu": {"proj": _put_linear(w, f"{bp}/mlp/geglu/proj"), "gelu": None}, "lin": _put_linear(w, f"{bp}/mlp/lin")}})
        j += 1
    return {"norm": _put_norm(w, f"{path}/norm", True), "proj_in": _put_linear(w, f"{path}/proj_in"), "blocks": blocks, "proj_out": _put_linear(w, f"{path}/proj_out")}


def _put_block(w, path, kind: str):
    if kind == "conv":
        return {"Conv": _put_linear(w, path, True)}
    if kind == "downsample":
        return {"Down": _put_linear(w, path, True)}
    if kind == "resnet":
        return {"Res": _put_res(w, path)}
    body = {"res": _put_res(w, f"{path}/res")}
    if "transformer" in kind:
        body["transformer"] = _put_st(w, f"{path}/transformer")
    if kind.endswith("upsample"):
        body["upsample"] = {"conv": _put_linear(w, f"{path}/upsample/conv", True)}
    return {{"resnet_transformer": "ResT", "resnet_transformer_upsample": "ResTU", "resnet_upsample": "ResU"}[kind]: body}


def weights_to_diffuser_record(cfg: UNetConfig, w: Dict[str, torch.Tensor]) -> Tree:
    from .config import block_program
    ins, mid, outs = block_program(cfg)
    unet = {"model_channels": None}
    for n in ("lin1_time_embed", "lin2_time_embed", "lin1_label_embed", "lin2_label_embed"):
        unet[n] = _put_linear(w, n)
        if n.startswith("lin1"):
            unet["silu" + n[4:]] = None
    unet["input_blocks"] = [_put_block(w, b.path, b.kind) for b in ins]
    unet["middle_block"] = {"res1": _put_res(w, "middle_block/res1"), "transformer": _put_st(w, "middle_block/transformer"),
                            "res2": _put_res(w, "middle_block/res2")}
    unet["output_blocks"] = [_put_block(w, b.path, b.kind) for b in outs]
    unet["norm_out"] = _put_norm(w, "norm_out", True)
    unet["silu_out"] = None
    unet["conv_out"] = _put_linear(w, "conv_out", True)
    return {"n_steps": None, "alpha_cumulative_products": _param(w["alphas_cumprod"]), "diffusion": unet, "is_refiner": None}


# ---------------------------------------------------------------------------------------------------
# .cfg (burn Config JSON) and the two entry points
# ---------------------------------------------------------------------------------------------------
def read_diffuser_cfg(path: str) -> UNetConfig:
    """DiffuserConfig (src/model/stablediffusion/mod.rs:269-278) -> UNetConfig."""
    with open(path) as fh:
        d = json.load(fh)
    try:
        return UNetConfig(adm_in_channels=int(d["adm_in_channels"]), model_channels=int(d["model_channels"]), channel_mults=tuple(int(x) for x in d["channel_mults"]),
                          transformer_depths=tuple(int(x) for x in d["transformer_depths"]), context_dim=int(d["context_dim"]), is_refiner=bool(d["is_refiner"]),
                          n_head_channels=int(d["num_head_channels"]))
    except KeyError as e:
        raise BurnRecordError(f"{path}: DiffuserConfig key {e} missing") from None


def write_diffuser_cfg(path: str, cfg: UNetConfig) -> None:
    """Refuses an edit UNet (cfg.is_edit): DiffuserConfig has no field for the edit layout, and a record read back without it would
    load as a plain UNet with an 8-channel latent."""
    if cfg.is_edit:
        raise BurnRecordError(f"{path}: DiffuserConfig cannot record the edit layout (is_edit); keep edit UNets in the diffusers format")
    with open(path, "w") as fh:
        json.dump({"adm_in_channels": cfg.adm_in_channels, "model_channels": cfg.model_channels, "channel_mults": list(cfg.channel_mults),
                   "num_head_channels": cfg.n_head_channels, "transformer_depths": list(cfg.transformer_depths), "context_dim": cfg.context_dim,
                   "is_refiner": cfg.is_refiner}, fh)


def load_diffuser(model_path: str) -> Tuple[UNetConfig, Dict[str, torch.Tensor]]:
    """== load_diffuser_model (src/bin/sample/main.rs:35-41): `<model_path>.cfg` + `<model_path>.mpk` -> config and weights in the
    dump-tree naming that Diffuser(...) / build_pack / sdxl_unet_load take."""
    cfg = read_diffuser_cfg(model_path + ".cfg")
    meta, item = read_mpk(model_path + ".mpk")
    w = diffuser_record_to_weights(item)
    if w["alphas_cumprod"].numel() != cfg.n_steps:
        cfg = UNetConfig(**{**cfg.__dict__, "n_steps": int(w["alphas_cumprod"].numel())})
    return cfg, w


def save_diffuser(model_path: str, cfg: UNetConfig, weights: Dict[str, torch.Tensor]) -> None:
    """Inverse of load_diffuser (what `convert` writes, src/bin/convert/main.rs:48-70)."""
    write_diffuser_cfg(model_path + ".cfg", cfg)
    write_mpk(model_path + ".mpk", weights_to_diffuser_record(cfg, weights))


# ---------------------------------------------------------------------------------------------------
# LatentDecoder record (src/model/stablediffusion/mod.rs:193-197: {autoencoder, scale_factor}) <-> dump-tree names of sdxl_vae_load
# ---------------------------------------------------------------------------------------------------
def _get_resnet_block(rec, out, path):     # autoencoder ResnetBlock (autoencoder/mod.rs:489-498)
    _get_norm(rec["norm1"], out, f"{path}/norm1")
    _get_linear(rec["conv1"], out, f"{path}/conv1")
    _get_norm(rec["norm2"], out, f"{path}/norm2")
    _get_linear(rec["conv2"], out, f"{path}/conv2")
    if rec.get("nin_shortcut") is not None:
        _get_linear(rec["nin_shortcut"], out, f"{path}/nin_shortcut")


def _get_mid(rec, out, path):              # Mid (autoencoder/mod.rs:436-441) with ConvSelfAttentionBlock (:541-548)
    _get_resnet_block(rec["block_1"], out, f"{path}/block_1")
    _get_norm(rec["attn"]["norm"], out, f"{path}/attn/norm")
    for n in ("q", "k", "v", "proj_out"):
        _get_linear(rec["attn"][n], out, f"{path}/attn/{n}")
    _get_resnet_block(rec["block_2"], out, f"{path}/block_2")


def latent_decoder_record_to_weights(item: Tree) -> Dict[str, torch.Tensor]:
    out: Dict[str, torch.Tensor] = {}
    ae = item["autoencoder"]
    _get_linear(ae["post_quant_conv"], out, "post_quant_conv")
    d = ae["decoder"]
    _get_linear(d["conv_in"], out, "decoder/conv_in")
    _get_mid(d["mid"], out, "decoder/mid")
    for i, b in enumerate(d["blocks"]):
        for r in ("res1", "res2", "res3"):
            _get_resnet_block(b[r], out, f"decoder/blocks/{i}/{r}")
        if b.get("upsampler") is not None:
            _get_linear(b["upsampler"], out, f"decoder/blocks/{i}/upsampler")
    _get_norm(d["norm_out"], out, "decoder/norm_out")
    _get_linear(d["conv_out"], out, "decoder/conv_out")
    e = ae["encoder"]
    _get_linear(e["conv_in"], out, "encoder/conv_in")
    for i, b in enumerate(e["blocks"]):
        for r in ("res1", "res2"):
            _get_resnet_block(b[r], out, f"encoder/blocks/{i}/{r}")
        if b.get("downsampler") is not None:          # PaddedConv2d {conv, kernel_size, stride, padding, padding_actual}
            _get_linear(b["downsampler"]["conv"], out, f"encoder/blocks/{i}/downsampler/conv")
    _get_mid(e["mid"], out, "encoder/mid")
    _get_norm(e["norm_out"], out, "encoder/norm_out")
    _get_linear(e["conv_out"], out, "encoder/conv_out")
    _get_linear(ae["quant_conv"], out, "quant_conv")
    return out


def _put_resnet_block(w, path):
    return {"norm1": _put_norm(w, f"{path}/norm1", True), "silu1": None, "conv1": _put_linear(w, f"{path}/conv1", True),
            "norm2": _put_norm(w, f"{path}/norm2", True), "silu2": None, "conv2": _put_linear(w, f"{path}/conv2", True),
            "nin_shortcut": _put_linear(w, f"{path}/nin_shortcut", True) if f"{path}/nin_shortcut/weight" in w else None}


def _put_mid(w, path):
    attn = {"norm": _put_norm(w, f"{path}/attn/norm", True)}
    for n in ("q", "k", "v", "proj_out"):
        attn[n] = _put_linear(w, f"{path}/attn/{n}", True)
    return {"block_1": _put_resnet_block(w, f"{path}/block_1"), "attn": attn, "block_2": _put_resnet_block(w, f"{path}/block_2")}


def weights_to_latent_decoder_record(w: Dict[str, torch.Tensor]) -> Tree:
    def count(prefix):
        i = 0
        while f"{prefix}/{i}/res1/norm1/weight" in w:
            i += 1
        return i
    dec_blocks = []
    for i in range(count("decoder/blocks")):
        bp = f"decoder/blocks/{i}"
        dec_blocks.append({"res1": _put_resnet_block(w, f"{bp}/res1"), "res2": _put_resnet_block(w, f"{bp}/res2"), "res3": _put_resnet_block(w, f"{bp}/res3"),
                           "upsampler": _put_linear(w, f"{bp}/upsampler", True) if f"{bp}/upsampler/weight" in w else None})
    enc_blocks = []
    for i in range(count("encoder/blocks")):
        bp = f"encoder/blocks/{i}"
        down = None
        if f"{bp}/downsampler/conv/weight" in w:
            down = {"conv": _put_linear(w, f"{bp}/downsampler/conv", True), "kernel_size": None, "stride": None,
                    "padding": {"pad_left": None, "pad_right": None, "pad_top": None, "pad_bottom": None}, "padding_actual": None}
        enc_blocks.append({"res1": _put_resnet_block(w, f"{bp}/res1"), "res2": _put_resnet_block(w, f"{bp}/res2"), "downsampler": down})
    decoder = {"conv_in": _put_linear(w, "decoder/conv_in", True), "mid": _put_mid(w, "decoder/mid"), "blocks": dec_blocks,
               "norm_out": _put_norm(w, "decoder/norm_out", True), "silu": None, "conv_out": _put_linear(w, "decoder/conv_out", True)}
    encoder = {"conv_in": _put_linear(w, "encoder/conv_in", True), "mid": _put_mid(w, "encoder/mid"), "blocks": enc_blocks,
               "norm_out": _put_norm(w, "encoder/norm_out", True), "silu": None, "conv_out": _put_linear(w, "encoder/conv_out", True)}
    return {"autoencoder": {"encoder": encoder, "decoder": decoder, "quant_conv": _put_linear(w, "quant_conv", True),
                            "post_quant_conv": _put_linear(w, "post_quant_conv", True)}, "scale_factor": None}


def _vae_config_from_weights(w: Dict[str, torch.Tensor], scale_factor: float) -> VaeConfig:
    """The reference hard-codes the autoencoder widths (AutoencoderConfig::new()); here they are read off the tensors, so that a
    reduced-width record (tests) and the real one both load."""
    def chans(prefix):
        out, i = [], 0
        while f"{prefix}/{i}/res1/conv1/weight" in w:
            t = w[f"{prefix}/{i}/res1/conv1/weight"]
            out.append((int(t.shape[1]), int(t.shape[0])))
            i += 1
        return tuple(out)
    ng = 32
    return VaeConfig(block_channels=chans("decoder/blocks"), latent_channels=int(w["post_quant_conv/weight"].shape[0]), n_group=ng,
                     scale_factor=float(scale_factor), enc_block_channels=chans("encoder/blocks"), enc_z_channels=int(w["quant_conv/weight"].shape[0]))


def load_latent_decoder(model_path: str) -> Tuple[VaeConfig, Dict[str, torch.Tensor]]:
    """== load_latent_decoder_model (src/bin/sample/main.rs:43-51): `<path>.cfg` ({"scale_factor": ..}, LatentDecoderConfig,
    stablediffusion/mod.rs:176-179) + `<path>.mpk` -> VaeConfig and weights in the names sdxl_vae_load / LatentDecoder(...) take."""
    with open(model_path + ".cfg") as fh:
        d = json.load(fh)
    if "scale_factor" not in d:
        raise BurnRecordError(f"{model_path}.cfg: LatentDecoderConfig key 'scale_factor' missing")
    _, item = read_mpk(model_path + ".mpk")
    w = latent_decoder_record_to_weights(item)
    return _vae_config_from_weights(w, d["scale_factor"]), w


def save_latent_decoder(model_path: str, cfg: VaeConfig, weights: Dict[str, torch.Tensor]) -> None:
    with open(model_path + ".cfg", "w") as fh:
        json.dump({"scale_factor": cfg.scale_factor}, fh)
    write_mpk(model_path + ".mpk", weights_to_latent_decoder_record(weights))


# ---------------------------------------------------------------------------------------------------
# Embedder record (stablediffusion/mod.rs:652-658: {clip, open_clip, clip_tokenizer, open_clip_tokenizer}); the tokenizers carry no
# parameters (they are rebuilt from the vocabulary files) and are skipped
# ---------------------------------------------------------------------------------------------------
def clip_record_to_weights(rec: Tree, where: str) -> Dict[str, torch.Tensor]:
    """CLIP (src/model/clip/mod.rs:62-69) -> the names of sdxl_clip_load."""
    out: Dict[str, torch.Tensor] = {}
    out["token_embedding/weight"] = _tensor(rec["token_embedding"]["weight"], where + ".token_embedding")
    out["position_embedding/weight"] = _tensor(rec["position_embedding"], where + ".position_embedding")
    for i, b in enumerate(rec["blocks"]):
        bp = f"blocks/{i}"
        _get_norm(b["attn_ln"], out, f"{bp}/attn_ln")
        _get_norm(b["mlp_ln"], out, f"{bp}/mlp_ln")
        for n in ("query", "key", "value", "out"):
            _get_linear(b["attn"][n], out, f"{bp}/attn/{n}")
        _get_linear(b["mlp"]["fc1"], out, f"{bp}/mlp/fc1")
        _get_linear(b["mlp"]["fc2"], out, f"{bp}/mlp/fc2")
    _get_norm(rec["layer_norm"], out, "layer_norm")
    if rec.get("text_projection") is not None:
        out["text_projection"] = _tensor(rec["text_projection"], where + ".text_projection")
    return out


def weights_to_clip_record(w: Dict[str, torch.Tensor]) -> Tree:
    blocks, i = [], 0
    while f"blocks/{i}/attn_ln/weight" in w:
        bp = f"blocks/{i}"
        attn = {"n_head": None}
        for n in ("query", "key", "value", "out"):
            attn[n] = _put_linear(w, f"{bp}/attn/{n}")
        blocks.append({"attn": attn, "attn_ln": _put_norm(w, f"{bp}/attn_ln", False),
                       "mlp": {"quick_gelu": None, "fc1": _put_linear(w, f"{bp}/mlp/fc1"), "qgelu": None, "gelu": None, "fc2": _put_linear(w, f"{bp}/mlp/fc2")},
                       "mlp_ln": _put_norm(w, f"{bp}/mlp_ln", False)})
        i += 1
    return {"token_embedding": {"weight": _param(w["token_embedding/weight"])}, "position_embedding": _param(w["position_embedding/weight"]),
            "blocks": blocks, "layer_norm": _put_norm(w, "layer_norm", False),
            "text_projection": _param(w["text_projection"]) if "text_projection" in w else None}


def _clip_cfg(d: dict, where: str) -> ClipConfig:
    try:
        return ClipConfig(n_vocab=int(d["n_vocab"]), n_state=int(d["n_state"]), embed_dim=int(d["embed_dim"]), n_head=int(d["n_head"]), n_ctx=int(d["n_ctx"]),
                          n_layer=int(d["n_layer"]), quick_gelu=bool(d["quick_gelu"]))
    except KeyError as e:
        raise BurnRecordError(f"{where}: CLIPConfig key {e} missing") from None


def load_embedder(model_path: str) -> Tuple[ClipConfig, Dict[str, torch.Tensor], ClipConfig, Dict[str, torch.Tensor]]:
    """== load_embedder_model (src/bin/sample/main.rs:28-33): EmbedderConfig JSON {clip_config, open_clip_config}
    (stablediffusion/mod.rs:626-630) + record -> (CLIP-L config, weights, OpenCLIP config, weights) for ClipTextEncoder(...)."""
    with open(model_path + ".cfg") as fh:
        d = json.load(fh)
    for k in ("clip_config", "open_clip_config"):
        if k not in d:
            raise BurnRecordError(f"{model_path}.cfg: EmbedderConfig key '{k}' missing")
    _, item = read_mpk(model_path + ".mpk")
    return (_clip_cfg(d["clip_config"], model_path + ".cfg"), clip_record_to_weights(item["clip"], "clip"),
            _clip_cfg(d["open_clip_config"], model_path + ".cfg"), clip_record_to_weights(item["open_clip"], "open_clip"))


def save_embedder(model_path: str, clip_cfg: ClipConfig, clip_w: Dict[str, torch.Tensor], open_cfg: ClipConfig, open_w: Dict[str, torch.Tensor]) -> None:
    with open(model_path + ".cfg", "w") as fh:
        json.dump({"clip_config": dict(clip_cfg.__dict__), "open_clip_config": dict(open_cfg.__dict__)}, fh)
    write_mpk(model_path + ".mpk", {"clip": weights_to_clip_record(clip_w), "open_clip": weights_to_clip_record(open_w),
                                    "clip_tokenizer": None, "open_clip_tokenizer": None})


def read_model_dir(model_dir: str, use_refiner: bool = False) -> dict:
    """The files of a reference download as `sample` addresses them (src/bin/sample/main.rs:156, 220, 242, 255, 274):
    `<model_dir>/{embedder, diffuser, refiner, latent_decoder}.{mpk,cfg}` -> {"embedder": (clip cfg, weights, open_clip cfg, weights),
    "diffuser": (cfg, weights), "refiner": (cfg, weights) | None, "latent_decoder": (cfg, weights)}. Host memory only."""
    import os
    return {"embedder": load_embedder(os.path.join(model_dir, "embedder")),
            "diffuser": load_diffuser(os.path.join(model_dir, "diffuser")),
            "refiner": load_diffuser(os.path.join(model_dir, "refiner")) if use_refiner else None,
            "latent_decoder": load_latent_decoder(os.path.join(model_dir, "latent_decoder"))}
