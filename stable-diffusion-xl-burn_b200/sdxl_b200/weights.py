"""Weight naming, deterministic synthetic weights and the flat weight pack.

Tensor names and layouts follow the reference's npy dump tree (src/model/unet/load.rs, python/save.py):
Linear `weight` is [in, out] (save.py:20-25 transposes PyTorch's), conv `weight` is OIHW (save.py:56-72),
norms have `weight`/`bias` [C]; values are f16 like the shipped `.mpk` (HalfPrecisionSettings,
src/bin/convert/main.rs:65-70). `alphas_cumprod` is the LegacyDDPMDiscretization schedule
(python/dump.py:29-36), also stored f16.

No SDXL checkpoint exists offline, so benchmarks and parity tests use the synthetic initialisation of
SURVEY.md 8(d): W ~ N(0, 1/fan_in), residual-branch output projections scaled down, biases ~ N(0, 0.02^2),
gamma = 1 + N(0, 0.05^2), beta ~ N(0, 0.05^2); one master seed.

Pack format ("SDXLPK01"): header {magic[8], u32 n_tensors, u32 0, u64 data_offset}, n_tensors entries
{char name[120], u32 dtype(0=f16, 1=f32), u32 ndim, u64 shape[4], u64 offset, u64 nbytes}, data (256B aligned).
Model weights are f16; f32 entries are used only by LoRA adapter packs (`alpha`).
"""
from __future__ import annotations

import struct
from typing import Dict, Iterable, List, Tuple

import numpy as np
import torch

from .config import ClipConfig, ControlNetConfig, T2IAdapterConfig, UNetConfig, VaeConfig, block_program

Spec = Tuple[str, Tuple[int, ...], str, float]  # name, shape, kind, scale

RESID_SCALE = 0.2


def _res_specs(path: str, c_in: int, c_out: int, ted: int) -> List[Spec]:
    s: List[Spec] = [
        (f"{path}/norm_in/weight", (c_in,), "gamma", 1.0), (f"{path}/norm_in/bias", (c_in,), "beta", 1.0),
        (f"{path}/conv_in/weight", (c_out, c_in, 3, 3), "conv", 1.0), (f"{path}/conv_in/bias", (c_out,), "bias", 1.0),
        (f"{path}/lin_embed/weight", (ted, c_out), "linear", 1.0), (f"{path}/lin_embed/bias", (c_out,), "bias", 1.0),
        (f"{path}/norm_out/weight", (c_out,), "gamma", 1.0), (f"{path}/norm_out/bias", (c_out,), "beta", 1.0),
        (f"{path}/conv_out/weight", (c_out, c_out, 3, 3), "conv", RESID_SCALE),
        (f"{path}/conv_out/bias", (c_out,), "bias", 1.0),
    ]
    if c_in != c_out:
        s += [(f"{path}/skip_connection/weight", (c_out, c_in, 1, 1), "conv", 1.0),
              (f"{path}/skip_connection/bias", (c_out,), "bias", 1.0)]
    return s


def _st_specs(path: str, c: int, ctx: int, depth: int) -> List[Spec]:
    s: List[Spec] = [
        (f"{path}/norm/weight", (c,), "gamma", 1.0), (f"{path}/norm/bias", (c,), "beta", 1.0),
        (f"{path}/proj_in/weight", (c, c), "linear", 1.0), (f"{path}/proj_in/bias", (c,), "bias", 1.0),
        (f"{path}/proj_out/weight", (c, c), "linear", RESID_SCALE), (f"{path}/proj_out/bias", (c,), "bias", 1.0),
    ]
    for j in range(depth):
        b = f"{path}/transformer_{j}"
        for n in ("norm1", "norm2", "norm3"):
            s += [(f"{b}/{n}/weight", (c,), "gamma", 1.0), (f"{b}/{n}/bias", (c,), "beta", 1.0)]
        s += [
            (f"{b}/attn1/query/weight", (c, c), "linear", 1.0), (f"{b}/attn1/key/weight", (c, c), "linear", 1.0),
            (f"{b}/attn1/value/weight", (c, c), "linear", 1.0),
            (f"{b}/attn1/out/weight", (c, c), "linear", RESID_SCALE), (f"{b}/attn1/out/bias", (c,), "bias", 1.0),
            (f"{b}/attn2/query/weight", (c, c), "linear", 1.0), (f"{b}/attn2/key/weight", (ctx, c), "linear", 1.0),
            (f"{b}/attn2/value/weight", (ctx, c), "linear", 1.0),
            (f"{b}/attn2/out/weight", (c, c), "linear", RESID_SCALE), (f"{b}/attn2/out/bias", (c,), "bias", 1.0),
            (f"{b}/mlp/geglu/proj/weight", (c, 8 * c), "linear", 1.0), (f"{b}/mlp/geglu/proj/bias", (8 * c,), "bias", 1.0),
            (f"{b}/mlp/lin/weight", (4 * c, c), "linear", RESID_SCALE), (f"{b}/mlp/lin/bias", (c,), "bias", 1.0),
        ]
    return s


def unet_tensor_specs(cfg: UNetConfig) -> List[Spec]:
    mc, ted = cfg.model_channels, cfg.time_embed_dim
    s: List[Spec] = [
        ("lin1_time_embed/weight", (mc, ted), "linear", 1.0), ("lin1_time_embed/bias", (ted,), "bias", 1.0),
        ("lin2_time_embed/weight", (ted, ted), "linear", 1.0), ("lin2_time_embed/bias", (ted,), "bias", 1.0),
        ("lin1_label_embed/weight", (cfg.adm_in_channels, ted), "linear", 1.0), ("lin1_label_embed/bias", (ted,), "bias", 1.0),
        ("lin2_label_embed/weight", (ted, ted), "linear", 1.0), ("lin2_label_embed/bias", (ted,), "bias", 1.0),
    ]
    ins, mid, outs = block_program(cfg)
    for b in ins + outs:
        if b.kind == "conv":
            s += [(f"{b.path}/weight", (b.c_out, b.c_in, 3, 3), "conv", 1.0), (f"{b.path}/bias", (b.c_out,), "bias", 1.0)]
        elif b.kind == "downsample":
            s += [(f"{b.path}/weight", (b.c_out, b.c_in, 3, 3), "conv", 1.0), (f"{b.path}/bias", (b.c_out,), "bias", 1.0)]
        elif b.kind == "resnet":
            s += _res_specs(b.path, b.c_in, b.c_out, ted)
        else:
            s += _res_specs(f"{b.path}/res", b.c_in, b.c_out, ted)
            if "transformer" in b.kind:
                s += _st_specs(f"{b.path}/transformer", b.c_out, cfg.context_dim, b.depth)
            if b.kind.endswith("upsample"):
                s += [(f"{b.path}/upsample/conv/weight", (b.c_out, b.c_out, 3, 3), "conv", 1.0),
                      (f"{b.path}/upsample/conv/bias", (b.c_out,), "bias", 1.0)]
    s += _res_specs("middle_block/res1", mid.c_in, mid.c_out, ted)
    s += _st_specs("middle_block/transformer", mid.c_out, cfg.context_dim, mid.depth)
    s += _res_specs("middle_block/res2", mid.c_in, mid.c_out, ted)
    s += [("norm_out/weight", (mc,), "gamma", 1.0), ("norm_out/bias", (mc,), "beta", 1.0),
          ("conv_out/weight", (cfg.out_channels, mc, 3, 3), "conv", 1.0), ("conv_out/bias", (cfg.out_channels,), "bias", 1.0)]
    return s


def controlnet_tensor_specs(cfg: ControlNetConfig) -> List[Spec]:
    """A ControlNet pack (include/sdxl_b200.h): the UNet's embeddings, input blocks and middle block under the UNet's names, the
    hint encoder (SGM indices input_hint_block/{0,2,...,14}), one 1x1 zero conv per skip tensor and middle_block_out. The
    synthetic zero convs and last hint conv (zero-initialised in training) get the residual-output scale, so controls matter."""
    s = [sp for sp in unet_tensor_specs(cfg.unet) if sp[0].startswith(("lin", "input_blocks/", "middle_block/"))]
    mc, hc = cfg.unet.model_channels, cfg.hint_block_channels
    convs = [(cfg.hint_in_channels, hc[0], 1.0)]
    for k in range(len(hc) - 1):
        convs += [(hc[k], hc[k], 1.0), (hc[k], hc[k + 1], 1.0)]
    convs.append((hc[-1], mc, RESID_SCALE))
    for i, (ci, co, sc) in enumerate(convs):
        s += [(f"input_hint_block/{2 * i}/weight", (co, ci, 3, 3), "conv", sc), (f"input_hint_block/{2 * i}/bias", (co,), "bias", 1.0)]
    ins, mid, _ = block_program(cfg.unet)
    for i, b in enumerate(ins):
        s += [(f"zero_convs/{i}/weight", (b.c_out, b.c_out, 1, 1), "conv", RESID_SCALE), (f"zero_convs/{i}/bias", (b.c_out,), "bias", 1.0)]
    s += [("middle_block_out/weight", (mid.c_out, mid.c_out, 1, 1), "conv", RESID_SCALE), ("middle_block_out/bias", (mid.c_out,), "bias", 1.0)]
    return s


def t2i_adapter_tensor_specs(cfg: T2IAdapterConfig) -> List[Spec]:
    """A T2I-Adapter pack (include/sdxl_b200.h): diffusers FullAdapterXL's keys without `adapter.`, `/`-separated. The synthetic
    block2 convs (the resnets' residual outputs) get the residual-output scale."""
    ch = cfg.channels
    s: List[Spec] = [("conv_in/weight", (ch[0], cfg.in_channels * 256, 3, 3), "conv", 1.0), ("conv_in/bias", (ch[0],), "bias", 1.0)]
    for k in range(4):
        if k in (1, 2):
            s += [(f"body/{k}/in_conv/weight", (ch[k], ch[k - 1], 1, 1), "conv", 1.0), (f"body/{k}/in_conv/bias", (ch[k],), "bias", 1.0)]
        for j in range(cfg.n_res_blocks):
            p = f"body/{k}/resnets/{j}"
            s += [(f"{p}/block1/weight", (ch[k], ch[k], 3, 3), "conv", 1.0), (f"{p}/block1/bias", (ch[k],), "bias", 1.0),
                  (f"{p}/block2/weight", (ch[k], ch[k], 1, 1), "conv", RESID_SCALE), (f"{p}/block2/bias", (ch[k],), "bias", 1.0)]
    return s


def _vres_specs(path: str, c_in: int, c_out: int) -> List[Spec]:
    s: List[Spec] = [
        (f"{path}/norm1/weight", (c_in,), "gamma", 1.0), (f"{path}/norm1/bias", (c_in,), "beta", 1.0),
        (f"{path}/conv1/weight", (c_out, c_in, 3, 3), "conv", 1.0), (f"{path}/conv1/bias", (c_out,), "bias", 1.0),
        (f"{path}/norm2/weight", (c_out,), "gamma", 1.0), (f"{path}/norm2/bias", (c_out,), "beta", 1.0),
        (f"{path}/conv2/weight", (c_out, c_out, 3, 3), "conv", RESID_SCALE), (f"{path}/conv2/bias", (c_out,), "bias", 1.0),
    ]
    if c_in != c_out:
        s += [(f"{path}/nin_shortcut/weight", (c_out, c_in, 1, 1), "conv", 1.0),
              (f"{path}/nin_shortcut/bias", (c_out,), "bias", 1.0)]
    return s


def vae_encoder_tensor_specs(cfg: VaeConfig) -> List[Spec]:
    """Encoder-side tensors of the autoencoder dump tree (reference src/model/autoencoder/load.rs:38-51, 80-116)."""
    if not cfg.enc_block_channels:
        return []
    c0, ce, cz = cfg.enc_block_channels[0][0], cfg.enc_block_channels[-1][1], cfg.enc_z_channels
    s: List[Spec] = [("encoder/conv_in/weight", (c0, 3, 3, 3), "conv", 1.0), ("encoder/conv_in/bias", (c0,), "bias", 1.0)]
    for i, (ci, co) in enumerate(cfg.enc_block_channels):
        b = f"encoder/blocks/{i}"
        s += _vres_specs(f"{b}/res1", ci, co) + _vres_specs(f"{b}/res2", co, co)
        if i != len(cfg.enc_block_channels) - 1:
            s += [(f"{b}/downsampler/conv/weight", (co, co, 3, 3), "conv", 1.0), (f"{b}/downsampler/conv/bias", (co,), "bias", 1.0)]
    s += _vres_specs("encoder/mid/block_1", ce, ce)
    s += [("encoder/mid/attn/norm/weight", (ce,), "gamma", 1.0), ("encoder/mid/attn/norm/bias", (ce,), "beta", 1.0)]
    for n, sc in (("q", 1.0), ("k", 1.0), ("v", 1.0), ("proj_out", RESID_SCALE)):
        s += [(f"encoder/mid/attn/{n}/weight", (ce, ce, 1, 1), "conv", sc), (f"encoder/mid/attn/{n}/bias", (ce,), "bias", 1.0)]
    s += _vres_specs("encoder/mid/block_2", ce, ce)
    s += [("encoder/norm_out/weight", (ce,), "gamma", 1.0), ("encoder/norm_out/bias", (ce,), "beta", 1.0),
          ("encoder/conv_out/weight", (cz, ce, 3, 3), "conv", 1.0), ("encoder/conv_out/bias", (cz,), "bias", 1.0),
          ("quant_conv/weight", (cz, cz, 1, 1), "conv", 1.0), ("quant_conv/bias", (cz,), "bias", 1.0)]
    return s


def vae_tensor_specs(cfg: VaeConfig) -> List[Spec]:
    """Decoder tensors first (so seeded synthetic decoder weights do not depend on the encoder), then the encoder's."""
    return vae_decoder_tensor_specs(cfg) + vae_encoder_tensor_specs(cfg)


def vae_decoder_tensor_specs(cfg: VaeConfig) -> List[Spec]:
    """Decoder-side tensors of the autoencoder dump tree (reference src/model/autoencoder/load.rs:17-76, 107-114)."""
    cl, c0 = cfg.latent_channels, cfg.block_channels[0][0]
    s: List[Spec] = [
        ("post_quant_conv/weight", (cl, cl, 1, 1), "conv", 1.0), ("post_quant_conv/bias", (cl,), "bias", 1.0),
        ("decoder/conv_in/weight", (c0, cl, 3, 3), "conv", 1.0), ("decoder/conv_in/bias", (c0,), "bias", 1.0),
    ]
    s += _vres_specs("decoder/mid/block_1", c0, c0)
    s += [("decoder/mid/attn/norm/weight", (c0,), "gamma", 1.0), ("decoder/mid/attn/norm/bias", (c0,), "beta", 1.0)]
    for n, sc in (("q", 1.0), ("k", 1.0), ("v", 1.0), ("proj_out", RESID_SCALE)):
        s += [(f"decoder/mid/attn/{n}/weight", (c0, c0, 1, 1), "conv", sc), (f"decoder/mid/attn/{n}/bias", (c0,), "bias", 1.0)]
    s += _vres_specs("decoder/mid/block_2", c0, c0)
    for i, (ci, co) in enumerate(cfg.block_channels):
        b = f"decoder/blocks/{i}"
        s += _vres_specs(f"{b}/res1", ci, co) + _vres_specs(f"{b}/res2", co, co) + _vres_specs(f"{b}/res3", co, co)
        if i != len(cfg.block_channels) - 1:
            s += [(f"{b}/upsampler/weight", (co, co, 3, 3), "conv", 1.0), (f"{b}/upsampler/bias", (co,), "bias", 1.0)]
    cf = cfg.block_channels[-1][1]
    s += [("decoder/norm_out/weight", (cf,), "gamma", 1.0), ("decoder/norm_out/bias", (cf,), "beta", 1.0),
          ("decoder/conv_out/weight", (3, cf, 3, 3), "conv", 1.0), ("decoder/conv_out/bias", (3,), "bias", 1.0)]
    return s


def clip_tensor_specs(cfg: ClipConfig) -> List[Spec]:
    """Text-encoder tensors of the dump tree (reference src/model/clip/load.rs:15-115)."""
    c = cfg.n_state
    s: List[Spec] = [("token_embedding/weight", (cfg.n_vocab, c), "embed", 1.0),
                     ("position_embedding/weight", (cfg.n_ctx, c), "embed", 0.5)]
    for i in range(cfg.n_layer):
        b = f"blocks/{i}"
        for n in ("attn_ln", "mlp_ln"):
            s += [(f"{b}/{n}/weight", (c,), "gamma", 1.0), (f"{b}/{n}/bias", (c,), "beta", 1.0)]
        for n, sc in (("query", 1.0), ("key", 1.0), ("value", 1.0), ("out", RESID_SCALE)):
            s += [(f"{b}/attn/{n}/weight", (c, c), "linear", sc), (f"{b}/attn/{n}/bias", (c,), "bias", 1.0)]
        s += [(f"{b}/mlp/fc1/weight", (c, 4 * c), "linear", 1.0), (f"{b}/mlp/fc1/bias", (4 * c,), "bias", 1.0),
              (f"{b}/mlp/fc2/weight", (4 * c, c), "linear", RESID_SCALE), (f"{b}/mlp/fc2/bias", (c,), "bias", 1.0)]
    s += [("layer_norm/weight", (c,), "gamma", 1.0), ("layer_norm/bias", (c,), "beta", 1.0),
          ("text_projection", (c, cfg.embed_dim), "linear", 1.0)]
    return s


def alphas_cumprod(n_steps: int = 1000) -> torch.Tensor:
    """LegacyDDPMDiscretization: scaled-linear betas 0.00085 -> 0.012 (reference python/dump.py:29-36)."""
    betas = np.linspace(0.00085 ** 0.5, 0.012 ** 0.5, n_steps, dtype=np.float64) ** 2
    return torch.from_numpy(np.cumprod(1.0 - betas, axis=0)).to(torch.float16)


def synth_weights(cfg, seed: int = 0, device: str = "cpu") -> Dict[str, torch.Tensor]:
    """Deterministic (per device type) synthetic f16 weights, reference layouts and names.
    cfg: UNetConfig (adds alphas_cumprod), VaeConfig (decoder tensors), ClipConfig (text encoder), ControlNetConfig or
    T2IAdapterConfig."""
    gen = torch.Generator(device=device)
    gen.manual_seed(seed)
    out: Dict[str, torch.Tensor] = {}
    is_vae = isinstance(cfg, VaeConfig)
    is_clip = isinstance(cfg, ClipConfig)
    is_cn = isinstance(cfg, ControlNetConfig)
    is_t2i = isinstance(cfg, T2IAdapterConfig)
    specs = (vae_tensor_specs(cfg) if is_vae else clip_tensor_specs(cfg) if is_clip else controlnet_tensor_specs(cfg) if is_cn
             else t2i_adapter_tensor_specs(cfg) if is_t2i else unet_tensor_specs(cfg))
    for name, shape, kind, scale in specs:
        if kind == "linear":
            t = torch.randn(shape, generator=gen, device=device) * (scale / shape[0] ** 0.5)
        elif kind == "conv":
            t = torch.randn(shape, generator=gen, device=device) * (scale / (shape[1] * shape[2] * shape[3]) ** 0.5)
        elif kind == "bias":
            t = torch.randn(shape, generator=gen, device=device) * 0.02
        elif kind == "gamma":
            t = 1.0 + torch.randn(shape, generator=gen, device=device) * 0.05
        elif kind == "beta":
            t = torch.randn(shape, generator=gen, device=device) * 0.05
        elif kind == "embed":
            t = torch.randn(shape, generator=gen, device=device) * scale
        else:
            raise ValueError(kind)
        out[name] = t.to(torch.float16)
    if not is_vae and not is_clip and not is_cn and not is_t2i:
        out["alphas_cumprod"] = alphas_cumprod(cfg.n_steps).to(device)
    return out


def n_params(cfg: UNetConfig) -> int:
    return sum(int(np.prod(s[1])) for s in unet_tensor_specs(cfg))


_ENTRY = struct.Struct("<120sII4QQQ")
_HEADER = struct.Struct("<8sIIQ")


def build_pack(tensors: Dict[str, torch.Tensor], device: str | None = None, pin: bool = False) -> torch.Tensor:
    """Serialises name->f16 (or f32) tensor into one flat uint8 tensor (on `device`, default: the tensors' device)."""
    items = list(tensors.items())
    if device is None:
        device = str(items[0][1].device)
    table_bytes = _HEADER.size + _ENTRY.size * len(items)
    off = (table_bytes + 255) // 256 * 256
    data_offset = off
    entries = []
    for name, t in items:
        if t.dtype not in (torch.float16, torch.float32):
            raise TypeError(f"{name}: pack tensors must be f16 or f32")
        if t.dim() > 4 or len(name.encode()) >= 120:
            raise ValueError(f"{name}: unsupported rank/name")
        nbytes = t.numel() * t.element_size()
        shape = list(t.shape) + [0] * (4 - t.dim())
        entries.append((name, t, off, nbytes, shape))
        off = (off + nbytes + 255) // 256 * 256
    total = off
    if device == "cpu":
        buf = torch.zeros(total, dtype=torch.uint8, pin_memory=pin)
    else:
        buf = torch.zeros(total, dtype=torch.uint8, device=device)
    head = bytearray(_HEADER.pack(b"SDXLPK01", len(items), 0, data_offset))
    for name, t, o, nbytes, shape in entries:
        head += _ENTRY.pack(name.encode(), int(t.dtype == torch.float32), t.dim(), *shape, o, nbytes)
    buf[: len(head)] = torch.frombuffer(head, dtype=torch.uint8).to(buf.device)
    for name, t, o, nbytes, shape in entries:
        buf[o:o + nbytes] = t.contiguous().reshape(-1).view(torch.uint8).to(buf.device)
    return buf
