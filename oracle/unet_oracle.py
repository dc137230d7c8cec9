"""ORACLE — test infrastructure only. Never imported by the product path (sdxl_b200 / libsdxl_b200.so).

CPU f32 restatement (PyTorch tensor ops, no CUDA) of the reference's diffusion sampling path, written
line-by-line from /root/reference (Gadersd/stable-diffusion-xl-burn @ 6650d90). The reference is Rust on
burn 0.13 / burn-tch (libtorch); neither cargo/rustc nor the un-vendored crates exist in this
environment, so the reference cannot be executed here and it ships no numeric goldens for this path
(its only test is a tokenizer KAT, src/token/clip.rs:232-249):

    *** PARITY UNPINNED *** — the goldens under tests/golden/ are produced by THIS oracle
    (tests/golden/make_golden.py). What pins the oracle is (a) every primitive is cross-checked against
    an independent PyTorch implementation of the same published op (F.group_norm, F.layer_norm,
    F.scaled_dot_product_attention — the exact libtorch call the reference's backend makes,
    src/backend.rs:66-74 —, F.gelu, F.conv2d, F.interpolate) in tests/test_oracle.py, and (b) the block
    program is checked against the parameter/FLOP totals SURVEY.md derives from the reference.

burn semantics relied on (burn 0.13, not verifiable here): mean_dim keeps the reduced dim; nn::Gelu is
the exact erf form; Tensor::repeat tiles a size-1 dim; mask_where(mask, v) takes v where mask is true;
nn::Linear is x.matmul(W[in,out]) + b.

Weights: dict name -> tensor using the reference's dump-tree names and layouts (src/model/unet/load.rs,
python/save.py): Linear weight [in,out], conv weight OIHW.
"""
from __future__ import annotations

import dataclasses
import math
from typing import Callable, Collection, Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

W = Dict[str, torch.Tensor]


@dataclasses.dataclass
class Attach:
    """What is attached to the UNet, one field per attachment kind of the engine (DESIGN.md §8-15). The defaults attach nothing.
    A row b of the UNet batch reads row b % n of every per-row tensor.

    controls: [(ControlNetConfig, f32 weights, hint [n, 3, H, W], scale)], residuals added to the skips and the middle in order.
    prompts: image prompts [(f32 adapter weights (pack names), tokens [B, S_ip, ctx], scales {transformer block path: s},
        mask [n_images, H, W] or None)], every prompt in each attn2.
    uncond_tokens: for forward_diffuser, the tokens of the unconditional rows, one per prompt (tokens are the conditional rows').
    t2i: (the summed T2I features [F_0, F_1, F_2, F_3] of rows [n, ...], t_min): added while timesteps[0] >= t_min.
    concat: the inpainting condition [n, C, h, w], concatenated to the latent before the first conv.
    pag_layers: transformer block paths whose self-attention computes the identity out(value(x)).
    pag_scale: for forward_diffuser, PAG's p_t of an integer timestep.
    freeu: diffusers' (s1, s2, b1, b2), at the skip pops of output blocks 0..5 when all four are nonzero."""
    controls: Sequence = ()
    prompts: Sequence = ()
    uncond_tokens: Sequence = ()
    t2i: Optional[Tuple[Sequence[torch.Tensor], int]] = None
    concat: Optional[torch.Tensor] = None
    pag_layers: Collection[str] = ()
    pag_scale: Optional[Callable[[int], float]] = None
    freeu: Optional[Sequence[float]] = None


NOTHING = Attach()


def _rows(t: torch.Tensor, n: int) -> torch.Tensor:
    """Row b of the result is row b % len(t) of t."""
    return t[torch.arange(n) % t.shape[0]]


# ---------------------------------------------------------------------------------------------------
# primitives
# ---------------------------------------------------------------------------------------------------
def layernorm_fn(x: torch.Tensor, eps: float) -> torch.Tensor:
    """src/model/layernorm/mod.rs:42-49 (== groupnorm/mod.rs:75-82): u = x - mean; u / sqrt(mean(u*u) + eps)."""
    u = x - x.mean(dim=-1, keepdim=True)
    return u / ((u * u).mean(dim=-1, keepdim=True) + eps).sqrt()


def layer_norm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    """LayerNorm::forward, src/model/layernorm/mod.rs:34-40."""
    return layernorm_fn(x, eps) * gamma.unsqueeze(0) + beta.unsqueeze(0)


def group_norm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, n_group: int = 32, eps: float = 1e-5) -> torch.Tensor:
    """GroupNorm::forward, src/model/groupnorm/mod.rs:52-73: reshape [B, G, rest] -> layernorm -> per-channel affine."""
    shape = x.shape
    n_batch = shape[0]
    y = layernorm_fn(x.reshape(n_batch, n_group, -1), eps).reshape(shape)
    aff = [1] * x.dim()
    aff[1] = gamma.shape[0]
    return y * gamma.reshape(aff) + beta.reshape(aff)


def silu(x: torch.Tensor) -> torch.Tensor:
    """SILU::forward, src/model/silu.rs:14-16."""
    return x * torch.sigmoid(x)


def gelu_erf(x: torch.Tensor) -> torch.Tensor:
    """burn::nn::Gelu (exact erf form)."""
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def linear(x: torch.Tensor, w: W, path: str) -> torch.Tensor:
    """nn::Linear::forward: x.matmul(W[in,out]) + b."""
    y = x.matmul(w[f"{path}/weight"])
    b = w.get(f"{path}/bias")
    return y if b is None else y + b


def conv2d(x: torch.Tensor, w: W, path: str, stride: int = 1, padding: int = 1) -> torch.Tensor:
    """nn::conv::Conv2d::forward (OIHW weight)."""
    return F.conv2d(x, w[f"{path}/weight"], w.get(f"{path}/bias"), stride=stride, padding=padding)


def qkv_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, mask: Optional[torch.Tensor], n_head: int) -> torch.Tensor:
    """Generic qkv_attention, src/backend.rs:88-128 (the path every non-libtorch backend runs)."""
    n_batch, n_qctx, n_state = q.shape
    n_ctx = k.shape[1]
    scale = (n_state / n_head) ** -0.25
    n_hstate = n_state // n_head
    q = q.reshape(n_batch, n_qctx, n_head, n_hstate).transpose(1, 2) * scale
    k = k.reshape(n_batch, n_ctx, n_head, n_hstate).transpose(1, 2).transpose(2, 3) * scale
    v = v.reshape(n_batch, n_ctx, n_head, n_hstate).transpose(1, 2)
    qk = q.matmul(k)
    if mask is not None:
        qk = qk + mask[:n_qctx, :n_ctx].unsqueeze(0).unsqueeze(0)
    w_ = torch.softmax(qk, dim=3)
    return w_.matmul(v).transpose(1, 2).flatten(2, 3)


def timestep_embedding(timesteps: torch.Tensor, dim: int, max_period: int = 10000) -> torch.Tensor:
    """src/model/unet/mod.rs:21-39: cat([cos(t*f), sin(t*f)]), f_i = exp(-ln(max_period) * i / half)."""
    half = dim // 2
    freqs = (torch.arange(half, dtype=torch.float32) * (-math.log(max_period) / half)).exp()
    args = timesteps.to(torch.float32).unsqueeze(0).transpose(0, 1).repeat(1, half) * freqs.unsqueeze(0)
    return torch.cat([args.cos(), args.sin()], dim=1)


def conditioning_embedding(pooled: torch.Tensor, dim: int, size: torch.Tensor, crop: torch.Tensor, ar: torch.Tensor) -> torch.Tensor:
    """src/model/unet/mod.rs:41-57."""
    cat = torch.cat([size, crop, ar], dim=1)
    n_batch, w_ = cat.shape
    embed = timestep_embedding(cat.reshape(n_batch * w_), dim, 10000).reshape(n_batch, w_ * dim)
    return torch.cat([pooled, embed], dim=1)


# ---------------------------------------------------------------------------------------------------
# blocks
# ---------------------------------------------------------------------------------------------------
def res_block(x: torch.Tensor, emb: torch.Tensor, w: W, p: str) -> torch.Tensor:
    """ResBlock::forward, src/model/unet/mod.rs:1082-1106."""
    h = group_norm(x, w[f"{p}/norm_in/weight"], w[f"{p}/norm_in/bias"])
    h = silu(h)
    h = conv2d(h, w, f"{p}/conv_in")
    embed_out = linear(silu(emb), w, f"{p}/lin_embed")
    h = h + embed_out.reshape(embed_out.shape[0], embed_out.shape[1], 1, 1)
    h = group_norm(h, w[f"{p}/norm_out/weight"], w[f"{p}/norm_out/bias"])
    h = silu(h)
    h = conv2d(h, w, f"{p}/conv_out")
    if f"{p}/skip_connection/weight" in w:
        return conv2d(x, w, f"{p}/skip_connection", padding=0) + h
    return x + h


def multi_head_attention(x: torch.Tensor, context: Optional[torch.Tensor], w: W, p: str, n_head: int) -> torch.Tensor:
    """MultiHeadAttention::forward, src/model/unet/mod.rs:1005-1023 (q/k/v bias-free, out with bias)."""
    xa = x if context is None else context
    q = linear(x, w, f"{p}/query")
    k = linear(xa, w, f"{p}/key")
    v = linear(xa, w, f"{p}/value")
    return linear(qkv_attention(q, k, v, None, n_head), w, f"{p}/out")


def geglu(x: torch.Tensor, w: W, p: str) -> torch.Tensor:
    """GEGLU::forward, src/model/unet/mod.rs:942-956: value half first, gate half second."""
    projected = linear(x, w, f"{p}/proj")
    n = projected.shape[-1] // 2
    return projected[..., :n] * gelu_erf(projected[..., n:])


def mask_grid(H: int, W: int, T: int):
    """(mh, mw) of diffusers' IPAdapterMaskProcessor.downsample for T queries and an H x W mask, both kept >= 1 (diffusers divides
    by zero there)."""
    ratio = W / H
    mh = max(1, int(math.sqrt(T / ratio)))
    mh += int(T % mh != 0)
    return mh, max(1, T // mh)


def downsample_mask(mask: torch.Tensor, T: int) -> torch.Tensor:
    """[n, H, W] -> [n, T]: bicubic to mask_grid, flattened row-major, zero-padded or cut to T."""
    n, H, W = mask.shape
    mh, mw = mask_grid(H, W, T)
    m = F.interpolate(mask[:, None].float(), size=(mh, mw), mode="bicubic", align_corners=False)[:, 0].reshape(n, -1)
    if m.shape[1] < T:
        return torch.cat([m, m.new_zeros(n, T - m.shape[1])], 1)
    return m[:, :T]


def multi_attention(q, k, v, sources: Sequence, n_head: int) -> torch.Tensor:
    """softmax(q k^T) v + sum over sources (k_s, v_s, s, m) of s * m[t] * softmax(q k_s^T) v_s (m None: 1), in order."""
    h = qkv_attention(q, k, v, None, n_head)
    for k_s, v_s, s, m in sources:
        a = s * qkv_attention(q, k_s, v_s, None, n_head)
        h = h + (a if m is None else a * m[None, :, None])
    return h


def prompt_sources(T: int, prompts: Sequence, a: str, p: str) -> list:
    """The attention sources of image prompts in the attn2 `a` of transformer block `p` for T queries: one per unmasked prompt
    (one softmax over all its tokens), one per image of a masked prompt, weighted per query by its downsampled mask."""
    out = []
    for wa, tokens, scales, mask in prompts:
        k, v = linear(tokens, wa, f"{a}/ip_key"), linear(tokens, wa, f"{a}/ip_value")
        if mask is None:
            out.append((k, v, scales[p], None))
            continue
        n = mask.shape[0]
        m = downsample_mask(mask, T)
        per = k.shape[1] // n
        out += [(k[:, i * per:(i + 1) * per], v[:, i * per:(i + 1) * per], scales[p], m[i]) for i in range(n)]
    return out


def transformer_block(x: torch.Tensor, context: torch.Tensor, w: W, p: str, n_head: int, att: Attach = NOTHING) -> torch.Tensor:
    """TransformerBlock::forward, src/model/unet/mod.rs:885-891; PAG's identity self-attention if p is in att.pag_layers, the image
    prompts' sources beside the text in attn2."""
    h = layer_norm(x, w[f"{p}/norm1/weight"], w[f"{p}/norm1/bias"])
    if p in att.pag_layers:
        x = x + linear(linear(h, w, f"{p}/attn1/value"), w, f"{p}/attn1/out")
    else:
        x = x + multi_head_attention(h, None, w, f"{p}/attn1", n_head)
    h = layer_norm(x, w[f"{p}/norm2/weight"], w[f"{p}/norm2/bias"])
    if att.prompts:
        a = f"{p}/attn2"
        q, k, v = linear(h, w, f"{a}/query"), linear(context, w, f"{a}/key"), linear(context, w, f"{a}/value")
        x = x + linear(multi_attention(q, k, v, prompt_sources(q.shape[1], att.prompts, a, p), n_head), w, f"{a}/out")
    else:
        x = x + multi_head_attention(h, context, w, f"{p}/attn2", n_head)
    h = layer_norm(x, w[f"{p}/norm3/weight"], w[f"{p}/norm3/bias"])
    return x + linear(geglu(h, w, f"{p}/mlp/geglu"), w, f"{p}/mlp/lin")  # MLP::forward :915-919


def spatial_transformer(x: torch.Tensor, context: torch.Tensor, w: W, p: str, n_head: int, depth: int,
                        att: Attach = NOTHING) -> torch.Tensor:
    """SpatialTransformer::forward, src/model/unet/mod.rs:820-845."""
    n_batch, n_channel, height, width = x.shape
    x_in = x
    x = group_norm(x, w[f"{p}/norm/weight"], w[f"{p}/norm/bias"])
    x = x.reshape(n_batch, n_channel, height * width).transpose(1, 2)
    x = linear(x, w, f"{p}/proj_in")
    for j in range(depth):
        x = transformer_block(x, context, w, f"{p}/transformer_{j}", n_head, att)
    x = linear(x, w, f"{p}/proj_out").transpose(1, 2).reshape(n_batch, n_channel, height, width)
    return x_in + x


def upsample(x: torch.Tensor, w: W, p: str) -> torch.Tensor:
    """Upsample::forward, src/model/unet/mod.rs:742-751: nearest 2x via reshape/repeat, then 3x3 conv."""
    n_batch, n_channel, height, width = x.shape
    x = x.reshape(n_batch, n_channel, height, 1, width, 1).repeat(1, 1, 1, 2, 1, 2).reshape(n_batch, n_channel, 2 * height, 2 * width)
    return conv2d(x, w, f"{p}/conv")


# ---------------------------------------------------------------------------------------------------
# UNet
# ---------------------------------------------------------------------------------------------------
def unet_blocks(cfg) -> Tuple[List[tuple], tuple, List[tuple]]:
    """Block program of UNetConfig::init, src/model/unet/mod.rs:115-173 (input), :238-248 (middle),
    :250-328 (output). Entries: (kind, path, n_head, depth)."""
    mc, nl = cfg.model_channels, len(cfg.channel_mults)
    n_head = lambda ch: ch // cfg.n_head_channels  # noqa: E731   (:113)
    ins = [("conv", "input_blocks/0", 0, 0)]
    idx = 1
    for level in range(nl):
        c_out = cfg.channel_mults[level] * mc
        for _ in range(2):
            if level != 1 and level != 2:                      # :125
                ins.append(("resnet", f"input_blocks/{idx}", 0, 0))
            else:
                ins.append(("resnet_transformer", f"input_blocks/{idx}", n_head(c_out), cfg.transformer_depths[level]))
            idx += 1
        if level != nl - 1:                                    # :169
            ins.append(("downsample", f"input_blocks/{idx}", 0, 0))
            idx += 1
    cm = cfg.channel_mults[-1] * mc
    mid = ("middle", "middle_block", n_head(cm), cfg.transformer_depths[-1])  # :238-248
    outs = []
    idx = 0
    for level in reversed(range(nl)):
        c_out = cfg.channel_mults[level] * mc
        for k in range(3):
            if level != 1 and level != 2:                      # :264
                kind = "resnet_upsample" if (k == 2 and level != 0) else "resnet"   # :273-281
                outs.append((kind, f"output_blocks/{idx}", 0, 0))
            else:
                kind = "resnet_transformer_upsample" if k == 2 else "resnet_transformer"  # :288-322
                outs.append((kind, f"output_blocks/{idx}", n_head(c_out), cfg.transformer_depths[level]))
            idx += 1
    return ins, mid, outs


def _run_block(kind: str, p: str, n_head: int, depth: int, x, emb, context, w: W, att: Attach = NOTHING):
    if kind == "conv":
        return conv2d(x, w, p)                                  # :776-780
    if kind == "downsample":
        return conv2d(x, w, p, stride=2, padding=1)             # :760-774
    if kind == "resnet":
        return res_block(x, emb, w, p)
    x = res_block(x, emb, w, f"{p}/res")                        # ResTransformer* :571-577, :657-663, ResUpsample :607-612
    if "transformer" in kind:
        x = spatial_transformer(x, context, w, f"{p}/transformer", n_head, depth, att)
    if kind.endswith("upsample"):
        x = upsample(x, w, f"{p}/upsample")
    return x


def _emb(cfg, w: W, timesteps: torch.Tensor, label: torch.Tensor) -> torch.Tensor:
    """The time + label embedding, src/model/unet/mod.rs:449-460."""
    t_emb = timestep_embedding(timesteps, cfg.model_channels, 10000)
    t_emb = linear(t_emb, w, "lin1_time_embed")
    t_emb = silu(t_emb)
    t_emb = linear(t_emb, w, "lin2_time_embed")
    label_emb = linear(label, w, "lin1_label_embed")
    label_emb = silu(label_emb)
    label_emb = linear(label_emb, w, "lin2_label_embed")
    return t_emb + label_emb


def encoder(cfg, w: W, x: torch.Tensor, emb: torch.Tensor, context: torch.Tensor, att: Attach = NOTHING,
            adds: Optional[Dict[str, torch.Tensor]] = None) -> Tuple[torch.Tensor, List[torch.Tensor]]:
    """The input blocks and the middle block: (the middle block's output, every input block's output). adds {block path or
    "middle_block": tensor} is added to that block's output (T2I features, the ControlNet's hint embedding)."""
    adds = adds or {}
    ins, mid, _ = unet_blocks(cfg)
    saved = []
    for kind, p, nh, d in ins:
        x = _run_block(kind, p, nh, d, x, emb, context, w, att)
        if p in adds:
            x = x + adds[p]
        saved.append(x)
    _, mp, nh, d = mid                                          # ResTransformerRes::forward :713-719
    x = res_block(x, emb, w, f"{mp}/res1")
    x = spatial_transformer(x, context, w, f"{mp}/transformer", nh, d, att)
    x = res_block(x, emb, w, f"{mp}/res2")
    if mp in adds:
        x = x + adds[mp]
    return x, saved


def unet_forward(cfg, w: W, x: torch.Tensor, timesteps: torch.Tensor, context: torch.Tensor, label: torch.Tensor,
                 att: Optional[Attach] = None) -> torch.Tensor:
    """UNet::forward, src/model/unet/mod.rs:449-493. x [B,4,h,w], timesteps Int [1] (or [B]),
    context [B,n_ctx,Cctx], label [B,adm]. The attachments go in where and in the order the engine's plan puts them: the
    inpainting condition before the first conv; T2I features on the injection blocks' and the middle block's outputs; ControlNet
    residuals (their nets see the latent without the condition, run unperturbed and without image prompts) on the skips and the
    middle; FreeU at the skip pops; PAG and image prompts in the transformer blocks."""
    att = att or NOTHING
    n = x.shape[0]
    latent = x
    if att.concat is not None:
        x = torch.cat([x, _rows(att.concat, n)], dim=1)
    emb = _emb(cfg, w, timesteps, label)
    adds = {}
    if att.t2i is not None and int(timesteps[0]) >= att.t2i[1]:
        adds = {p: _rows(f, n) for p, f in zip(injection_blocks(cfg) + ["middle_block"], att.t2i[0])}
    x, saved = encoder(cfg, w, x, emb, context, att, adds)
    for ncfg, wc, hint, scale in att.controls:
        res, r_mid = controlnet_forward(ncfg, wc, latent, timesteps, context, label, hint_embedding(ncfg, wc, hint))
        saved = [s + scale * r for s, r in zip(saved, res)]
        x = x + scale * r_mid
    for i, (kind, p, nh, d) in enumerate(unet_blocks(cfg)[2]):
        skip = saved.pop()
        if freeu_enabled(att.freeu) and i // 3 < 2:           # up_blocks[0] and [1]: three output blocks each
            x, skip = apply_freeu(i // 3, x, skip, att.freeu)
        x = torch.cat([x, skip], dim=1)                         # :484
        x = _run_block(kind, p, nh, d, x, emb, context, w, att)
    x = group_norm(x, w["norm_out/weight"], w["norm_out/bias"])
    x = silu(x)
    return conv2d(x, w, "conv_out")


# ---------------------------------------------------------------------------------------------------
# attachments the forward computes
# ---------------------------------------------------------------------------------------------------
def hint_embedding(ncfg, w: W, hint: torch.Tensor) -> torch.Tensor:
    """SGM input_hint_block: conv(in -> c0), then SiLU + conv after each conv, stride 2 on every second, last conv(c_last -> mc)."""
    x = conv2d(hint, w, "input_hint_block/0")
    idx = 2
    for _ in range(len(ncfg.hint_block_channels) - 1):
        x = conv2d(silu(x), w, f"input_hint_block/{idx}")
        x = conv2d(silu(x), w, f"input_hint_block/{idx + 2}", stride=2)
        idx += 4
    return conv2d(silu(x), w, f"input_hint_block/{idx}")


def controlnet_forward(ncfg, w: W, x, timesteps, context, label, hint_emb):
    """The control branch: (residuals r_i = zero_conv_i(h_i) for every input block, r_mid = middle_block_out(mid)), the hint
    embedding (row b reads row b % n) added to the first conv's output."""
    cfg = ncfg.unet
    h, saved = encoder(cfg, w, x, _emb(cfg, w, timesteps, label), context, adds={"input_blocks/0": _rows(hint_emb, x.shape[0])})
    return [conv2d(s, w, f"zero_convs/{i}", padding=0) for i, s in enumerate(saved)], conv2d(h, w, "middle_block_out", padding=0)


def injection_blocks(cfg) -> List[str]:
    """Input blocks receiving the T2I features F_0..F_2: a level's last resnet+transformer block, or for a transformer-free level
    its last block (its Downsample); F_3 follows the middle block."""
    ins, _, _ = unet_blocks(cfg)
    per_level, level = [[]], 0
    for kind, p, _, _ in ins[1:]:
        per_level[level].append((kind, p))
        if kind == "downsample":
            level += 1
            per_level.append([])
    out = []
    for blocks in per_level:
        tr = [p for kind, p in blocks if "transformer" in kind]
        out.append(tr[-1] if tr else blocks[-1][1])
    return out


def fourier_filter(x_in: torch.Tensor, threshold: int, scale: float) -> torch.Tensor:
    """diffusers.utils.torch_utils.fourier_filter on a real [B, C, H, W] tensor (its f16 / bf16 upcast does not apply here)."""
    x = x_in
    B, C, H, W = x.shape
    x_freq = torch.fft.fftn(x, dim=(-2, -1))
    x_freq = torch.fft.fftshift(x_freq, dim=(-2, -1))
    mask = torch.ones((B, C, H, W), dtype=x.dtype, device=x.device)
    crow, ccol = H // 2, W // 2
    mask[..., crow - threshold:crow + threshold, ccol - threshold:ccol + threshold] = scale
    x_freq = x_freq * mask
    x_freq = torch.fft.ifftshift(x_freq, dim=(-2, -1))
    x_filtered = torch.fft.ifftn(x_freq, dim=(-2, -1)).real
    return x_filtered.to(dtype=x_in.dtype)


def freeu_enabled(freeu: Optional[Sequence[float]]) -> bool:
    """diffusers' is_freeu_enabled: all four values given and nonzero."""
    return freeu is not None and all(freeu)


def apply_freeu(k: int, x: torch.Tensor, res: torch.Tensor, freeu: Sequence[float]):
    """diffusers' apply_freeu at resolution_idx k (0, 1): x's first half of channels times b, the skip filtered with s."""
    s, b = freeu[k], freeu[2 + k]
    half = x.shape[1] // 2
    x = torch.cat([x[:, :half] * b, x[:, half:]], dim=1)
    return x, fourier_filter(res, 1, s)


def to_f32(weights: W) -> W:
    """The reference stores f16 records and the oracle computes in f32: widen once."""
    return {k: v.detach().to("cpu", torch.float32) for k, v in weights.items()}


# ---------------------------------------------------------------------------------------------------
# Diffuser (sampler)
# ---------------------------------------------------------------------------------------------------
class OracleConditioning:
    """Conditioning record, src/model/stablediffusion/mod.rs:544-555 (f32 here)."""

    def __init__(self, **kw):
        self.context_full = kw.get("context_full")
        self.context_open_clip = kw.get("context_open_clip")
        self.unconditional_context_full = kw.get("unconditional_context_full")
        self.unconditional_context_open_clip = kw.get("unconditional_context_open_clip")
        self.channel_context = kw.get("channel_context")
        self.channel_context_refiner = kw.get("channel_context_refiner")
        self.unconditional_channel_context = kw.get("unconditional_channel_context")
        self.unconditional_channel_context_refiner = kw.get("unconditional_channel_context_refiner")
        self.resolution = kw.get("resolution", (1024, 1024))


def forward_diffuser(cfg, w: W, latent: torch.Tensor, timestep: torch.Tensor, c: OracleConditioning, guidance: float,
                     att: Optional[Attach] = None) -> torch.Tensor:
    """Diffuser::forward_diffuser, src/model/stablediffusion/mod.rs:494-541, with the attachments on every row. Image prompts: the
    conditional (and perturbed) rows of image b see tokens b % n_batch, the unconditional rows uncond_tokens b % n_batch. PAG adds
    p_t * (c - perturbed) to the guided noise (to the conditional noise on the refiner), the perturbed rows being the conditional
    ones with the identity self-attention in att.pag_layers."""
    n_batch = latent.shape[0]
    att = att or NOTHING
    if not cfg.is_refiner:
        uctx, ctx, uy, y = c.unconditional_context_full, c.context_full, c.unconditional_channel_context, c.channel_context
    else:
        uctx, ctx, uy, y = (c.unconditional_context_open_clip, c.context_open_clip,
                            c.unconditional_channel_context_refiner, c.channel_context_refiner)
    cond = dataclasses.replace(att, prompts=[(wa, _rows(t, n_batch), s, m) for wa, t, s, m in att.prompts], pag_layers=())
    conditional = unet_forward(cfg, w, latent, timestep, ctx, y, cond)
    if att.pag_layers:
        perturbed = unet_forward(cfg, w, latent, timestep, ctx, y, dataclasses.replace(cond, pag_layers=att.pag_layers))
        p_t = att.pag_scale(int(timestep[0]))
    if cfg.is_refiner:                                          # :528-530
        return conditional + p_t * (conditional - perturbed) if att.pag_layers else conditional
    unc = dataclasses.replace(cond, prompts=[(wa, _rows(t, n_batch), s, m) for (wa, _, s, m), t in zip(att.prompts, att.uncond_tokens,
                                                                                                      strict=True)])
    unconditional = unet_forward(cfg, w, latent, timestep, uctx.unsqueeze(0).repeat(n_batch, 1, 1),
                                 uy.unsqueeze(0).repeat(n_batch, 1), unc)
    guided = unconditional + (conditional - unconditional) * guidance   # :539-540
    return guided + p_t * (conditional - perturbed) if att.pag_layers else guided


def get_alpha(alphas: torch.Tensor, i: int) -> float:
    """Diffuser::get_alpha, :485-492 — the record stores f16; the scalar is widened to f64."""
    return float(alphas[i].to(torch.float16).to(torch.float64))


def diffuse_latent(cfg, w: W, alphas: torch.Tensor, latent: torch.Tensor, c: OracleConditioning, step_start: int, n_steps: int,
                   guidance: float, reference: Optional[torch.Tensor] = None, mask: Optional[torch.Tensor] = None,
                   step_noise: Optional[Sequence[torch.Tensor]] = None, trace=None, att: Optional[Attach] = None) -> torch.Tensor:
    """Diffuser::diffuse_latent (:390-432) and diffuse_latent_with_inpainting (:434-483); DDIM, sigma = 0.
    `trace(iteration, latent)` (test aid, not in the reference) is called after every loop iteration."""
    total = cfg.n_steps
    step_size = total // n_steps                                # :400
    start = total - step_start                                  # :404
    it = 0
    for t in range(start - 1, -1, -step_size):                  # (0..start).rev().step_by(step_size)  :406
        current_alpha = get_alpha(alphas, t)
        prev_alpha = get_alpha(alphas, t - step_size) if t >= step_size else 1.0   # :408-412
        sqrt_noise = math.sqrt(1.0 - current_alpha)
        if reference is not None:                               # :463-465
            noised_reference = reference * math.sqrt(current_alpha) + step_noise[it] * sqrt_noise
            latent = torch.where(mask.bool(), latent, noised_reference)   # mask_where: mask true keeps latent
        timestep = torch.tensor([t], dtype=torch.int32)
        pred_noise = forward_diffuser(cfg, w, latent, timestep, c, guidance, att)
        predx0 = (latent - pred_noise * sqrt_noise) / math.sqrt(current_alpha)     # :423
        dir_latent = pred_noise * math.sqrt(1.0 - prev_alpha)                      # :424
        latent = predx0 * math.sqrt(prev_alpha) + dir_latent                       # :426-428 (sigma = 0)
        it += 1
        if trace is not None:
            trace(it, latent)
    return latent


def sample_latent(cfg, w, alphas, noise, c, guidance, n_steps, trace=None, att=None):
    """Diffuser::sample_latent, :317-332 (noise = gen_noise(), injected)."""
    return diffuse_latent(cfg, w, alphas, noise, c, 0, n_steps, guidance, trace=trace, att=att)


def sample_latent_with_inpainting(cfg, w, alphas, noise, c, guidance, n_steps, reference, mask, step_noise, att=None):
    """Diffuser::sample_latent_with_inpainting, :334-353."""
    return diffuse_latent(cfg, w, alphas, noise, c, 0, n_steps, guidance, reference, mask, step_noise, att=att)


def refine_latent(cfg, w, alphas, latent, c, guidance, step_start, n_steps, noise, att=None):
    """Diffuser::refine_latent, :355-376."""
    t = cfg.n_steps - step_start
    start_alpha = get_alpha(alphas, t)
    noised = latent * math.sqrt(start_alpha) + noise * math.sqrt(1.0 - start_alpha)
    return diffuse_latent(cfg, w, alphas, noised, c, step_start, n_steps, guidance, att=att)


def make_inpaint_mask(img_w: int, img_h: int, lat_w: int, lat_h: int, crop_left: Optional[int], crop_right: Optional[int],
                      crop_top: Optional[int], crop_bottom: Optional[int], crop_out: bool) -> torch.Tensor:
    """The `sample` binary's mask, src/bin/sample/main.rs:144-190: ones [crop_h, crop_w] padded with zeros to the latent extent,
    Bool, expanded to [1, 4, h, w], inverted by --crop-out."""
    crop_left = 0 if crop_left is None else crop_left                # :144-147
    crop_right = img_w if crop_right is None else crop_right
    crop_top = 0 if crop_top is None else crop_top
    crop_bottom = img_h if crop_bottom is None else crop_bottom
    scale = img_h // lat_h                                          # :164
    crop_left, crop_right, crop_top, crop_bottom = crop_left // scale, crop_right // scale, crop_top // scale, crop_bottom // scale   # :165-168
    ones = torch.ones(crop_bottom - crop_top, crop_right - crop_left)
    mask = F.pad(ones, (crop_left, lat_w - crop_right, crop_top, lat_h - crop_bottom), value=0.0).bool()   # :177-179
    mask = mask.unsqueeze(0).unsqueeze(0).expand(1, 4, lat_h, lat_w)
    return ~mask if crop_out else mask                               # :183-187


def n_iterations(n_steps: int, step_start: int = 0, total: int = 1000) -> int:
    """ceil((total - step_start) / floor(total / n_steps)) — SURVEY D6/D7."""
    step = total // n_steps
    return len(range(total - step_start - 1, -1, -step))


# ---------------------------------------------------------------------------------------------------
# FLOP counter (SURVEY 8(d) rule: 2*MAC over Linear, conv, QK^T, PV only)
# ---------------------------------------------------------------------------------------------------
def unet_flops(cfg, w_shapes: Dict[str, Tuple[int, ...]], h: int, wd: int, n_ctx: int = 77, batch: int = 1) -> float:
    fl = 0.0
    mc, ted = cfg.model_channels, 4 * cfg.model_channels

    def lin(path, rows):
        nonlocal fl
        k, n = w_shapes[f"{path}/weight"]
        fl += 2.0 * rows * k * n

    def conv(path, ho, wo):
        nonlocal fl
        o, i, kh, kw = w_shapes[f"{path}/weight"]
        fl += 2.0 * batch * ho * wo * o * i * kh * kw

    def res(p, hh, ww):
        conv(f"{p}/conv_in", hh, ww)
        lin(f"{p}/lin_embed", batch)
        conv(f"{p}/conv_out", hh, ww)
        if f"{p}/skip_connection/weight" in w_shapes:
            conv(f"{p}/skip_connection", hh, ww)

    def st(p, hh, ww, depth):
        nonlocal fl
        t = hh * ww
        c = w_shapes[f"{p}/proj_in/weight"][0]
        lin(f"{p}/proj_in", batch * t)
        for j in range(depth):
            b = f"{p}/transformer_{j}"
            for nm in ("query", "key", "value", "out"):
                lin(f"{b}/attn1/{nm}", batch * t)
            fl += 4.0 * batch * t * t * c
            lin(f"{b}/attn2/query", batch * t)
            lin(f"{b}/attn2/key", batch * n_ctx)
            lin(f"{b}/attn2/value", batch * n_ctx)
            lin(f"{b}/attn2/out", batch * t)
            fl += 4.0 * batch * t * n_ctx * c
            lin(f"{b}/mlp/geglu/proj", batch * t)
            lin(f"{b}/mlp/lin", batch * t)
        lin(f"{p}/proj_out", batch * t)

    lin("lin1_time_embed", 1)
    lin("lin2_time_embed", 1)
    lin("lin1_label_embed", batch)
    lin("lin2_label_embed", batch)
    ins, mid, outs = unet_blocks(cfg)
    hh, ww = h, wd
    for kind, p, nh, d in ins:
        if kind == "conv":
            conv(p, hh, ww)
        elif kind == "downsample":
            hh, ww = hh // 2, ww // 2
            conv(p, hh, ww)
        elif kind == "resnet":
            res(p, hh, ww)
        else:
            res(f"{p}/res", hh, ww)
            st(f"{p}/transformer", hh, ww, d)
    res("middle_block/res1", hh, ww)
    st("middle_block/transformer", hh, ww, mid[3])
    res("middle_block/res2", hh, ww)
    for kind, p, nh, d in outs:
        if kind == "resnet":
            res(p, hh, ww)
            continue
        res(f"{p}/res", hh, ww)
        if "transformer" in kind:
            st(f"{p}/transformer", hh, ww, d)
        if kind.endswith("upsample"):
            hh, ww = hh * 2, ww * 2
            conv(f"{p}/upsample/conv", hh, ww)
    conv("conv_out", hh, ww)
    return fl
