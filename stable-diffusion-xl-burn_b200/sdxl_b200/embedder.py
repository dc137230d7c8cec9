"""Host-side mirror of the reference's CLIP text encoder and Embedder (src/model/clip/mod.rs,
src/model/stablediffusion/mod.rs:626-776) over libsdxl_b200.so: tokenizers and encoders are the library's."""
from __future__ import annotations

import ctypes as C
import math
from typing import List, Sequence, Tuple

import torch

from . import _lib
from .config import ClipConfig
from .engine import Conditioning, Context, _ptr, set_adapters
from .tokenizer import _Tokenizer
from .weights import build_pack


class ClipTextEncoder:
    """== CLIP<B> (src/model/clip/mod.rs:73-147)."""

    def __init__(self, ctx: Context, cfg: ClipConfig, weights):
        self.ctx, self.cfg = ctx, cfg
        pack = weights if isinstance(weights, torch.Tensor) else build_pack(weights)
        on_device = pack.is_cuda
        ctx.enter()
        if on_device:
            torch.cuda.current_stream(ctx.device).synchronize()
        cs = _lib.ClipCfg(cfg.n_vocab, cfg.n_state, cfg.embed_dim, cfg.n_head, cfg.n_ctx, cfg.n_layer, int(cfg.quick_gelu))
        h = C.c_void_p()
        ctx.check(ctx.lib.sdxl_clip_load(ctx.h, C.byref(cs), pack.data_ptr(), pack.numel(), int(on_device), C.byref(h)), "sdxl_clip_load")
        self.h = h

    def close(self) -> None:
        if getattr(self, "h", None):
            self.ctx.lib.sdxl_clip_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_adapters(self, adapters) -> None:
        """Replaces the active LoRA set with [(adapter, scale), ...] (sdxl_clip_set_adapters); [] restores the loaded weights."""
        set_adapters(self.ctx, self.ctx.lib.sdxl_clip_set_adapters, self.h, adapters, "sdxl_clip_set_adapters")

    def max_sequence_length(self) -> int:
        return self.cfg.n_ctx

    def num_layers(self) -> int:
        return self.cfg.n_layer

    def _tokens(self, tokens) -> Tuple[int, "C.Array"]:
        t = torch.as_tensor(tokens, dtype=torch.int32).reshape(-1, self.cfg.n_ctx).contiguous().cpu()
        B = t.shape[0]
        arr = (C.c_int32 * (B * self.cfg.n_ctx))(*t.flatten().tolist())
        return B, arr

    def forward_hidden(self, tokens, hidden_idx: int) -> torch.Tensor:
        """tokens int [B, n_ctx] -> f32 [B, n_ctx, n_state] on the device (stream after blocks[0..hidden_idx])."""
        B, arr = self._tokens(tokens)
        out = torch.empty((B, self.cfg.n_ctx, self.cfg.n_state), dtype=torch.float32, device=self.ctx.device)
        self.ctx.enter()
        self.ctx.check(self.ctx.lib.sdxl_clip_forward_hidden(self.h, B, arr, hidden_idx, _ptr(out), 0), "sdxl_clip_forward_hidden")
        self.ctx.leave()
        return out

    def forward_hidden_pooled(self, tokens, hidden_idx: int) -> Tuple[torch.Tensor, torch.Tensor]:
        B, arr = self._tokens(tokens)
        out = torch.empty((B, self.cfg.n_ctx, self.cfg.n_state), dtype=torch.float32, device=self.ctx.device)
        pooled = torch.empty((B, self.cfg.embed_dim), dtype=torch.float32, device=self.ctx.device)
        self.ctx.enter()
        self.ctx.check(self.ctx.lib.sdxl_clip_forward_hidden_pooled(self.h, B, arr, hidden_idx, _ptr(out), _ptr(pooled), 0),
                       "sdxl_clip_forward_hidden_pooled")
        self.ctx.leave()
        return out, pooled

    @property
    def plan_flops(self) -> float:
        return float(self.ctx.lib.sdxl_clip_plan_flops(self.h))


def conditioning_embedding(ctx: Context, pooled: torch.Tensor, dim: int, size: Sequence[int], crop: Sequence[int],
                           ar: Sequence[int]) -> torch.Tensor:
    """== conditioning_embedding (src/model/unet/mod.rs:41-57): cat([pooled, timestep_embedding(cat[size, crop, ar], dim)])
    for one sample; the sinusoid comes from the library's timestep_embedding kernel."""
    vals = [int(v) for v in (*size, *crop, *ar)]
    emb = ctx.timestep_embedding(vals, dim).reshape(1, len(vals) * dim)
    return torch.cat([pooled.reshape(1, -1).to(emb.device, torch.float32), emb], dim=1)


class Embedder:
    """== Embedder<B> (src/model/stablediffusion/mod.rs:646-776): two tokenizers + two text encoders -> Conditioning."""

    def __init__(self, ctx: Context, clip: ClipTextEncoder, open_clip: ClipTextEncoder, clip_tokenizer: _Tokenizer,
                 open_clip_tokenizer: _Tokenizer):
        self.ctx, self.clip, self.open_clip = ctx, clip, open_clip
        self.clip_tokenizer, self.open_clip_tokenizer = clip_tokenizer, open_clip_tokenizer

    def _context(self, text: str, size, crop, ar):
        """Embedder::context / unconditional_context (mod.rs:691-759); batch 1 like the reference's `sample`."""
        t1 = self.clip_tokenizer.tokenize_text(text, self.clip.max_sequence_length())            # text_to_context_clip
        clip_context = self.clip.forward_hidden([t1], self.clip.num_layers() - 1)                 # penultimate layer
        t2 = self.open_clip_tokenizer.tokenize_text(text, self.open_clip.max_sequence_length())  # text_to_context_open_clip
        open_clip_context, pooled = self.open_clip.forward_hidden_pooled([t2], self.open_clip.num_layers() - 1)
        aesthetic = [6]  # Tensor::from_ints([6]) (mod.rs:703,741): the refiner's label has 5 sinusoid blocks, 1280 + 5*256 = 2560
        return (torch.cat([clip_context, open_clip_context], dim=2), open_clip_context,
                conditioning_embedding(self.ctx, pooled, 256, size, crop, ar),
                conditioning_embedding(self.ctx, pooled, 256, size, crop, aesthetic))

    def text_to_conditioning(self, text: str, size: Sequence[int], crop: Sequence[int], ar: Sequence[int]) -> Conditioning:
        """== Embedder::text_to_conditioning (mod.rs:654-689). size/crop/ar are [h, w] pairs; resolution = ar."""
        u_full, u_oc, u_ch, u_ch_ref = self._context("", size, crop, ar)
        c_full, c_oc, c_ch, c_ch_ref = self._context(text, size, crop, ar)
        h = torch.float16  # Conditioning::convert -> the Diffuser's f16 backend (stablediffusion/mod.rs:557-580)
        return Conditioning(context_full=c_full.to(h), context_open_clip=c_oc.to(h), channel_context=c_ch.to(h),
                            channel_context_refiner=c_ch_ref.to(h), unconditional_context_full=u_full.squeeze(0).to(h),
                            unconditional_context_open_clip=u_oc.squeeze(0).to(h), unconditional_channel_context=u_ch.squeeze(0).to(h),
                            unconditional_channel_context_refiner=u_ch_ref.squeeze(0).to(h), resolution=(int(ar[0]), int(ar[1])))
