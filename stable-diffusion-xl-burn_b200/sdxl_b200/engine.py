"""Host-side mirror of the reference's module surface for the diffusion sampling path, bound to the
C ABI (libsdxl_b200.so). PyTorch is used only for device memory and streams.

Mirrored reference interfaces (file:line relative to the reference root):
  UNet::forward(x, timesteps, context, label)                 src/model/unet/mod.rs:449-493
  Diffuser::sample_latent / sample_latent_with_inpainting /
            refine_latent                                     src/model/stablediffusion/mod.rs:317-376
  Conditioning                                                src/model/stablediffusion/mod.rs:544-555
  Backend::qkv_attention                                      src/backend.rs:4-10
Error behaviour: the reference panics on shape errors; here every failure raises SdxlError carrying
sdxl_last_error().
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import SdxlError
from .config import UNetConfig, VaeConfig
from .weights import build_pack


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


class Context:
    """One (device, stream). Replaces the reference's fixed LibTorchDevice::Cuda(0) (sample/main.rs:131)."""

    def __init__(self, device: int = 0):
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise SdxlError("sdxl_b200 needs a CUDA device (sm_90); there is no CPU fallback")
        self.device = torch.device("cuda", device)
        torch.cuda.set_device(self.device)
        self.stream = torch.cuda.Stream(self.device)
        h = C.c_void_p()
        rc = self.lib.sdxl_ctx_create(device, C.c_void_p(self.stream.cuda_stream), C.byref(h))
        if rc != 0:
            raise SdxlError(f"sdxl_ctx_create failed with {rc}")
        self.h = h

    def check(self, rc: int, what: str) -> None:
        if rc != 0:
            msg = self.lib.sdxl_last_error(self.h)
            raise SdxlError(f"{what} failed ({rc}): {msg.decode() if msg else ''}")

    def enter(self) -> None:
        """Order the ctx stream after work already queued on torch's current stream."""
        self.stream.wait_stream(torch.cuda.current_stream(self.device))

    def leave(self) -> None:
        torch.cuda.current_stream(self.device).wait_stream(self.stream)

    def call(self, what: str, fn, *args) -> None:
        """fn(*args): a library call queued on the ctx stream after torch's work so far; torch's stream then waits for it, also
        when it fails. A failure raises SdxlError naming `what`."""
        self.enter()
        try:
            self.check(fn(*args), what)
        finally:
            self.leave()

    def synchronize(self) -> None:
        self.check(self.lib.sdxl_ctx_synchronize(self.h), "sdxl_ctx_synchronize")

    @property
    def launch_count(self) -> int:
        return int(self.lib.sdxl_ctx_launch_count(self.h))

    def close(self) -> None:
        if getattr(self, "h", None):
            self.lib.sdxl_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- operator level ------------------------------------------------------------------------
    def qkv_attention(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, mask: Optional[torch.Tensor],
                      n_head: int) -> torch.Tensor:
        """== Backend::qkv_attention (src/backend.rs:4-10). q [B,T,C], k/v [B,S,C] f16; mask: additive [T,S] (the text
        encoders' decoder mask) or None (UNet / VAE)."""
        B, T, Cc = q.shape
        S = k.shape[1]
        q, k, v = (t.to(self.device, torch.float16).contiguous() for t in (q, k, v))
        if mask is not None:
            if tuple(mask.shape) != (T, S):
                raise SdxlError(f"qkv_attention: mask must be [{T},{S}], got {tuple(mask.shape)}")
            mask = mask.to(self.device, torch.float16).contiguous()
        out = torch.empty_like(q)
        self.call("sdxl_qkv_attention", self.lib.sdxl_qkv_attention, self.h, _ptr(q), _ptr(k), _ptr(v), _ptr(mask), B, T, S, Cc,
                  n_head, _ptr(out))
        return out

    def linear(self, x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None,
               residual: Optional[torch.Tensor] = None, geglu: bool = False, out_f16: bool = False) -> torch.Tensor:
        """== nn::Linear::forward, weight [in,out]. x [M,K] f16."""
        x = x.to(self.device, torch.float16).contiguous()
        w = w.to(self.device, torch.float16).contiguous()
        M, K = x.shape
        N = w.shape[1]
        bias = None if bias is None else bias.to(self.device, torch.float16).contiguous()
        residual = None if residual is None else residual.to(self.device, torch.float32).contiguous()
        if geglu:
            out = torch.empty(M, N // 2, device=self.device, dtype=torch.float16)
        else:
            out = torch.empty(M, N, device=self.device, dtype=torch.float16 if out_f16 else torch.float32)
        self.call("sdxl_op_linear", self.lib.sdxl_op_linear, self.h, _ptr(x), _ptr(w), _ptr(bias), _ptr(residual), M, K, N, int(geglu),
                  int(out_f16), _ptr(out))
        return out

    def conv2d(self, x_nhwc: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], stride: int = 1,
               upsample: bool = False) -> torch.Tensor:
        """== Conv2d::forward on NHWC f32 input, OIHW f16 weight; pad = k//2."""
        x = x_nhwc.to(self.device, torch.float32).contiguous()
        w = w.to(self.device, torch.float16).contiguous()
        bias = None if bias is None else bias.to(self.device, torch.float16).contiguous()
        B, H, W, Cin = x.shape
        Cout, _, ks, _ = w.shape
        Ho, Wo = (H // 2, W // 2) if stride == 2 else ((2 * H, 2 * W) if upsample else (H, W))
        out = torch.empty(B, Ho, Wo, Cout, device=self.device, dtype=torch.float32)
        self.call("sdxl_op_conv2d", self.lib.sdxl_op_conv2d, self.h, _ptr(x), _ptr(w), _ptr(bias), B, H, W, Cin, Cout, ks, stride,
                  int(upsample), _ptr(out))
        return out

    def group_norm(self, x1: torch.Tensor, x2: Optional[torch.Tensor], gamma: torch.Tensor, beta: torch.Tensor,
                   n_group: int = 32, eps: float = 1e-5, silu: bool = False) -> torch.Tensor:
        """== GroupNorm::forward (+SiLU) on NHWC f32 [B,HW,C]; x2 is channel-concatenated after x1."""
        x1 = x1.to(self.device, torch.float32).contiguous()
        x2 = None if x2 is None else x2.to(self.device, torch.float32).contiguous()
        B, HW, C1 = x1.shape
        C2 = 0 if x2 is None else x2.shape[2]
        gamma = gamma.to(self.device, torch.float32).contiguous()
        beta = beta.to(self.device, torch.float32).contiguous()
        out = torch.empty(B, HW, C1 + C2, device=self.device, dtype=torch.float16)
        self.call("sdxl_op_group_norm", self.lib.sdxl_op_group_norm, self.h, _ptr(x1), C1, _ptr(x2), C2, B, HW, n_group, _ptr(gamma),
                  _ptr(beta), eps, int(silu), _ptr(out))
        return out

    def layer_norm(self, x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
        x = x.to(self.device, torch.float32).contiguous()
        rows, Cc = x.shape
        gamma = gamma.to(self.device, torch.float32).contiguous()
        beta = beta.to(self.device, torch.float32).contiguous()
        out = torch.empty(rows, Cc, device=self.device, dtype=torch.float16)
        self.call("sdxl_op_layer_norm", self.lib.sdxl_op_layer_norm, self.h, _ptr(x), _ptr(gamma), _ptr(beta), eps, rows, Cc, _ptr(out))
        return out

    def timestep_embedding(self, timesteps: Sequence[int], dim: int, max_period: int = 10000) -> torch.Tensor:
        n = len(timesteps)
        arr = (C.c_int32 * n)(*[int(t) for t in timesteps])
        out = torch.empty(n, dim, device=self.device, dtype=torch.float32)
        self.call("sdxl_op_timestep_embedding", self.lib.sdxl_op_timestep_embedding, self.h, arr, n, dim, max_period, _ptr(out))
        return out

    def randn(self, n: int, seed: int, subsequence: int = 0) -> torch.Tensor:
        out = torch.empty(n, device=self.device, dtype=torch.float32)
        self.call("sdxl_randn", self.lib.sdxl_randn, self.h, _ptr(out), n, seed, subsequence)
        return out


def set_adapters(ctx: "Context", fn, h, adapters: Sequence, what: str) -> None:
    """Calls sdxl_{unet,clip}_set_adapters with [(adapter, scale), ...]; an adapter is a reference-named tensor dict
    (sdxl_b200.lora) or a built pack (uint8 tensor, host or device)."""
    adapters = list(adapters)
    if len(adapters) > _lib.MAX_ADAPTERS:
        raise SdxlError(f"{what}: at most {_lib.MAX_ADAPTERS} adapters per call, got {len(adapters)}")
    packs = [a if isinstance(a, torch.Tensor) else build_pack(a) for a, _ in adapters]
    arr = (_lib.Adapter * max(1, len(packs)))()
    for i, (pk, (_, scale)) in enumerate(zip(packs, adapters)):
        arr[i].pack, arr[i].bytes, arr[i].pack_on_device, arr[i].scale = pk.data_ptr(), pk.numel(), int(pk.is_cuda), float(scale)
    if any(pk.is_cuda for pk in packs):
        torch.cuda.current_stream(ctx.device).synchronize()
    ctx.call(what, fn, h, len(packs), arr)


@dataclass
class Conditioning:
    """Mirror of the reference's Conditioning record (stablediffusion/mod.rs:544-555); f16 tensors."""
    context_full: Optional[torch.Tensor] = None                       # [B,77,2048]
    context_open_clip: Optional[torch.Tensor] = None                  # [B,77,1280]
    unconditional_context_full: Optional[torch.Tensor] = None         # [77,2048]
    unconditional_context_open_clip: Optional[torch.Tensor] = None    # [77,1280]
    channel_context: Optional[torch.Tensor] = None                    # [B,2816]
    channel_context_refiner: Optional[torch.Tensor] = None            # [B,2560]
    unconditional_channel_context: Optional[torch.Tensor] = None      # [2816]
    unconditional_channel_context_refiner: Optional[torch.Tensor] = None  # [2560]
    resolution: Sequence[int] = (1024, 1024)                          # (height, width)

    def _fields(self) -> List[str]:
        return ["context_full", "context_open_clip", "unconditional_context_full", "unconditional_context_open_clip",
                "channel_context", "channel_context_refiner", "unconditional_channel_context",
                "unconditional_channel_context_refiner"]

    def to_struct(self, device: Optional[torch.device]):
        """Returns (ctypes struct, keep-alive list). device=None => host pointers (pinned f16 copies)."""
        keep = []
        s = _lib.Conditioning()
        on_host = device is None
        s.on_host = int(on_host)
        ref = self.context_full if self.context_full is not None else self.context_open_clip
        s.n_batch = int(ref.shape[0])
        s.n_ctx = int(ref.shape[1])
        for f in self._fields():
            t = getattr(self, f)
            if t is None:
                setattr(s, f, None)
                continue
            t = t.to(torch.float16)
            t = t.cpu().contiguous() if on_host else t.to(device).contiguous()
            keep.append(t)
            setattr(s, f, t.data_ptr())
        s.resolution[0], s.resolution[1] = int(self.resolution[0]), int(self.resolution[1])
        return s, keep


class AttachableModel:
    """A device-resident model a UNet can hold (ControlNet, T2IAdapter, IPAdapter). Subclasses name their load and destroy entry
    points and the Diffuser call that detaches them; close() is refused while a UNet holds the model."""
    _load_fn = _destroy_fn = _detach_call = ""

    def _load(self, ctx: "Context", cfg_struct, weights) -> None:
        """Loads weights (a pack-named tensor dict or a built pack, host or device) through _load_fn with cfg_struct."""
        self.ctx = ctx
        pack = weights if isinstance(weights, torch.Tensor) else build_pack(weights)
        if pack.is_cuda:
            torch.cuda.current_stream(ctx.device).synchronize()
        h = C.c_void_p()
        ctx.call(self._load_fn, getattr(ctx.lib, self._load_fn), ctx.h, C.byref(cfg_struct), pack.data_ptr(), pack.numel(),
                 int(pack.is_cuda), C.byref(h))
        self.h = h
        self.attached = 0   # UNets holding the model (Diffuser._attach)

    def handle(self) -> int:
        if not getattr(self, "h", None):
            raise SdxlError(f"{type(self).__name__} is closed")
        return self.h.value

    def close(self) -> None:
        """Frees the device weights. Refused while a UNet holds the model: detach it first."""
        if getattr(self, "attached", 0) > 0:
            raise SdxlError(f"{type(self).__name__}.close: the model is still attached to a UNet (detach it with "
                            f"{self._detach_call} first)")
        if getattr(self, "h", None):
            getattr(self.ctx.lib, self._destroy_fn)(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _cfg_struct(cfg: UNetConfig) -> _lib.UnetCfg:
    s = _lib.UnetCfg()
    s.adm_in_channels = cfg.adm_in_channels
    s.in_channels = cfg.in_channels
    s.out_channels = cfg.out_channels
    s.model_channels = cfg.model_channels
    s.n_levels = cfg.n_levels
    for i, m in enumerate(cfg.channel_mults):
        s.channel_mults[i] = m
    for i, d in enumerate(cfg.transformer_depths):
        s.transformer_depths[i] = d
    s.n_head_channels = cfg.n_head_channels
    s.context_dim = cfg.context_dim
    s.is_refiner = int(cfg.is_refiner)
    s.n_steps = cfg.n_steps
    s.edit_layout = int(cfg.is_edit)
    return s


class Diffuser:
    """Mirror of the reference's Diffuser (UNet + alphas + sampler loops), device-resident."""

    def __init__(self, ctx: Context, cfg: UNetConfig, weights, nccl_comm=None, rank: int = 0, root: int = 0):
        """weights: dict name->f16 tensor (reference layouts) or an already-built pack (uint8 tensor).
        nccl_comm (an ncclComm_t, see sharding.nccl_comm_init): multi-GPU load through sdxl_unet_load_broadcast — only `root`
        passes weights, every other rank passes None and receives the pack over NCCL inside the library."""
        self.ctx, self.cfg = ctx, cfg
        h = C.c_void_p()
        cs = _cfg_struct(cfg)
        pack = None
        if weights is not None:
            pack = weights if isinstance(weights, torch.Tensor) else build_pack(weights)
        on_device = bool(pack is not None and pack.is_cuda)
        if on_device:
            torch.cuda.current_stream(ctx.device).synchronize()
        if nccl_comm is not None:
            ctx.call("sdxl_unet_load_broadcast", ctx.lib.sdxl_unet_load_broadcast, ctx.h, C.byref(cs), None if pack is None else pack.data_ptr(),
                     0 if pack is None else pack.numel(), int(on_device), nccl_comm, rank, root, C.byref(h))
        else:
            ctx.call("sdxl_unet_load", ctx.lib.sdxl_unet_load, ctx.h, C.byref(cs), pack.data_ptr(), pack.numel(), int(on_device), C.byref(h))
        self.h = h
        self._cond_key = None
        self._keep = None
        self._attached: Dict[str, list] = {}   # kind -> the AttachableModels the UNet holds (_attach)

    def _attach(self, kind: str, objects: Sequence["AttachableModel"]) -> None:
        """Records, after a successful set call, the models the UNet now holds for `kind` ("controls", "image_prompts",
        "t2i_adapters"; [] after a detach): the ones held before are released, the new ones cannot be closed while held."""
        for o in self._attached.get(kind, []):
            o.attached -= 1
        self._attached[kind] = list(objects)
        for o in self._attached[kind]:
            o.attached += 1

    def close(self) -> None:
        if getattr(self, "h", None):
            self.ctx.lib.sdxl_unet_destroy(self.h)
            self.h = None
            for kind in list(self._attached):   # the destroyed UNet no longer holds its models
                self._attach(kind, [])

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_adapters(self, adapters: Sequence) -> None:
        """Replaces the active LoRA set with [(adapter, scale), ...] (sdxl_unet_set_adapters); [] restores the loaded weights."""
        set_adapters(self.ctx, self.ctx.lib.sdxl_unet_set_adapters, self.h, adapters, "sdxl_unet_set_adapters")

    def set_controls(self, controls: Sequence) -> None:
        """Replaces the attached ControlNets with [(ControlNet, hint, scale), ...] (sdxl_unet_set_controls); [] detaches.
        hint: f32 [n, 3, H, W] in [0, 1] or u8 [n, H, W, 3]; image b of a batch uses hint b % n."""
        from .controlnet import set_controls
        set_controls(self, controls)

    def set_image_prompt(self, adapter, embeds=None, scale=1.0, negative=None) -> None:
        """Attaches an IP-Adapter image prompt (sdxl_unet_set_image_prompt); adapter None detaches. embeds: f32 [n_batch, D] or
        [n_batch, n_images, D] (CLIP vision image_embeds); image b of a batch uses prompt b % n_batch. scale: float, or one per
        transformer block in execution order (ip_adapter.transformer_block_paths). negative: the CFG rows' embeddings (zeros).
        IP-Adapter Plus: embeds and negative (required) are vision hidden states [n_batch, n_images, L, D] (IPAdapter.image_embeds)."""
        from .ip_adapter import set_image_prompt
        set_image_prompt(self, adapter, embeds, scale, negative)

    def set_image_prompts(self, prompts: Sequence) -> None:
        """Replaces the attached image prompts with [(adapter, embeds, scale, negative, mask), ...] (sdxl_unet_set_image_prompts,
        DESIGN.md §13); [] detaches. Up to four prompts of any adapters; mask None or [n_images, H, W] limits each image of the prompt
        to its region (binarised at 0.5)."""
        from .ip_adapter import set_image_prompts
        set_image_prompts(self, prompts)

    def set_t2i_adapters(self, adapters: Sequence, t_min: int = 0) -> None:
        """Replaces the attached T2I-Adapters with [(T2IAdapter, hint, scale), ...] (sdxl_unet_set_t2i_adapters); [] detaches.
        hint: u8 [n, H, W, C] or f32 [n, C, H, W] in [0, 1], H and W multiples of 32; image b of a batch uses hint b % n. The features
        are added at timesteps t >= t_min (t2i_adapter.t2i_t_min maps diffusers' adapter_conditioning_factor)."""
        from .t2i_adapter import set_t2i_adapters
        set_t2i_adapters(self, adapters, t_min)

    def set_inpaint_condition(self, cond: Optional[torch.Tensor]) -> None:
        """Attaches the inpainting UNet's condition (sdxl_unet_set_inpaint_condition); None detaches. cond: f32
        [n, in_channels - out_channels, h, w] (pipeline.prepare_inpaint_condition): the mask (1 = repaint), then the masked image's
        latent; image b of a batch uses row b % n, at every step until it is replaced or detached."""
        ctx = self.ctx
        s = None
        if cond is not None:
            if cond.dim() != 4:
                raise SdxlError(f"inpainting condition must be f32 [n, C, h, w], got {tuple(cond.shape)}")
            if self.cfg.is_inpaint and cond.shape[1] != self.cfg.in_channels - self.cfg.out_channels:
                raise SdxlError(f"inpainting condition must have {self.cfg.in_channels - self.cfg.out_channels} channels, got "
                                f"{tuple(cond.shape)}")
            cond = cond.to(ctx.device, torch.float32).contiguous()
            s = _lib.InpaintCondition()
            s.cond, s.on_host, s.n = cond.data_ptr(), 0, cond.shape[0]
            s.height, s.width = 8 * cond.shape[2], 8 * cond.shape[3]
        ctx.call("sdxl_unet_set_inpaint_condition", ctx.lib.sdxl_unet_set_inpaint_condition, self.h, None if s is None else C.byref(s))

    def set_edit_image(self, latent: Optional[torch.Tensor], image_guidance: float = 1.5) -> None:
        """Attaches the edit UNet's source image (sdxl_unet_set_edit_image, DESIGN.md §21); None detaches. latent: f32
        [n, out_channels, h, w] (pipeline.prepare_edit_latent), image b of a batch uses row b % n; image_guidance: diffusers'
        image_guidance_scale. The sampling loops with CFG then run [cond | img | uncond] and guide with
        (u + s * (c - i)) + image_guidance * (i - u)."""
        ctx = self.ctx
        s = None
        if latent is not None:
            if latent.dim() != 4 or latent.shape[1] != self.cfg.out_channels:
                raise SdxlError(f"edit image latent must be f32 [n, {self.cfg.out_channels}, h, w], got {tuple(latent.shape)}")
            latent = latent.to(ctx.device, torch.float32).contiguous()
            s = _lib.EditImage()
            s.latent, s.on_host, s.n = latent.data_ptr(), 0, latent.shape[0]
            s.height, s.width, s.image_guidance = 8 * latent.shape[2], 8 * latent.shape[3], float(image_guidance)
        ctx.call("sdxl_unet_set_edit_image", ctx.lib.sdxl_unet_set_edit_image, self.h, None if s is None else C.byref(s))

    def set_pag(self, layers="mid", scale: float = 3.0, adaptive_scale: float = 0.0) -> None:
        """Attaches perturbed-attention guidance (sdxl_unet_set_pag, DESIGN.md §14); layers None or scale 0 detaches. layers: diffusers'
        pag_applied_layers, one regular expression or a list (pag.layer_mask); the sampler then runs the row groups [cond | uncond |
        perturbed] and adds scale * (cond - perturbed) to the guided noise (adaptive_scale: diffusers' pag_adaptive_scale)."""
        if layers is None or scale == 0:
            self._pag = None
            self._set_pag(None)
            return
        from .pag import layer_mask
        mask = layer_mask(self.cfg, layers)
        self._set_pag((mask, float(scale), float(adaptive_scale), 0))
        self._pag = (mask, float(scale), float(adaptive_scale))

    def _set_pag(self, p) -> None:
        s, keep = None, None
        if p is not None:
            mask, scale, adaptive, rows = p
            keep = (C.c_uint8 * len(mask))(*mask)
            s = _lib.Pag()
            s.scale, s.adaptive_scale, s.n_layers, s.layers_host, s.forward_perturbed_rows = scale, adaptive, len(mask), C.addressof(keep), rows
        self.ctx.call("sdxl_unet_set_pag", self.ctx.lib.sdxl_unet_set_pag, self.h, None if s is None else C.byref(s))

    def set_freeu(self, s1: Optional[float], s2: Optional[float] = None, b1: Optional[float] = None, b2: Optional[float] = None) -> None:
        """Attaches FreeU (sdxl_unet_set_freeu, DESIGN.md §15), diffusers' enable_freeu(s1, s2, b1, b2): in the output blocks of the
        two deepest levels the first half of the backbone channels is scaled by b1 (deepest) / b2 and the skip's lowest frequencies
        by s1 / s2. s1 None, or any value 0, detaches (diffusers' disable_freeu). The FreeU authors recommend
        set_freeu(0.9, 0.2, 1.3, 1.4) for SDXL."""
        s = None
        if s1 is not None:
            if s2 is None or b1 is None or b2 is None:
                raise SdxlError("set_freeu: give all four values s1, s2, b1, b2, or None to detach")
            s = _lib.Freeu()
            s.s1, s.s2, s.b1, s.b2 = float(s1), float(s2), float(b1), float(b2)
        self.ctx.call("sdxl_unet_set_freeu", self.ctx.lib.sdxl_unet_set_freeu, self.h, None if s is None else C.byref(s))

    def set_deepcache(self, interval: Optional[int], branch: int = 0) -> None:
        """Attaches DeepCache (sdxl_unet_set_deepcache, DESIGN.md §17; Ma et al. 2024, uniform schedule): every sampling call runs the
        whole UNet on its first step and every interval-th one after it, and on the steps between only the shallow branch (the first
        conv and input blocks 1..branch, then the last branch + 1 output blocks and the head) on the deep feature the last full step
        kept. The count is of UNet evaluations: a Heun or DPM2 step at interval 2 runs one full and one cached evaluation (DESIGN.md
        §20). interval None detaches. Direct unet_forward calls run the full forward unless unet_forward(cached=True)."""
        if interval is None:
            self._deepcache = None
            self._set_deepcache(None)
            return
        self._set_deepcache((int(interval), int(branch), 0))
        self._deepcache = (int(interval), int(branch))

    def _set_deepcache(self, d) -> None:
        s = None
        if d is not None:
            s = _lib.Deepcache()
            s.interval, s.branch, s.forward_cached = d
        self.ctx.call("sdxl_unet_set_deepcache", self.ctx.lib.sdxl_unet_set_deepcache, self.h, None if s is None else C.byref(s))

    def set_prediction(self, prediction: str = "epsilon", guidance_rescale: float = 0.0, zero_terminal_snr: bool = False,
                       alphas=None) -> None:
        """What the sampling loops read the UNet's output as (sdxl_unet_set_prediction, DESIGN.md §18): diffusers' prediction_type
        ("epsilon" or "v_prediction"), guidance_rescale (phi in [0, 1], diffusers' pipeline argument; calls with CFG rows only) and the
        noise table: alphas (f64 [cfg.n_steps]) if given, else with zero_terminal_snr schedulers.alphas_cumprod(cfg.n_steps,
        zero_terminal_snr=True), else the loaded table. The default arguments detach: epsilon, phi 0 and the loaded table."""
        if prediction not in _lib.PREDICTIONS:
            raise SdxlError(f"set_prediction: prediction = {prediction!r} is not one of {sorted(_lib.PREDICTIONS)}")
        if alphas is None and zero_terminal_snr:
            from .schedulers import alphas_cumprod
            alphas = alphas_cumprod(self.cfg.n_steps, zero_terminal_snr=True)
        self._set_prediction((prediction, float(guidance_rescale), None if alphas is None else np.asarray(alphas, dtype=np.float64)))

    def _set_prediction(self, p) -> None:
        prediction, phi, alphas = p
        s, a = None, None
        if prediction != "epsilon" or phi != 0.0 or alphas is not None:
            s = _lib.Prediction()
            s.type, s.guidance_rescale = _lib.PREDICTIONS[prediction], phi
            if alphas is not None:
                a = np.ascontiguousarray(alphas, dtype=np.float64)
                s.n_alphas, s.alphas_cumprod_host = a.size, a.ctypes.data
        self.ctx.call("sdxl_unet_set_prediction", self.ctx.lib.sdxl_unet_set_prediction, self.h, None if s is None else C.byref(s))
        self._prediction = (prediction, phi, alphas)

    @property
    def prediction(self):
        """(prediction, guidance_rescale, alphas or None) as set_prediction last set them."""
        return getattr(self, "_prediction", ("epsilon", 0.0, None))

    @classmethod
    def from_diffusers_dir(cls, ctx: Context, path: str) -> "Diffuser":
        """A diffusers UNet2DConditionModel directory (the `unet/` folder of an SDXL pipeline: base, inpainting or InstructPix2Pix
        edit): config.json +
        diffusion_pytorch_model[.fp16].safetensors (diffusers_unet.from_diffusers). When the pipeline's scheduler/scheduler_config.json
        sits next to it and says prediction_type "v_prediction" or rescale_betas_zero_snr true, the model is set to that prediction
        and noise table (schedulers.prediction_of_config, set_prediction); prediction_type "sample" and a beta_schedule other than
        "scaled_linear" are refused."""
        import json
        import os
        from .diffusers_unet import from_diffusers, read_model_dir
        from .schedulers import prediction_of_config
        sched = os.path.join(os.path.dirname(os.path.normpath(path)), "scheduler", "scheduler_config.json")
        pred = None
        if os.path.exists(sched):
            with open(sched) as f:
                pred = prediction_of_config(json.load(f))
        d = cls(ctx, *from_diffusers(*read_model_dir(path)))
        if pred is not None:
            try:
                d.set_prediction(**pred)
            except Exception:
                d.close()
                raise
        return d

    # ---- UNet::forward -------------------------------------------------------------------------
    def set_conditioning(self, context: torch.Tensor, label: torch.Tensor) -> None:
        ctx = self.ctx
        context = context.to(ctx.device, torch.float16).contiguous()
        label = label.to(ctx.device, torch.float16).contiguous()
        B, n_ctx, _ = context.shape
        ctx.call("sdxl_unet_set_conditioning", ctx.lib.sdxl_unet_set_conditioning, self.h, B, n_ctx, _ptr(context), _ptr(label))
        self._keep = (context, label)

    def unet_forward(self, x: torch.Tensor, timesteps, context: Optional[torch.Tensor] = None,
                     label: Optional[torch.Tensor] = None, perturbed_rows: Optional[int] = None,
                     cached: Optional[bool] = None) -> torch.Tensor:
        """== UNet::forward(x [B,4,h,w], timesteps Int[1], context [B,77,Cctx], label [B,adm]).
        f32 in -> f32 out (no I/O rounding), f16 in -> f16 out (the reference's tensors). perturbed_rows (PAG attached, set_pag): the
        last this-many rows of the batch run the attached layers' identity self-attention, from this forward on (0: none). cached
        (DeepCache attached, set_deepcache): True runs the cached forward on the feature the last full forward kept, False the full
        forward, from this forward on."""
        ctx = self.ctx
        if cached is not None:
            if getattr(self, "_deepcache", None) is None:
                if cached:
                    raise SdxlError("unet_forward: cached needs DeepCache attached (set_deepcache)")
            else:
                self._set_deepcache((*self._deepcache, int(bool(cached))))
        if perturbed_rows is not None:
            if getattr(self, "_pag", None) is None:
                if perturbed_rows:
                    raise SdxlError("unet_forward: perturbed_rows needs PAG attached (set_pag)")
            else:
                self._set_pag((*self._pag, int(perturbed_rows)))
        if context is not None:
            self.set_conditioning(context, label)
        t = float(timesteps[0]) if hasattr(timesteps, "__len__") else float(timesteps)   # fractional: between two training timesteps
        B, _, h, w = x.shape
        # convert first, then enter: the ctx stream must wait for the cast / copy kernels torch queues on its own stream
        f16 = x.dtype == torch.float16
        x = x.to(ctx.device, torch.float16 if f16 else torch.float32).contiguous()
        out = torch.empty_like(x)
        if f16:
            if t != int(t):
                raise SdxlError(f"unet_forward: a fractional timestep ({t}) needs an f32 latent")
            ctx.call("sdxl_unet_forward", ctx.lib.sdxl_unet_forward, self.h, B, h, w, _ptr(x), int(t), _ptr(out))
        else:
            ctx.call("sdxl_unet_forward_f32_at", ctx.lib.sdxl_unet_forward_f32_at, self.h, B, h, w, _ptr(x), t, _ptr(out))
        return out

    @property
    def plan_flops(self) -> float:
        return float(self.ctx.lib.sdxl_unet_plan_flops(self.h))

    @property
    def plan_flops_executed(self) -> float:
        return float(self.ctx.lib.sdxl_unet_plan_flops_executed(self.h))

    @property
    def plan_num_ops(self) -> int:
        return int(self.ctx.lib.sdxl_unet_plan_num_ops(self.h))

    KIND_NAMES = ["igemm_wgmma", "attention_wgmma", "group_norm", "layer_norm", "gemv", "timestep_embedding",
                  "conv_in", "upsample2x", "phase_split", "cast_f16"]
    # kinds only the UNet plan launches, by kind index (KIND_NAMES is positional and LatentDecoder.KIND_NAMES extends it)
    UNET_KINDS = {17: "t2i_add", 18: "pag_identity", 19: "freeu", 20: "copy"}

    def profile_plan(self) -> Dict[str, Dict[str, float]]:
        """Per-kernel-kind device time (ms), algorithmic FLOPs and launch count of one plan execution."""
        ms, fl, ln = (C.c_double * _lib.PROFILE_KINDS)(), (C.c_double * _lib.PROFILE_KINDS)(), (C.c_int * _lib.PROFILE_KINDS)()
        self.ctx.check(self.ctx.lib.sdxl_unet_profile_plan(self.h, ms, fl, ln), "sdxl_unet_profile_plan")
        kinds = list(enumerate(self.KIND_NAMES)) + list(self.UNET_KINDS.items())
        return {n: {"ms": ms[i], "flops": fl[i], "launches": ln[i]} for i, n in kinds if ln[i]}

    def profile_dump(self, path: str) -> None:
        self.ctx.check(self.ctx.lib.sdxl_unet_profile_dump(self.h, path.encode()), "sdxl_unet_profile_dump")

    def alpha(self, i: int) -> float:
        return float(self.ctx.lib.sdxl_unet_alpha(self.h, i))

    # ---- Diffuser::* ---------------------------------------------------------------------------
    def _sample(self, cond: Conditioning, guidance: float, n_steps: int, step_start: int,
                init_latent: Optional[torch.Tensor], noise: Optional[torch.Tensor], seed: int,
                ref: Optional[torch.Tensor], mask: Optional[torch.Tensor], host: bool = False, schedule=None) -> torch.Tensor:
        """schedule (schedulers.Schedule): sdxl_sample_latent_scheduled with its sampler and spacing; n_steps and step_start are
        then unused (the schedule carries them). None: sdxl_sample_latent's DDIM loop."""
        ctx = self.ctx
        s, keep = cond.to_struct(None if host else ctx.device)
        h, w = cond.resolution[0] // 8, cond.resolution[1] // 8
        dev = torch.device("cpu") if host else ctx.device

        def prep(t, dt):
            return None if t is None else t.to(dev, dt).contiguous()
        init_latent = prep(init_latent, torch.float32)
        noise = prep(noise, torch.float32)
        ref = prep(ref, torch.float32)
        mask = prep(mask, torch.uint8)
        n_noise = 0 if noise is None else (noise.shape[0] if noise.dim() == 5 else 1)
        out = torch.empty(s.n_batch, self.cfg.latent_channels, h, w, device=dev, dtype=torch.float32)
        if schedule is not None:
            sch = schedule.to_struct()
            ctx.call("sdxl_sample_latent_scheduled", ctx.lib.sdxl_sample_latent_scheduled, self.h, C.byref(s), float(guidance), C.byref(sch),
                     _ptr(init_latent), _ptr(noise), n_noise, seed, _ptr(ref), _ptr(mask), _ptr(out))
        else:
            ctx.call("sdxl_sample_latent", ctx.lib.sdxl_sample_latent, self.h, C.byref(s), float(guidance), n_steps, step_start,
                     _ptr(init_latent), _ptr(noise), n_noise, seed, _ptr(ref), _ptr(mask), _ptr(out))
        del keep
        return out

    def sample_latent(self, conditioning: Conditioning, unconditional_guidance_scale: float, n_steps: int,
                      noise: Optional[torch.Tensor] = None, seed: int = 0, host: bool = False, schedule=None,
                      step_noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        """== Diffuser::sample_latent (mod.rs:317-332). `noise` injects gen_noise()'s tensor (the reference's
        RNG is unseeded libtorch Philox; parity tests inject it). schedule (schedulers.Schedule): its sampler, spacing and steps
        instead of n_steps DDIM steps; step_noise [k, n, 4, h, w] then injects the sampler's per-step noise."""
        return self._sample(conditioning, unconditional_guidance_scale, n_steps, 0, noise, step_noise, seed, None, None, host, schedule)

    def sample_latent_with_inpainting(self, conditioning: Conditioning, unconditional_guidance_scale: float,
                                      n_steps: int, reference: torch.Tensor, mask: torch.Tensor,
                                      init_noise: Optional[torch.Tensor] = None,
                                      step_noise: Optional[torch.Tensor] = None, seed: int = 0, schedule=None) -> torch.Tensor:
        """== Diffuser::sample_latent_with_inpainting (mod.rs:334-353); mask True keeps the generated latent. With a schedule the
        blend is xh = mask ? xh : reference + sigma_k z before each forward."""
        return self._sample(conditioning, unconditional_guidance_scale, n_steps, 0, init_noise, step_noise, seed,
                            reference, mask.to(torch.uint8), schedule=schedule)

    def refine_latent(self, latent: torch.Tensor, conditioning: Conditioning, unconditional_guidance_scale: float,
                      step_start: int, n_steps: int, noise: Optional[torch.Tensor] = None, seed: int = 0, schedule=None) -> torch.Tensor:
        """== Diffuser::refine_latent (mod.rs:355-376). With a schedule its first_step / renoise say where the latent enters."""
        return self._sample(conditioning, unconditional_guidance_scale, n_steps, step_start, latent, noise, seed, None, None,
                            schedule=schedule)

    # ---- step-wise (bench) ---------------------------------------------------------------------
    def sampler_begin(self, cond: Conditioning, guidance: float) -> None:
        s, keep = cond.to_struct(self.ctx.device)
        self.ctx.call("sdxl_sampler_begin", self.ctx.lib.sdxl_sampler_begin, self.h, C.byref(s), float(guidance))
        self.ctx.synchronize()
        del keep

    def sampler_set_latent(self, x: torch.Tensor) -> None:
        x = x.to(self.ctx.device, torch.float32).contiguous()
        self.ctx.call("sdxl_sampler_set_latent", self.ctx.lib.sdxl_sampler_set_latent, self.h, _ptr(x), 0)
        self.ctx.synchronize()

    def sampler_get_latent(self, like: torch.Tensor) -> torch.Tensor:
        out = torch.empty_like(like, dtype=torch.float32, device=self.ctx.device)
        self.ctx.check(self.ctx.lib.sdxl_sampler_get_latent(self.h, _ptr(out), 0), "sdxl_sampler_get_latent")
        self.ctx.synchronize()
        return out

    def sampler_step(self, t: int, t_prev: int) -> None:
        self.ctx.check(self.ctx.lib.sdxl_sampler_step(self.h, t, t_prev), "sdxl_sampler_step")

    def sampler_step_host(self, t: int, t_prev: int, latent_host: torch.Tensor) -> None:
        assert latent_host.device.type == "cpu" and latent_host.dtype == torch.float32 and latent_host.is_contiguous()
        self.ctx.check(self.ctx.lib.sdxl_sampler_step_host(self.h, t, t_prev, latent_host.data_ptr()),
                       "sdxl_sampler_step_host")


class LatentDecoder:
    """Mirror of the reference's LatentDecoder (decode half): `decode_latent` and `latent_to_image`
    (src/model/stablediffusion/mod.rs:199-237, 263-266) over the device-resident VAE decoder."""

    KIND_NAMES = Diffuser.KIND_NAMES + ["softmax_rows", "transpose_f16", "post_quant"]

    def __init__(self, ctx: Context, cfg: VaeConfig, weights):
        self.ctx, self.cfg = ctx, cfg
        pack = weights if isinstance(weights, torch.Tensor) else build_pack(weights)
        on_device = pack.is_cuda
        if on_device:
            torch.cuda.current_stream(ctx.device).synchronize()
        cs = _lib.VaeCfg()
        cs.latent_channels, cs.n_blocks, cs.n_group = cfg.latent_channels, len(cfg.block_channels), cfg.n_group
        cs.scale_factor = cfg.scale_factor
        for i, (ci, co) in enumerate(cfg.block_channels):
            cs.block_in[i], cs.block_out[i] = ci, co
        cs.n_enc_blocks, cs.enc_z_channels = len(cfg.enc_block_channels), cfg.enc_z_channels
        for i, (ci, co) in enumerate(cfg.enc_block_channels):
            cs.enc_in[i], cs.enc_out[i] = ci, co
        h = C.c_void_p()
        ctx.call("sdxl_vae_load", ctx.lib.sdxl_vae_load, ctx.h, C.byref(cs), pack.data_ptr(), pack.numel(), int(on_device), C.byref(h))
        self.h = h

    def close(self) -> None:
        if getattr(self, "h", None):
            self.ctx.lib.sdxl_vae_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _prep(self, latent: torch.Tensor):
        host = not latent.is_cuda
        latent = latent.to(torch.float32).contiguous()
        B, _, h, w = latent.shape
        up = self.cfg.upscale
        return latent, host, B, h, w, up

    def decode_latent(self, latent: torch.Tensor) -> torch.Tensor:
        """latent f32 [B,4,h,w] (host or device) -> image f32 [B,3,8h,8w] on the same side."""
        latent, host, B, h, w, up = self._prep(latent)
        out = torch.empty((B, 3, h * up, w * up), dtype=torch.float32, device="cpu" if host else self.ctx.device)
        self.ctx.call("sdxl_vae_decode_latent", self.ctx.lib.sdxl_vae_decode_latent, self.h, B, h, w, _ptr(latent), int(host), _ptr(out))
        return out

    def latent_to_image(self, latent: torch.Tensor) -> torch.Tensor:
        """RawImages buffer: u8 [B, 8h, 8w, 3]."""
        latent, host, B, h, w, up = self._prep(latent)
        out = torch.empty((B, h * up, w * up, 3), dtype=torch.uint8, device="cpu" if host else self.ctx.device)
        self.ctx.call("sdxl_vae_latent_to_image", self.ctx.lib.sdxl_vae_latent_to_image, self.h, B, h, w, _ptr(latent), int(host), _ptr(out))
        return out

    def encode_image(self, image: torch.Tensor) -> torch.Tensor:
        """== LatentDecoder::encode_image: image f32 [B,3,H,W] in [-1,1] (host or device) -> latent f32 [B,4,H/8,W/8]."""
        host = not image.is_cuda
        image = image.to(torch.float32).contiguous()
        B, _, H, W = image.shape
        d = 2 ** (len(self.cfg.enc_block_channels) - 1)
        out = torch.empty((B, self.cfg.latent_channels, H // d, W // d), dtype=torch.float32, device="cpu" if host else self.ctx.device)
        self.ctx.call("sdxl_vae_encode_image", self.ctx.lib.sdxl_vae_encode_image, self.h, B, H, W, _ptr(image), int(host), _ptr(out))
        return out

    def image_to_latent(self, rgb: torch.Tensor) -> torch.Tensor:
        """== LatentDecoder::image_to_latent: RawImages u8 [B,H,W,3] -> latent f32 [B,4,H/8,W/8]."""
        host = not rgb.is_cuda
        rgb = rgb.to(torch.uint8).contiguous()
        B, H, W, _ = rgb.shape
        d = 2 ** (len(self.cfg.enc_block_channels) - 1)
        out = torch.empty((B, self.cfg.latent_channels, H // d, W // d), dtype=torch.float32, device="cpu" if host else self.ctx.device)
        self.ctx.call("sdxl_vae_image_to_latent", self.ctx.lib.sdxl_vae_image_to_latent, self.h, B, H, W, _ptr(rgb), int(host), _ptr(out))
        return out

    @property
    def encode_plan_flops(self) -> float:
        return float(self.ctx.lib.sdxl_vae_encode_plan_flops(self.h))

    @property
    def plan_flops(self) -> float:
        return float(self.ctx.lib.sdxl_vae_plan_flops(self.h))

    def profile_plan(self) -> Dict[str, Dict[str, float]]:
        ms, fl, ln = (C.c_double * _lib.PROFILE_KINDS)(), (C.c_double * _lib.PROFILE_KINDS)(), (C.c_int * _lib.PROFILE_KINDS)()
        self.ctx.check(self.ctx.lib.sdxl_vae_profile_plan(self.h, ms, fl, ln), "sdxl_vae_profile_plan")
        return {n: {"ms": ms[i], "flops": fl[i], "launches": ln[i]} for i, n in enumerate(self.KIND_NAMES) if ln[i]}

    def profile_dump(self, path: str) -> None:
        self.ctx.check(self.ctx.lib.sdxl_vae_profile_dump(self.h, path.encode()), "sdxl_vae_profile_dump")


def ddim_timesteps(n_steps: int, step_start: int = 0, total: int = 1000) -> List[int]:
    """(0..total-step_start).rev().step_by(total / n_steps)  (reference mod.rs:400-406)."""
    step = total // n_steps
    return list(range(total - step_start - 1, -1, -step))
