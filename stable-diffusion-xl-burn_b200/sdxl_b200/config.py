"""Model configurations (mirror of the reference's DiffuserConfig / UNetConfig).

reference: src/model/stablediffusion/mod.rs:269-306 (DiffuserConfig), src/model/unet/mod.rs:59-69
(UNetConfig). The `.cfg` JSON files live on HuggingFace, not in the reference repo; the values below
are the ones SURVEY.md section 5 derives from the code and dump scripts.
"""
from __future__ import annotations

from dataclasses import dataclass, field, replace
from typing import List, Tuple


@dataclass(frozen=True)
class UNetConfig:
    adm_in_channels: int
    model_channels: int
    channel_mults: Tuple[int, ...]
    transformer_depths: Tuple[int, ...]
    context_dim: int
    is_refiner: bool = False
    in_channels: int = 4
    out_channels: int = 4
    n_head_channels: int = 64
    n_steps: int = 1000
    is_edit: bool = False   # the instruction-editing layout (DESIGN.md §21): in_channels = 2 * out_channels, the second half attached

    @property
    def n_levels(self) -> int:
        return len(self.channel_mults)

    @property
    def time_embed_dim(self) -> int:
        return 4 * self.model_channels

    @property
    def is_inpaint(self) -> bool:
        """The inpainting layout (DESIGN.md §12): the first conv reads the latent, a mask and the masked image's latent."""
        return self.in_channels > 8 and self.in_channels == 2 * self.out_channels + 1

    @property
    def latent_channels(self) -> int:
        """Channels of the latent the forward and the sampler take (the rest of an inpainting or edit UNet's input is attached)."""
        return self.out_channels if self.is_inpaint or self.is_edit else self.in_channels


# SDXL base: diffuser.cfg
SDXL_BASE = UNetConfig(adm_in_channels=2816, model_channels=320, channel_mults=(1, 2, 4),
                       transformer_depths=(0, 2, 10), context_dim=2048, is_refiner=False)
# SDXL refiner: refiner.cfg (middle depth = transformer_depths[-1] = 4, inferred; SURVEY 3.2)
SDXL_REFINER = UNetConfig(adm_in_channels=2560, model_channels=384, channel_mults=(1, 2, 4, 4),
                          transformer_depths=(0, 4, 4, 4), context_dim=1280, is_refiner=True)
# Tiny config for known-answer tests (the reference's `test_tiny_unet` probe method,
# src/bin/test/main.rs:128-140): same topology rules (transformers on levels 1 and 2, head dim 64).
TINY = UNetConfig(adm_in_channels=8, model_channels=64, channel_mults=(1, 2, 4),
                  transformer_depths=(0, 1, 2), context_dim=24, is_refiner=False)
TINY_REFINER = UNetConfig(adm_in_channels=16, model_channels=64, channel_mults=(1, 2, 4),
                          transformer_depths=(0, 1, 1), context_dim=40, is_refiner=True)
# The inpainting UNet (diffusers stable-diffusion-xl-1.0-inpainting-0.1): SDXL base with the latent, the mask and the masked image's
# latent as input (4 + 1 + 4 channels), and its tiny counterpart.
SDXL_INPAINT = replace(SDXL_BASE, in_channels=9)
TINY_INPAINT = replace(TINY, in_channels=9)
# The instruction-editing UNet (diffusers/sdxl-instructpix2pix-768): SDXL base with the latent and the source image's latent as input
# (4 + 4 channels), and its tiny counterpart.
SDXL_EDIT = replace(SDXL_BASE, in_channels=8, is_edit=True)
TINY_EDIT = replace(TINY, in_channels=8, is_edit=True)


@dataclass(frozen=True)
class ControlNetConfig:
    """An SDXL ControlNet (DESIGN.md §8): the encoder half of `unet` (which must match the UNet it is attached to) plus the hint
    encoder: conv(hint_in -> c0), then per level conv(c_k -> c_k), conv(c_k -> c_k+1, stride 2), then conv(c_last -> mc)
    (diffusers' conditioning_embedding_out_channels)."""
    unet: UNetConfig
    hint_in_channels: int = 3
    hint_block_channels: Tuple[int, ...] = (16, 32, 96, 256)


SDXL_CONTROLNET = ControlNetConfig(SDXL_BASE)
TINY_CONTROLNET = ControlNetConfig(TINY, hint_block_channels=(8, 16, 24, 32))


@dataclass(frozen=True)
class T2IAdapterConfig:
    """An SDXL T2I-Adapter (DESIGN.md §11, diffusers FullAdapterXL) for `unet`, which must be SDXL-base-shaped and match the UNet it is
    attached to. Its four feature widths follow from the UNet's."""
    unet: UNetConfig
    in_channels: int = 3
    n_res_blocks: int = 2

    @property
    def channels(self) -> Tuple[int, int, int, int]:
        mc, m = self.unet.model_channels, self.unet.channel_mults
        return (mc * m[0], mc * m[1], mc * m[2], mc * m[2])


SDXL_T2I_ADAPTER = T2IAdapterConfig(SDXL_BASE)
TINY_T2I_ADAPTER = T2IAdapterConfig(TINY)


@dataclass(frozen=True)
class VaeConfig:
    """Decoder half of AutoencoderConfig (reference src/model/autoencoder/mod.rs:28-45: the widths are hard-coded
    there; parameters here so a small instance can be tested) + LatentDecoder.scale_factor."""
    block_channels: Tuple[Tuple[int, int], ...]
    latent_channels: int = 4
    n_group: int = 32
    scale_factor: float = 0.13025
    enc_block_channels: Tuple[Tuple[int, int], ...] = ()   # EncoderConfig channels; () = decoder only
    enc_z_channels: int = 8

    @property
    def upscale(self) -> int:
        return 2 ** (len(self.block_channels) - 1)


# SDXL VAE decoder: DecoderConfig::new(vec![(512,512),(512,512),(512,256),(256,128)], 32)
# and EncoderConfig::new(vec![(128,128),(128,256),(256,512),(512,512)], 32, 8)
SDXL_VAE = VaeConfig(block_channels=((512, 512), (512, 512), (512, 256), (256, 128)),
                     enc_block_channels=((128, 128), (128, 256), (256, 512), (512, 512)))
# small instance with the same topology rules (3 ResnetBlocks per level, nin_shortcut where widths change)
TINY_VAE = VaeConfig(block_channels=((128, 128), (128, 64), (64, 64)), enc_block_channels=((64, 64), (64, 128), (128, 128)))


@dataclass(frozen=True)
class ClipConfig:
    """== CLIPConfig (reference src/model/clip/mod.rs:18-26)."""
    n_vocab: int
    n_state: int
    embed_dim: int
    n_head: int
    n_ctx: int
    n_layer: int
    quick_gelu: bool


# SDXL's two text encoders (SURVEY.md §8(f): CLIP ViT-L/14 text tower, OpenCLIP ViT-bigG/14 text tower)
SDXL_CLIP_L = ClipConfig(n_vocab=49408, n_state=768, embed_dim=768, n_head=12, n_ctx=77, n_layer=12, quick_gelu=True)
SDXL_OPEN_CLIP_G = ClipConfig(n_vocab=49408, n_state=1280, embed_dim=1280, n_head=20, n_ctx=77, n_layer=32, quick_gelu=False)
# small instances for known-answer tests (vocabulary sized for tests/golden/mini_bpe plus the hard-coded 49406/49407)
TINY_CLIP = ClipConfig(n_vocab=49408, n_state=128, embed_dim=128, n_head=2, n_ctx=77, n_layer=3, quick_gelu=True)
TINY_OPEN_CLIP = ClipConfig(n_vocab=49408, n_state=192, embed_dim=64, n_head=3, n_ctx=77, n_layer=4, quick_gelu=False)


@dataclass
class BlockSpec:
    kind: str              # conv | resnet | downsample | resnet_transformer | resnet_transformer_upsample | resnet_upsample
    path: str
    c_in: int
    c_out: int
    depth: int = 0         # transformer depth
    n_head: int = 0


def block_program(cfg: UNetConfig) -> Tuple[List[BlockSpec], BlockSpec, List[BlockSpec]]:
    """Input / middle / output block lists exactly as UNetConfig::init builds them
    (reference src/model/unet/mod.rs:115-173, 238-248, 250-328)."""
    mc = cfg.model_channels
    nl = cfg.n_levels
    ins: List[BlockSpec] = [BlockSpec("conv", "input_blocks/0", cfg.in_channels, mc)]
    idx = 1
    for level in range(nl):
        c_in = cfg.channel_mults[max(level - 1, 0)] * mc
        c_out = cfg.channel_mults[level] * mc
        tr = level in (1, 2)
        for k in range(2):
            ci = c_in if k == 0 else c_out
            if tr:
                ins.append(BlockSpec("resnet_transformer", f"input_blocks/{idx}", ci, c_out,
                                     cfg.transformer_depths[level], c_out // cfg.n_head_channels))
            else:
                ins.append(BlockSpec("resnet", f"input_blocks/{idx}", ci, c_out))
            idx += 1
        if level != nl - 1:
            ins.append(BlockSpec("downsample", f"input_blocks/{idx}", c_out, c_out))
            idx += 1
    cm = cfg.channel_mults[-1] * mc
    mid = BlockSpec("middle", "middle_block", cm, cm, cfg.transformer_depths[-1], cm // cfg.n_head_channels)
    outs: List[BlockSpec] = []
    idx = 0
    for level in reversed(range(nl)):
        next_level = level + 1 if level != nl - 1 else level
        c_out = cfg.channel_mults[level] * mc
        cins = (cfg.channel_mults[next_level] * mc + c_out, 2 * c_out,
                c_out + cfg.channel_mults[max(level - 1, 0)] * mc)
        tr = level in (1, 2)
        for k in range(3):
            up = k == 2 and (tr or level != 0)
            if tr:
                kind = "resnet_transformer_upsample" if up else "resnet_transformer"
                outs.append(BlockSpec(kind, f"output_blocks/{idx}", cins[k], c_out,
                                      cfg.transformer_depths[level], c_out // cfg.n_head_channels))
            else:
                outs.append(BlockSpec("resnet_upsample" if up else "resnet", f"output_blocks/{idx}", cins[k], c_out))
            idx += 1
    return ins, mid, outs
