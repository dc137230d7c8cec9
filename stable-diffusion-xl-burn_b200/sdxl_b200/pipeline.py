"""The `sample` binary's flow (reference src/bin/sample/main.rs:128-285) over the library: crop window -> inpainting mask,
text -> conditioning -> base sampling (plain or inpainting) -> optional refiner hand-off -> latent -> image."""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib

REFINER_STEP_START = 800   # main.rs:263: the refiner re-noises to t0 = 1000 - 800 and runs the remaining iterations


def make_inpaint_mask(img_hw: Tuple[int, int], latent_hw: Tuple[int, int], crop_left: Optional[int] = None, crop_right: Optional[int] = None,
                      crop_top: Optional[int] = None, crop_bottom: Optional[int] = None, crop_out: bool = False, n_channels: int = 4) -> torch.Tensor:
    """== main.rs:144-190 (sdxl_make_inpaint_mask). Returns Bool [1, n_channels, h, w]; True keeps the generated latent."""
    lib = _lib.load()
    (ih, iw), (lh, lw) = img_hw, latent_hw
    out = np.empty((n_channels, lh, lw), dtype=np.uint8)
    opt = lambda v: -1 if v is None else int(v)  # noqa: E731
    rc = lib.sdxl_make_inpaint_mask(iw, ih, lw, lh, opt(crop_left), opt(crop_right), opt(crop_top), opt(crop_bottom), int(crop_out), n_channels, out.ctypes.data)
    if rc != 0:
        raise _lib.SdxlError(f"sdxl_make_inpaint_mask failed with {rc}: invalid crop parameters")
    return torch.from_numpy(out).bool().unsqueeze(0)


def prepare_inpaint_condition(decoder, rgb: torch.Tensor, pixel_mask: torch.Tensor) -> torch.Tensor:
    """The inpainting UNet's condition (Diffuser.set_inpaint_condition) of images rgb u8 [n, H, W, 3] and pixel_mask bool [n, 1, H, W]
    (True = repaint), as diffusers' StableDiffusionXLInpaintPipeline.prepare_mask_latents builds it: the image normalised to [-1, 1],
    masked = image * (mask < 0.5), the masked image's latent decoder.encode_image(masked) and the mask channel F.interpolate(mask,
    (H/8, W/8)) (nearest: mask[8i, 8j]; the latent's extent for a VAE with another factor). Returns f32 [n, 1 + latent_channels,
    H/8, W/8] on the decoder's device.
    One difference: diffusers samples the VAE posterior with the call's generator, this engine's encoder returns its mean (as the
    reference's does), so the masked latent is deterministic."""
    import torch.nn.functional as F
    from ._lib import SdxlError
    if rgb.dim() != 4 or rgb.shape[3] != 3 or rgb.dtype != torch.uint8:
        raise SdxlError(f"inpainting image must be u8 [n, H, W, 3], got {rgb.dtype} {tuple(rgb.shape)}")
    n, H, W, _ = rgb.shape
    if tuple(pixel_mask.shape) != (n, 1, H, W):
        raise SdxlError(f"inpainting mask must be [{n}, 1, {H}, {W}], got {tuple(pixel_mask.shape)}")
    dev = decoder.ctx.device
    image = rgb.to(dev).permute(0, 3, 1, 2).to(torch.float32) / 255.0 * 2.0 - 1.0
    mask = pixel_mask.to(dev).to(torch.float32)
    masked = image * (mask < 0.5)
    masked_lat = decoder.encode_image(masked.contiguous())
    mask_lat = F.interpolate(mask, size=tuple(masked_lat.shape[2:]))   # the latent's extent: H/8 x W/8 for the SDXL VAE
    return torch.cat([mask_lat, masked_lat], dim=1)


def prepare_edit_latent(decoder, rgb: torch.Tensor, size: Optional[Tuple[int, int]] = None) -> torch.Tensor:
    """The edit UNet's source latent (Diffuser.set_edit_image) of images rgb u8 [n, H, W, 3], as diffusers'
    StableDiffusionXLInstructPix2PixPipeline.prepare_image_latents makes it: the image (resized bilinearly to size = (height, width)
    when given and different) mapped to [-1, 1] and encoded to the VAE posterior mean (retrieve_latents(..., sample_mode="argmax")),
    without the VAE scaling factor: decoder.encode_image's scaled latent divided by it again. Returns f32 [n, latent_channels, H/8, W/8]
    on the decoder's device."""
    import torch.nn.functional as F
    from ._lib import SdxlError
    if rgb.dim() != 4 or rgb.shape[3] != 3 or rgb.dtype != torch.uint8:
        raise SdxlError(f"edit image must be u8 [n, H, W, 3], got {rgb.dtype} {tuple(rgb.shape)}")
    image = rgb.to(decoder.ctx.device).permute(0, 3, 1, 2).to(torch.float32) / 255.0 * 2.0 - 1.0
    if size is not None and tuple(size) != tuple(image.shape[2:]):
        image = F.interpolate(image, size=(int(size[0]), int(size[1])), mode="bilinear", align_corners=False)
    return decoder.encode_image(image.contiguous()) / decoder.cfg.scale_factor


def sample(embedder, diffuser, decoder, prompt: str, guidance: float = 7.5, n_steps: int = 30, refiner=None,
           reference_rgb: Optional[torch.Tensor] = None, crop: Sequence[Optional[int]] = (None, None, None, None), crop_out: bool = False,
           resolution: Tuple[int, int] = (1024, 1024), seed: int = 0, noise: Optional[torch.Tensor] = None,
           loras: Optional[Sequence] = None, controls: Optional[Sequence] = None, image_prompt: Optional[Sequence] = None,
           t2i_adapters: Optional[Sequence] = None, t2i_factor: float = 1.0, pag: Optional[Sequence] = None,
           freeu: Optional[Sequence[float]] = None, sampler: Optional[str] = None, spacing: Optional[str] = None,
           no_cfg: bool = False, deepcache: Optional[Sequence[int]] = None, guidance_rescale: float = 0.0,
           edit_image: Optional[torch.Tensor] = None, image_guidance: float = 1.5) -> torch.Tensor:
    """One image, like `sample --prompt ... [--reference-img ... --crop-* ...] [--use-refiner]`.
    reference_rgb: uint8 [1, H, W, 3] (the reference image: switches to inpainting, main.rs:131-197); crop = (left, right, top,
    bottom) in pixels. With an inpainting UNet (cfg.is_inpaint, DESIGN.md §12) reference_rgb is required: the crop window becomes the
    pixel mask (1 = repaint), prepare_inpaint_condition's condition is attached for the call and the latent is sampled from noise
    without blending. loras: [(adapter .safetensors path / bytes / tensor dict, scale), ...] (any format lora.load_adapter reads) merged into the base UNet and both
    text encoders for this call (the refiner is left alone) and removed again afterwards, which also clears any adapter set
    those models had. controls: [(ControlNet, image u8 [1, H, W, 3] or f32 [1, 3, H, W], scale), ...] attached to the base UNet
    for this call and detached afterwards (the refiner is left alone). image_prompt: (IPAdapter, ClipVisionEncoder, images u8
    [n_images, H, W, 3], scale): the images are encoded (IPAdapter.image_embeds: image_embeds for the base adapter, hidden states for
    IP-Adapter Plus) and attached to the base UNet as one prompt of n_images images for this call and detached afterwards; or a list
    of up to four (IPAdapter, ClipVisionEncoder, images, scale[, mask]) attached together (Diffuser.set_image_prompts; mask None or
    [n_images, H, W] at the output resolution).
    t2i_adapters: [(T2IAdapter, image u8 [1, H, W, C] or f32 [1, C, H, W], scale), ...] attached to the base UNet for this call and
    detached afterwards, their features added on the first int(n_steps * t2i_factor) iterations (diffusers'
    adapter_conditioning_factor). pag: (scale, layers[, adaptive_scale]) perturbed-attention guidance (Diffuser.set_pag, diffusers'
    pag_scale, pag_applied_layers, pag_adaptive_scale) attached to the base UNet for this call and detached afterwards (the refiner is
    left alone). freeu: (s1, s2, b1, b2) FreeU (Diffuser.set_freeu, diffusers' enable_freeu) attached to the base UNet for this call
    and detached afterwards (the refiner is left alone). sampler / spacing (schedulers.ALL_SAMPLERS / SPACINGS; one given, the other
    defaults to "euler" / "leading") and no_cfg (one conditional forward per step, for few-step distilled models) build one
    schedulers.Schedule of n_steps for the base model; a refiner then runs the same schedule from the first step whose timestep is
    below 1000 - REFINER_STEP_START, re-noising the base latent to that step's sigma. All three None / False: the reference's DDIM
    loop. deepcache: (interval[, branch]) DeepCache (Diffuser.set_deepcache) attached to the base UNet for this call and detached
    afterwards (the refiner is left alone). guidance_rescale: diffusers' guidance_rescale (phi, DESIGN.md §18) set on the base UNet
    for this call, with the prediction type and noise table the model has (Diffuser.set_prediction), and the previous phi restored
    afterwards. edit_image: u8 [1, H, W, 3], required with an edit UNet (cfg.is_edit, DESIGN.md §21) and refused otherwise: the output
    has the image's size, its latent (prepare_edit_latent) is attached for the call with image_guidance (diffusers'
    image_guidance_scale) and detached afterwards. As diffusers does, the call runs without CFG (no_cfg) when guidance <= 1 or
    image_guidance < 1; without a sampler or spacing that is the reference's DDIM update (Euler on the reference spacing). Returns
    uint8 [1, H, W, 3]."""
    sch = dict(sampler=sampler, spacing=spacing, no_cfg=no_cfg, edit_image=edit_image, image_guidance=image_guidance)
    if guidance_rescale:
        prev = diffuser.prediction
        diffuser.set_prediction(prev[0], guidance_rescale, alphas=prev[2])
        try:
            return sample(embedder, diffuser, decoder, prompt, guidance, n_steps, refiner, reference_rgb, crop, crop_out, resolution,
                          seed, noise, loras, controls, image_prompt, t2i_adapters, t2i_factor, pag, freeu, deepcache=deepcache, **sch)
        finally:
            diffuser.set_prediction(prev[0], prev[1], alphas=prev[2])
    if deepcache:
        diffuser.set_deepcache(*deepcache)
        try:
            return sample(embedder, diffuser, decoder, prompt, guidance, n_steps, refiner, reference_rgb, crop, crop_out, resolution,
                          seed, noise, loras, controls, image_prompt, t2i_adapters, t2i_factor, pag, freeu, **sch)
        finally:
            diffuser.set_deepcache(None)
    if freeu:
        diffuser.set_freeu(*freeu)
        try:
            return sample(embedder, diffuser, decoder, prompt, guidance, n_steps, refiner, reference_rgb, crop, crop_out, resolution,
                          seed, noise, loras, controls, image_prompt, t2i_adapters, t2i_factor, pag, **sch)
        finally:
            diffuser.set_freeu(None)
    if pag:
        diffuser.set_pag(pag[1], pag[0], *pag[2:3])
        try:
            return sample(embedder, diffuser, decoder, prompt, guidance, n_steps, refiner, reference_rgb, crop, crop_out, resolution,
                          seed, noise, loras, controls, image_prompt, t2i_adapters, t2i_factor, **sch)
        finally:
            diffuser.set_pag(None)
    if image_prompt:
        if isinstance(image_prompt, list):
            if len(image_prompt) > 4:
                raise _lib.SdxlError(f"image_prompt: {len(image_prompt)} prompts given, at most 4")
            prompts = []
            for item in image_prompt:
                adapter, encoder, images, scale = item[:4]
                e, neg = adapter.image_embeds(encoder, images)
                prompts.append((adapter, e.unsqueeze(0), scale, neg.unsqueeze(0), item[4] if len(item) > 4 else None))
            diffuser.set_image_prompts(prompts)
        else:
            adapter, encoder, images, scale = image_prompt
            e, neg = adapter.image_embeds(encoder, images)
            diffuser.set_image_prompt(adapter, e.unsqueeze(0), scale, negative=neg.unsqueeze(0))
        try:
            return sample(embedder, diffuser, decoder, prompt, guidance, n_steps, refiner, reference_rgb, crop, crop_out, resolution,
                          seed, noise, loras, controls, t2i_adapters=t2i_adapters, t2i_factor=t2i_factor, **sch)
        finally:
            diffuser.set_image_prompt(None)
    if controls:
        diffuser.set_controls(controls)
        try:
            return sample(embedder, diffuser, decoder, prompt, guidance, n_steps, refiner, reference_rgb, crop, crop_out, resolution,
                          seed, noise, loras, t2i_adapters=t2i_adapters, t2i_factor=t2i_factor, **sch)
        finally:
            diffuser.set_controls([])
    if t2i_adapters:
        schedule = _schedule(n_steps, sampler, spacing, no_cfg)
        if schedule is None:
            from .t2i_adapter import t2i_t_min
            t_min = t2i_t_min(n_steps, t2i_factor)
        else:   # the window follows the timesteps this schedule writes
            from .schedulers import t2i_t_min
            t_min = t2i_t_min(_alphas(diffuser), schedule, t2i_factor)
        diffuser.set_t2i_adapters(t2i_adapters, t_min=t_min)
        try:
            return sample(embedder, diffuser, decoder, prompt, guidance, n_steps, refiner, reference_rgb, crop, crop_out, resolution,
                          seed, noise, loras, **sch)
        finally:
            diffuser.set_t2i_adapters([])
    if not loras:
        return _sample(embedder, diffuser, decoder, prompt, guidance, n_steps, refiner, reference_rgb, crop, crop_out, resolution,
                       seed, noise, **sch)
    from .lora import load_adapter
    parts = [load_adapter(src, diffuser.cfg, embedder.clip.cfg, embedder.open_clip.cfg) for src, _ in loras]
    active = []
    try:
        for model, key in ((diffuser, "unet"), (embedder.clip, "te1"), (embedder.open_clip, "te2")):
            sets = [(p[key], scale) for p, (_, scale) in zip(parts, loras) if p[key]]
            if sets:
                active.append(model)
                model.set_adapters(sets)
        return _sample(embedder, diffuser, decoder, prompt, guidance, n_steps, refiner, reference_rgb, crop, crop_out, resolution,
                       seed, noise, **sch)
    finally:
        for model in active:
            model.set_adapters([])


def _schedule(n_steps, sampler=None, spacing=None, no_cfg=False):
    """sample()'s schedule: None (the reference's DDIM loop) unless one of the three is given."""
    if sampler is None and spacing is None and not no_cfg:
        return None
    from .schedulers import Schedule
    return Schedule(sampler or "euler", spacing or "leading", n_steps, no_cfg=no_cfg)


def _alphas(model):
    return [model.alpha(i) for i in range(model.cfg.n_steps)]


def refiner_schedule(refiner, schedule):
    """The refiner's part of the base model's schedule: from the first step whose timestep is below n_steps - REFINER_STEP_START,
    re-noising the base latent to that step's sigma. Refused when the schedule has no such step or starts below it: the hand-off
    the caller asked for does not exist."""
    from dataclasses import replace
    from .schedulers import build
    t, _ = build(_alphas(refiner), schedule)
    limit = refiner.cfg.n_steps - REFINER_STEP_START
    below = [k for k in range(schedule.n_steps) if t[k] < limit]
    if not below or below[0] == 0:
        raise _lib.SdxlError(f"sample: the refiner takes over at the first timestep below {limit}, but the {schedule.spacing} schedule of "
                             f"{schedule.n_steps} steps runs from t = {t[0]:g} to {t[-1]:g}: {'every' if below else 'no'} step is below it")
    return replace(schedule, first_step=below[0], renoise=True)


def _sample(embedder, diffuser, decoder, prompt, guidance, n_steps, refiner, reference_rgb, crop, crop_out, resolution, seed, noise,
            sampler=None, spacing=None, no_cfg=False, edit_image=None, image_guidance=1.5):
    if diffuser.cfg.is_edit != (edit_image is not None):
        raise _lib.SdxlError("sample: an edit UNet needs edit_image (the image to edit)" if diffuser.cfg.is_edit else
                             "sample: edit_image needs an edit UNet (cfg.is_edit)")
    if edit_image is None:
        return _sample_image(embedder, diffuser, decoder, prompt, guidance, n_steps, refiner, reference_rgb, crop, crop_out, resolution,
                             seed, noise, sampler, spacing, no_cfg)
    if refiner is not None or reference_rgb is not None:
        raise _lib.SdxlError("sample: edit_image does not go with a refiner or reference_rgb")
    if guidance <= 1 or image_guidance < 1:   # diffusers' do_classifier_free_guidance is off
        no_cfg = True
        spacing = spacing or (None if sampler else "reference")
    resolution = (int(edit_image.shape[1]), int(edit_image.shape[2]))
    latent = prepare_edit_latent(decoder, edit_image, resolution)
    diffuser.set_edit_image(latent, image_guidance)
    try:
        return _sample_image(embedder, diffuser, decoder, prompt, guidance, n_steps, None, None, crop, crop_out, resolution, seed, noise,
                             sampler, spacing, no_cfg, tuple(latent.shape[2:]))
    finally:
        diffuser.set_edit_image(None)


def _sample_image(embedder, diffuser, decoder, prompt, guidance, n_steps, refiner, reference_rgb, crop, crop_out, resolution, seed, noise,
                  sampler=None, spacing=None, no_cfg=False, latent_hw=None):
    """latent_hw: the extent of an attached edit image's latent, which the sampled latent takes (the image size / the VAE's factor)."""
    schedule = _schedule(n_steps, sampler, spacing, no_cfg)
    kw = {} if schedule is None else {"schedule": schedule}   # None: the calls below are the reference's, argument for argument
    refine = refiner_schedule(refiner, schedule) if refiner is not None and schedule is not None else None   # before any sampling
    inpaint_unet = diffuser.cfg.is_inpaint
    if inpaint_unet and reference_rgb is None:
        raise _lib.SdxlError("sample: an inpainting UNet needs reference_rgb (the image to repaint)")
    if reference_rgb is not None:
        resolution = (int(reference_rgb.shape[1]), int(reference_rgb.shape[2]))        # main.rs:225-229: orig_dims
    size = [int(resolution[0]), int(resolution[1])]
    cond = embedder.text_to_conditioning(prompt, size, [0, 0], size)                     # main.rs:231-235: size, crop = 0, ar = size
    if latent_hw is not None:
        cond.resolution = (8 * int(latent_hw[0]), 8 * int(latent_hw[1]))
    if inpaint_unet:
        # the UNet sees the mask and the masked image at every step and samples from noise, without blending (as diffusers does
        # for 9-channel UNets); the crop window at scale 1 is the exact pixel box, 1 = repaint
        pixel_mask = make_inpaint_mask(resolution, resolution, *crop, crop_out=crop_out, n_channels=1)
        c = prepare_inpaint_condition(decoder, reference_rgb, pixel_mask)
        cond.resolution = (8 * int(c.shape[2]), 8 * int(c.shape[3]))
        diffuser.set_inpaint_condition(c)
        try:
            latent = diffuser.sample_latent(cond, guidance, n_steps, noise=noise, seed=seed, **kw)
        finally:
            diffuser.set_inpaint_condition(None)
    elif reference_rgb is not None:
        ref_latent = decoder.image_to_latent(reference_rgb)                              # main.rs:158
        lh, lw = int(ref_latent.shape[2]), int(ref_latent.shape[3])
        cond.resolution = (8 * lh, 8 * lw)   # the sampler's latent extent follows the encoded reference (== the image size for the x8 SDXL VAE)
        mask = make_inpaint_mask(resolution, (lh, lw), *crop, crop_out=crop_out)
        latent = diffuser.sample_latent_with_inpainting(cond, guidance, n_steps, ref_latent, mask, init_noise=noise, seed=seed, **kw)   # main.rs:246
    else:
        latent = diffuser.sample_latent(cond, guidance, n_steps, noise=noise, seed=seed, **kw)                                   # main.rs:249
    if refine is not None:
        latent = refiner.refine_latent(latent, cond, guidance, 0, n_steps, seed=seed + 1, schedule=refine)
    elif refiner is not None:
        latent = refiner.refine_latent(latent, cond, guidance, REFINER_STEP_START, n_steps, seed=seed + 1)                    # main.rs:258-265
    return decoder.latent_to_image(latent)                                                                                   # main.rs:277


def load_models(ctx, model_dir: str, use_refiner: bool = False, tokenizer_dir: str = "tokenizer", tokenizers=None):
    """The four loads of the reference's `sample` (src/bin/sample/main.rs:156, 220, 242, 255, 274): `<model_dir>/embedder`,
    `/diffuser`, `/refiner` (optional) and `/latent_decoder`, each a burn record `<name>.mpk` + `<name>.cfg`
    (burn_record.read_model_dir); the tokenizers read `<tokenizer_dir>/clip/bpe_simple_vocab_16e6.txt` and
    `<tokenizer_dir>/open_clip/{merges,vocab}.txt` like the reference (src/token/clip.rs:97, open_clip.rs:88-89) unless a
    (clip, open_clip) pair is passed. Returns (embedder, diffuser, refiner | None, decoder), ready for `sample()`."""
    import os
    from . import burn_record as BR
    from .embedder import ClipTextEncoder, Embedder
    from .engine import Diffuser, LatentDecoder
    from .tokenizer import ClipTokenizer, OpenClipTokenizer
    files = BR.read_model_dir(model_dir, use_refiner)
    if tokenizers is None:
        tokenizers = (ClipTokenizer(os.path.join(tokenizer_dir, "clip", "bpe_simple_vocab_16e6.txt")),
                      OpenClipTokenizer(os.path.join(tokenizer_dir, "open_clip", "merges.txt"), os.path.join(tokenizer_dir, "open_clip", "vocab.txt")))
    ca, wa, cb, wb = files["embedder"]
    emb = Embedder(ctx, ClipTextEncoder(ctx, ca, wa), ClipTextEncoder(ctx, cb, wb), tokenizers[0], tokenizers[1])
    dif = Diffuser(ctx, *files["diffuser"])
    ref = Diffuser(ctx, *files["refiner"]) if files["refiner"] is not None else None
    dec = LatentDecoder(ctx, *files["latent_decoder"])
    return emb, dif, ref, dec
