"""ctypes binding of libsdxl_b200.so (the C ABI in include/sdxl_b200.h).

There is deliberately no fallback: if the CUDA library is missing the import of the product path
fails loudly (`SdxlLibraryMissing`), it never routes through the CPU oracle.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libsdxl_b200.so")

SDXL_MAX_LEVELS = 8


class SdxlLibraryMissing(RuntimeError):
    pass


class SdxlError(RuntimeError):
    pass


class UnetCfg(C.Structure):
    _fields_ = [
        ("adm_in_channels", C.c_int32), ("in_channels", C.c_int32), ("out_channels", C.c_int32),
        ("model_channels", C.c_int32), ("n_levels", C.c_int32), ("channel_mults", C.c_int32 * SDXL_MAX_LEVELS),
        ("n_head_channels", C.c_int32), ("transformer_depths", C.c_int32 * SDXL_MAX_LEVELS),
        ("context_dim", C.c_int32), ("is_refiner", C.c_int32), ("n_steps", C.c_int32), ("edit_layout", C.c_int32),
    ]


class Conditioning(C.Structure):
    _fields_ = [
        ("on_host", C.c_int32), ("n_batch", C.c_int32), ("n_ctx", C.c_int32),
        ("context_full", C.c_void_p), ("context_open_clip", C.c_void_p),
        ("unconditional_context_full", C.c_void_p), ("unconditional_context_open_clip", C.c_void_p),
        ("channel_context", C.c_void_p), ("channel_context_refiner", C.c_void_p),
        ("unconditional_channel_context", C.c_void_p), ("unconditional_channel_context_refiner", C.c_void_p),
        ("resolution", C.c_int32 * 2),
    ]


class VaeCfg(C.Structure):
    _fields_ = [
        ("latent_channels", C.c_int32), ("n_blocks", C.c_int32),
        ("block_in", C.c_int32 * SDXL_MAX_LEVELS), ("block_out", C.c_int32 * SDXL_MAX_LEVELS),
        ("n_group", C.c_int32), ("scale_factor", C.c_double),
        ("n_enc_blocks", C.c_int32), ("enc_in", C.c_int32 * SDXL_MAX_LEVELS), ("enc_out", C.c_int32 * SDXL_MAX_LEVELS),
        ("enc_z_channels", C.c_int32),
    ]


class ClipCfg(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_vocab", "n_state", "embed_dim", "n_head", "n_ctx", "n_layer", "quick_gelu")]


class Adapter(C.Structure):
    _fields_ = [("pack", C.c_void_p), ("bytes", C.c_size_t), ("pack_on_device", C.c_int32), ("scale", C.c_float)]


MAX_ADAPTERS = 16   # SDXL_MAX_ADAPTERS (include/sdxl_b200.h)


class ControlNetCfg(C.Structure):
    _fields_ = [("unet", UnetCfg), ("hint_in_channels", C.c_int32), ("n_hint_blocks", C.c_int32),
                ("hint_block_channels", C.c_int32 * SDXL_MAX_LEVELS)]


class Control(C.Structure):
    _fields_ = [("net", C.c_void_p), ("hint", C.c_void_p), ("hint_on_host", C.c_int32), ("n_hint", C.c_int32),
                ("height", C.c_int32), ("width", C.c_int32), ("scale", C.c_float)]


MAX_CONTROLS = 4    # SDXL_MAX_CONTROLS (include/sdxl_b200.h)


class ClipVisionCfg(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_state", "n_head", "n_layer", "mlp_dim", "image_size", "patch_size", "proj_dim", "quick_gelu")]


class IpAdapterCfg(C.Structure):
    _fields_ = [("unet", UnetCfg), ("image_embed_dim", C.c_int32), ("tokens_per_image", C.c_int32), ("resampler_depth", C.c_int32),
                ("resampler_heads", C.c_int32)]


class ImagePrompt(C.Structure):
    _fields_ = [("adapter", C.c_void_p), ("embeds", C.c_void_p), ("negative_embeds", C.c_void_p), ("on_host", C.c_int32),
                ("n_batch", C.c_int32), ("n_images", C.c_int32), ("scale", C.c_float), ("block_scales_host", C.c_void_p),
                ("seq_len", C.c_int32)]


class IpMask(C.Structure):
    _fields_ = [("mask", C.c_void_p), ("on_host", C.c_int32), ("height", C.c_int32), ("width", C.c_int32)]


class T2IAdapterCfg(C.Structure):
    _fields_ = [("unet", UnetCfg), ("in_channels", C.c_int32), ("n_res_blocks", C.c_int32)]


class T2IControl(C.Structure):
    _fields_ = [("adapter", C.c_void_p), ("hint", C.c_void_p), ("hint_on_host", C.c_int32), ("n_hint", C.c_int32),
                ("height", C.c_int32), ("width", C.c_int32), ("scale", C.c_float)]


MAX_T2I_ADAPTERS = 4   # SDXL_MAX_T2I_ADAPTERS (include/sdxl_b200.h)


class InpaintCondition(C.Structure):
    _fields_ = [("cond", C.c_void_p), ("on_host", C.c_int32), ("n", C.c_int32), ("height", C.c_int32), ("width", C.c_int32)]


class EditImage(C.Structure):
    _fields_ = [("latent", C.c_void_p), ("on_host", C.c_int32), ("n", C.c_int32), ("height", C.c_int32), ("width", C.c_int32),
                ("image_guidance", C.c_float)]


class Pag(C.Structure):
    _fields_ = [("scale", C.c_float), ("adaptive_scale", C.c_float), ("n_layers", C.c_int32), ("layers_host", C.c_void_p),
                ("forward_perturbed_rows", C.c_int32)]


class Freeu(C.Structure):
    _fields_ = [("s1", C.c_float), ("s2", C.c_float), ("b1", C.c_float), ("b2", C.c_float)]


class Deepcache(C.Structure):
    _fields_ = [("interval", C.c_int32), ("branch", C.c_int32), ("forward_cached", C.c_int32)]


class Prediction(C.Structure):
    _fields_ = [("type", C.c_int32), ("guidance_rescale", C.c_float), ("n_alphas", C.c_int32), ("alphas_cumprod_host", C.c_void_p)]


PREDICTIONS = {"epsilon": 0, "v_prediction": 1}   # SDXL_PREDICTION_* (include/sdxl_b200.h), by diffusers' prediction_type


class Schedule(C.Structure):
    _fields_ = [("sampler", C.c_int32), ("spacing", C.c_int32), ("n_steps", C.c_int32), ("first_step", C.c_int32),
                ("last_step", C.c_int32), ("renoise", C.c_int32), ("no_cfg", C.c_int32), ("karras_rho", C.c_float),
                ("eta", C.c_float), ("s_noise", C.c_float)]


# name -> (restype, argtypes); every symbol include/sdxl_b200.h declares
P = C.c_void_p
I = C.c_int
PROTOTYPES = {
    "sdxl_ctx_create": (I, [I, P, C.POINTER(P)]),
    "sdxl_ctx_destroy": (None, [P]),
    "sdxl_last_error": (C.c_char_p, [P]),
    "sdxl_ctx_synchronize": (I, [P]),
    "sdxl_ctx_launch_count": (C.c_uint64, [P]),
    "sdxl_debug_fill": (I, []),
    "sdxl_unet_load": (I, [P, C.POINTER(UnetCfg), P, C.c_size_t, I, C.POINTER(P)]),
    "sdxl_unet_destroy": (None, [P]),
    "sdxl_unet_set_conditioning": (I, [P, I, I, P, P]),
    "sdxl_unet_forward": (I, [P, I, I, I, P, C.c_int32, P]),
    "sdxl_unet_forward_f32": (I, [P, I, I, I, P, C.c_int32, P]),
    "sdxl_sample_latent": (I, [P, C.POINTER(Conditioning), C.c_double, I, I, P, P, I, C.c_uint64, P, P, P]),
    "sdxl_schedule_build": (I, [P, I, C.POINTER(Schedule), P, P]),
    "sdxl_schedule_last_error": (C.c_char_p, []),
    "sdxl_sample_latent_scheduled": (I, [P, C.POINTER(Conditioning), C.c_double, C.POINTER(Schedule), P, P, I, C.c_uint64, P, P, P]),
    "sdxl_unet_forward_f32_at": (I, [P, I, I, I, P, C.c_double, P]),
    "sdxl_sampler_begin": (I, [P, C.POINTER(Conditioning), C.c_double]),
    "sdxl_sampler_step": (I, [P, I, I]),
    "sdxl_sampler_step_host": (I, [P, I, I, P]),
    "sdxl_sampler_set_latent": (I, [P, P, I]),
    "sdxl_sampler_get_latent": (I, [P, P, I]),
    "sdxl_unet_alpha": (C.c_double, [P, I]),
    "sdxl_unet_load_broadcast": (I, [P, C.POINTER(UnetCfg), P, C.c_size_t, I, P, I, I, C.POINTER(P)]),
    "sdxl_unet_plan_flops": (C.c_double, [P]),
    "sdxl_unet_plan_num_ops": (I, [P]),
    "sdxl_unet_plan_flops_executed": (C.c_double, [P]),
    "sdxl_unet_profile_plan": (I, [P, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int)]),
    "sdxl_unet_profile_dump": (I, [P, C.c_char_p]),
    "sdxl_randn": (I, [P, P, C.c_size_t, C.c_uint64, C.c_uint64]),
    "sdxl_qkv_attention": (I, [P, P, P, P, P, I, I, I, I, I, P]),
    "sdxl_op_linear": (I, [P, P, P, P, P, I, I, I, I, I, P]),
    "sdxl_op_conv2d": (I, [P, P, P, P, I, I, I, I, I, I, I, I, P]),
    "sdxl_op_group_norm": (I, [P, P, I, P, I, I, I, I, P, P, C.c_float, I, P]),
    "sdxl_op_layer_norm": (I, [P, P, P, P, C.c_float, I, I, P]),
    "sdxl_op_timestep_embedding": (I, [P, P, I, I, I, P]),
    "sdxl_vae_load": (I, [P, C.POINTER(VaeCfg), P, C.c_size_t, I, C.POINTER(P)]),
    "sdxl_vae_destroy": (None, [P]),
    "sdxl_vae_decode_latent": (I, [P, I, I, I, P, I, P]),
    "sdxl_vae_latent_to_image": (I, [P, I, I, I, P, I, P]),
    "sdxl_vae_encode_image": (I, [P, I, I, I, P, I, P]),
    "sdxl_vae_image_to_latent": (I, [P, I, I, I, P, I, P]),
    "sdxl_vae_encode_plan_flops": (C.c_double, [P]),
    "sdxl_vae_plan_flops": (C.c_double, [P]),
    "sdxl_vae_profile_plan": (I, [P, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int)]),
    "sdxl_vae_profile_dump": (I, [P, C.c_char_p]),
    "sdxl_tokenizer_last_error": (C.c_char_p, []),
    "sdxl_tokenizer_create_clip": (I, [C.c_char_p, C.POINTER(P)]),
    "sdxl_tokenizer_create_open_clip": (I, [C.c_char_p, C.c_char_p, C.POINTER(P)]),
    "sdxl_tokenizer_destroy": (None, [P]),
    "sdxl_tokenizer_encode": (I, [P, C.c_char_p, I, I, C.POINTER(C.c_uint32), I, C.POINTER(I)]),
    "sdxl_tokenizer_decode": (I, [P, C.POINTER(C.c_uint32), I, C.c_char_p, I, C.POINTER(I)]),
    "sdxl_tokenize_text": (I, [P, C.c_char_p, I, C.POINTER(C.c_int32)]),
    "sdxl_tokenizer_special": (I, [P, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    "sdxl_clip_load": (I, [P, C.POINTER(ClipCfg), P, C.c_size_t, I, C.POINTER(P)]),
    "sdxl_clip_destroy": (None, [P]),
    "sdxl_clip_forward_hidden": (I, [P, I, C.POINTER(C.c_int32), I, P, I]),
    "sdxl_clip_forward_hidden_pooled": (I, [P, I, C.POINTER(C.c_int32), I, P, P, I]),
    "sdxl_clip_plan_flops": (C.c_double, [P]),
    "sdxl_unet_set_adapters": (I, [P, I, C.POINTER(Adapter)]),
    "sdxl_clip_set_adapters": (I, [P, I, C.POINTER(Adapter)]),
    "sdxl_controlnet_load": (I, [P, C.POINTER(ControlNetCfg), P, C.c_size_t, I, C.POINTER(P)]),
    "sdxl_controlnet_destroy": (None, [P]),
    "sdxl_unet_set_controls": (I, [P, I, C.POINTER(Control)]),
    "sdxl_controlnet_embed_hint": (I, [P, I, I, I, P, I, P]),
    "sdxl_clip_vision_load": (I, [P, C.POINTER(ClipVisionCfg), P, C.c_size_t, I, C.POINTER(P)]),
    "sdxl_clip_vision_destroy": (None, [P]),
    "sdxl_clip_vision_encode": (I, [P, I, P, I, P]),
    "sdxl_clip_vision_encode_hidden": (I, [P, I, P, I, I, P]),
    "sdxl_unet_plan_builds": (C.c_uint64, [P]),
    "sdxl_ip_adapter_load": (I, [P, C.POINTER(IpAdapterCfg), P, C.c_size_t, I, C.POINTER(P)]),
    "sdxl_ip_adapter_destroy": (None, [P]),
    "sdxl_unet_set_image_prompt": (I, [P, C.POINTER(ImagePrompt)]),
    "sdxl_unet_set_image_prompts": (I, [P, I, C.POINTER(ImagePrompt), C.POINTER(IpMask)]),
    "sdxl_ip_adapter_project": (I, [P, I, P, I, P]),
    "sdxl_ip_adapter_resample": (I, [P, I, I, P, I, P]),
    "sdxl_op_ip_attention": (I, [P, P, P, P, P, P, I, I, I, I, I, I, C.c_float, P]),
    "sdxl_t2i_adapter_load": (I, [P, C.POINTER(T2IAdapterCfg), P, C.c_size_t, I, C.POINTER(P)]),
    "sdxl_t2i_adapter_destroy": (None, [P]),
    "sdxl_unet_set_t2i_adapters": (I, [P, I, C.POINTER(T2IControl), C.c_int32]),
    "sdxl_t2i_adapter_features": (I, [P, I, I, I, P, I, P]),
    "sdxl_unet_set_inpaint_condition": (I, [P, C.POINTER(InpaintCondition)]),
    "sdxl_unet_set_edit_image": (I, [P, C.POINTER(EditImage)]),
    "sdxl_unet_num_self_attentions": (I, [P]),
    "sdxl_unet_set_pag": (I, [P, C.POINTER(Pag)]),
    "sdxl_unet_set_freeu": (I, [P, C.POINTER(Freeu)]),
    "sdxl_unet_set_deepcache": (I, [P, C.POINTER(Deepcache)]),
    "sdxl_unet_set_prediction": (I, [P, C.POINTER(Prediction)]),
    "sdxl_make_inpaint_mask": (I, [I, I, I, I, I, I, I, I, I, I, P]),
    "sdxl_mpk_decode_u16": (I, [P, C.c_size_t, C.c_size_t, P, C.POINTER(C.c_size_t)]),
    "sdxl_mpk_encode_u16": (C.c_size_t, [P, C.c_size_t, P]),
}

PROFILE_KINDS = 24   # SDXL_PROFILE_KINDS (include/sdxl_b200.h)
_lib = None


def load() -> C.CDLL:
    """dlopen the library and bind every prototype. Works without a GPU (no CUDA call is made)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SdxlLibraryMissing(
            f"{LIB_PATH} not found: build it with `python stable-diffusion-xl-burn_b200/build.py` "
            "(or __graft_entry__.build()). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib
