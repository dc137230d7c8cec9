"""sdxl_b200 — host-side mirror of the reference's diffusion sampling surface over libsdxl_b200.so."""
from .config import SDXL_BASE, SDXL_REFINER, TINY, TINY_REFINER, SDXL_VAE, TINY_VAE, SDXL_CLIP_L, SDXL_OPEN_CLIP_G, TINY_CLIP, TINY_OPEN_CLIP, ClipConfig, UNetConfig, VaeConfig, block_program  # noqa: F401
from .config import SDXL_CONTROLNET, TINY_CONTROLNET, ControlNetConfig  # noqa: F401
from .config import SDXL_T2I_ADAPTER, TINY_T2I_ADAPTER, T2IAdapterConfig  # noqa: F401
from .config import SDXL_INPAINT, TINY_INPAINT  # noqa: F401
from .config import SDXL_EDIT, TINY_EDIT  # noqa: F401
from .weights import alphas_cumprod, build_pack, n_params, synth_weights, unet_tensor_specs, vae_decoder_tensor_specs, vae_encoder_tensor_specs, vae_tensor_specs, clip_tensor_specs  # noqa: F401
from .weights import controlnet_tensor_specs, t2i_adapter_tensor_specs  # noqa: F401
from ._lib import LIB_PATH, PROTOTYPES, SdxlError, SdxlLibraryMissing, load  # noqa: F401
from .engine import Conditioning, Context, Diffuser, LatentDecoder, ddim_timesteps  # noqa: F401
from .tokenizer import ClipTokenizer, OpenClipTokenizer  # noqa: F401
from .embedder import ClipTextEncoder, Embedder, conditioning_embedding  # noqa: F401
from .pipeline import load_models, make_inpaint_mask, prepare_edit_latent, prepare_inpaint_condition, sample  # noqa: F401
from . import diffusers_unet  # noqa: F401
from . import schedulers  # noqa: F401
from .schedulers import Schedule  # noqa: F401
from .controlnet import ControlNet  # noqa: F401
from .ip_adapter import IPAdapter  # noqa: F401
from .t2i_adapter import T2IAdapter, t2i_t_min  # noqa: F401
from .pag import layer_mask as pag_layer_mask, pag_scale_at, self_attention_names  # noqa: F401
from .clip_vision import SDXL_VIT_BIGG, SDXL_VIT_H, ClipVisionConfig, ClipVisionEncoder, clip_preprocess  # noqa: F401
from . import burn_record  # noqa: F401
