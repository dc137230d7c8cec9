"""Goldens of the CLIP vision encoder: transformers' CLIPVisionModelWithProjection (f32, CPU) on the repo's seeded synthetic
weights (sdxl_b200.clip_vision.synth_vision_weights, f16 values widened) and seeded pixels, for the tiny d = 80 and d = 104
configs and for ViT-H/14 at full size with 2 images. Writes tests/golden/ip_adapter_vision.npz (image_embeds only: the GPU tests
regenerate weights and pixels from the same seeds).

    python tests/golden/make_ip_adapter_golden.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "stable-diffusion-xl-burn_b200"))

from sdxl_b200.clip_vision import SDXL_VIT_H, TINY_VIT_80, TINY_VIT_104, synth_vision_weights, to_hf  # noqa: E402

# name -> (config, weight seed, pixel seed, number of images)
CASES = {"tiny80": (TINY_VIT_80, 1, 11, 3), "tiny104": (TINY_VIT_104, 2, 12, 2), "vit_h": (SDXL_VIT_H, 3, 13, 2)}


def pixels(cfg, seed, n):
    """Seeded pixels in the range CLIPImageProcessor produces."""
    return torch.randn(n, 3, cfg.image_size, cfg.image_size, generator=torch.Generator().manual_seed(seed)).clamp(-1.8, 2.2)


def reference_embeds(cfg, w):
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    hc = CLIPVisionConfig(hidden_size=cfg.n_state, intermediate_size=cfg.mlp_dim, projection_dim=cfg.proj_dim, num_hidden_layers=cfg.n_layer,
                          num_attention_heads=cfg.n_head, image_size=cfg.image_size, patch_size=cfg.patch_size,
                          hidden_act="quick_gelu" if cfg.quick_gelu else "gelu", layer_norm_eps=1e-5)
    model = CLIPVisionModelWithProjection(hc).eval()
    missing, unexpected = model.load_state_dict(to_hf(w, cfg), strict=False)
    assert not unexpected and all(k.endswith("position_ids") for k in missing), (missing, unexpected)
    return model


def main():
    out = {}
    for name, (cfg, ws, ps, n) in CASES.items():
        w = synth_vision_weights(cfg, seed=ws)
        model = reference_embeds(cfg, w)
        with torch.no_grad():
            e = model(pixel_values=pixels(cfg, ps, n)).image_embeds
        out[name] = e.numpy().astype(np.float32)
        print(name, tuple(e.shape), float(e.norm()))
    np.savez(os.path.join(ROOT, "tests", "golden", "ip_adapter_vision.npz"), **out)


if __name__ == "__main__":
    main()
