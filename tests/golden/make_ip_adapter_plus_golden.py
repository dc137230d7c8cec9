"""Goldens of the CLIP vision encoder's hidden states (the image features of IP-Adapter Plus): transformers'
CLIPVisionModelWithProjection(output_hidden_states=True) (f32, CPU) on the seeded synthetic weights and pixels of
make_ip_adapter_golden.CASES. For hidden_idx in (0, n_layer - 1, n_layer) it stores hidden_states[hidden_idx] projected onto 16
seeded random columns (`<case>_h<idx>`, [N, T, 16]: every row is pinned, the file stays small) and, for the tiny configs, the full
hidden_states[-2] (`<case>_full`). Writes tests/golden/ip_adapter_vision_hidden.npz.

    python tests/golden/make_ip_adapter_plus_golden.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_ip_adapter_golden as G  # noqa: E402

from sdxl_b200.clip_vision import synth_vision_weights  # noqa: E402

N_COLS = 16


def columns(cfg):
    """The seeded projection [n_state, 16] of a config's hidden states."""
    return torch.randn(cfg.n_state, N_COLS, generator=torch.Generator().manual_seed(99)) / cfg.n_state ** 0.5


def hidden_indices(cfg):
    return (0, cfg.n_layer - 1, cfg.n_layer)


def main():
    out = {}
    for name, (cfg, ws, ps, n) in G.CASES.items():
        model = G.reference_embeds(cfg, synth_vision_weights(cfg, seed=ws))
        with torch.no_grad():
            hs = model(pixel_values=G.pixels(cfg, ps, n), output_hidden_states=True).hidden_states
        assert len(hs) == cfg.n_layer + 1
        for i in hidden_indices(cfg):
            out[f"{name}_h{i}"] = (hs[i] @ columns(cfg)).numpy().astype(np.float32)
        if name != "vit_h":
            out[f"{name}_full"] = hs[-2].numpy().astype(np.float32)
        print(name, tuple(hs[-2].shape), float(hs[-2].norm()))
    np.savez(os.path.join(HERE, "ip_adapter_vision_hidden.npz"), **out)


if __name__ == "__main__":
    main()
