"""GPU tests of the CLIP vision encoder's hidden states (sdxl_clip_vision_encode_hidden, the image features of IP-Adapter Plus)
against transformers' CLIPVisionModelWithProjection(output_hidden_states=True), through the goldens of
tests/golden/make_ip_adapter_plus_golden.py (weights and pixels regenerated from the same seeds)."""
import os
import sys

import numpy as np
import pytest
import torch

from sdxl_b200 import SdxlError
from sdxl_b200.clip_vision import ClipVisionEncoder, synth_vision_weights

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
# The bound of test_clip_vision_gpu's image_embeds (f16 GEMM operands, f32 residual stream): the hidden states are the same
# stream before post_layernorm and the projection, so the same normwise relative bound applies.
TOL = 2e-3


def _golden():
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_ip_adapter_plus_golden as GP
    return GP, np.load(os.path.join(HERE, "golden", "ip_adapter_vision_hidden.npz"))


def golden_rel_err(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("name", ["tiny80", "tiny104", "vit_h"])
def test_encode_hidden_against_transformers(ctx, name):
    GP, gold = _golden()
    cfg, ws, ps, n = GP.G.CASES[name]
    enc = ClipVisionEncoder(ctx, cfg, synth_vision_weights(cfg, seed=ws))
    px = GP.G.pixels(cfg, ps, n)
    cols = GP.columns(cfg).double()
    for idx in GP.hidden_indices(cfg):
        got = enc.encode_hidden(px, idx).cpu()
        assert got.shape == (n, cfg.n_tokens, cfg.n_state)
        err = golden_rel_err(got.double() @ cols, torch.from_numpy(gold[f"{name}_h{idx}"]))
        print(f"{name} hidden_states[{idx}] (16 projected columns): rel err {err:.3e}")
        assert err < TOL
    if name != "vit_h":
        err = golden_rel_err(enc.encode_hidden(px), torch.from_numpy(gold[f"{name}_full"]))   # default: hidden_states[-2]
        print(f"{name} hidden_states[-2] (full): rel err {err:.3e}")
        assert err < TOL
    enc.close()


def test_encode_hidden_and_embeds_share_the_encoder(ctx):
    """Alternating hidden-state and image_embeds calls rebuild the plan per (N, hidden_idx) and give the same values each time;
    hidden_idx outside [0, n_layer] is refused."""
    GP, _ = _golden()
    cfg, ws, ps, n = GP.G.CASES["tiny80"]
    enc = ClipVisionEncoder(ctx, cfg, synth_vision_weights(cfg, seed=ws))
    px = GP.G.pixels(cfg, ps, n)
    e1, h1 = enc.encode(px), enc.encode_hidden(px, 1)
    e2, h2 = enc.encode(px), enc.encode_hidden(px, 1)
    assert torch.equal(e1, e2) and torch.equal(h1, h2)
    assert torch.equal(enc.encode_hidden(px[:1], 1), h1[:1])
    for bad in (-1, cfg.n_layer + 1):
        with pytest.raises(SdxlError, match="hidden_idx"):
            enc.encode_hidden(px, bad)
    enc.close()
