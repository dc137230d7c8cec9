"""GPU tests of the CLIP vision encoder (sdxl_clip_vision_encode) against transformers' CLIPVisionModelWithProjection, through
the goldens of tests/golden/make_ip_adapter_golden.py (weights and pixels regenerated from the same seeds)."""
import os

import numpy as np
import pytest
import torch

from sdxl_b200.clip_vision import ClipVisionEncoder, synth_vision_weights

pytestmark = pytest.mark.gpu
TOL = 2e-3
HERE = os.path.dirname(os.path.abspath(__file__))


def _golden():
    import sys
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_ip_adapter_golden as G
    return G, np.load(os.path.join(HERE, "golden", "ip_adapter_vision.npz"))


@pytest.mark.parametrize("name", ["tiny80", "tiny104", "vit_h"])
def test_encode_against_transformers(ctx, name):
    G, gold = _golden()
    cfg, ws, ps, n = G.CASES[name]
    enc = ClipVisionEncoder(ctx, cfg, synth_vision_weights(cfg, seed=ws))
    got = enc.encode(G.pixels(cfg, ps, n)).cpu().double()
    enc.close()
    ref = torch.from_numpy(gold[name]).double()
    err = float((got - ref).norm() / ref.norm())
    print(f"{name}: rel err {err:.3e}")
    assert err < TOL
