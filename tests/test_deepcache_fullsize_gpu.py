"""DeepCache on SDXL base (synthetic weights, the seed and conditioning of tests/fullsize_cases.py) at 1024^2 with CFG: the cached
forward right after a full one on the same inputs is that forward bit for bit for branches 0 and 3, and a 30-step DDIM loop at
interval 3 stays finite."""
import pytest
import torch

import sdxl_b200
from sdxl_b200 import SDXL_BASE, Conditioning, Diffuser
import fullsize_cases as FC
from harness import first_difference

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def base(ctx):
    d = Diffuser(ctx, SDXL_BASE, sdxl_b200.synth_weights(SDXL_BASE, seed=FC.BASE_WEIGHT_SEED))
    yield d
    d.close()


@pytest.mark.parametrize("b", [0, 3])
def test_cached_after_full_is_the_full_forward_1024(base, b):
    x, c, y = FC.fwd_1024_inputs()
    x, c, y = torch.cat([x, 0.5 * x]), torch.cat([c, c.flip(1)]), torch.cat([y, y.flip(1)])   # [cond | uncond]-sized batch
    base.set_deepcache(3, b)
    try:
        full = base.unet_forward(x, [FC.FWD_1024_T], c, y, cached=False).cpu()
        cached = base.unet_forward(x, [FC.FWD_1024_T], c, y, cached=True).cpu()
    finally:
        base.set_deepcache(None)
    assert bool(torch.isfinite(full).all())
    assert torch.equal(cached, full), first_difference(full, cached)


def test_ddim_30_steps_interval_3_is_finite(base):
    base.set_deepcache(3, 0)
    try:
        out = base.sample_latent(Conditioning(**FC.base_conditioning(1024)), 7.5, 30, noise=FC.base_noise(1024)).cpu()
    finally:
        base.set_deepcache(None)
    assert bool(torch.isfinite(out).all()) and float(out.abs().max()) > 0
