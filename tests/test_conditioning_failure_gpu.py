"""A set_conditioning whose buffers cannot be allocated fails and leaves the UNet's previous conditioning, and the launch plan
over it, in effect: the next forward is bit-identical to the one before the failed call."""
import pytest
import torch

from sdxl_b200 import TINY, Diffuser, SdxlError, synth_weights
from sdxl_b200.config import block_program
from harness import arb, plan_builds

pytestmark = pytest.mark.gpu
T = 499


def test_failed_set_conditioning_keeps_the_previous_one(ctx):
    d = Diffuser(ctx, TINY, synth_weights(TINY, seed=0))
    x = arb(2, 4, 16, 16)
    y = arb(2, TINY.adm_in_channels).half()
    want = d.unet_forward(x, [T], arb(2, 7, TINY.context_dim).half(), y)
    n_builds = plan_builds(d)
    # hoisted K/V of one context row: f16 [K | V] of width 2C for every transformer block (about 15 KB at TINY)
    ins, mid, outs = block_program(TINY)
    kv_row = sum(2 * 2 * b.c_out * b.depth for b in ins + [mid] + outs)
    total = torch.cuda.mem_get_info(ctx.device)[1]
    n_ctx = total // (2 * kv_row) + 1   # two rows of this length need more K/V than the device has: cudaMalloc refuses the request
    big = torch.zeros(2, n_ctx, TINY.context_dim, dtype=torch.float16, device=ctx.device)
    with pytest.raises(SdxlError, match="cannot allocate"):
        d.set_conditioning(big, y)
    del big
    assert torch.equal(d.unet_forward(x, [T]), want)   # the retained conditioning, on the same plan
    assert plan_builds(d) == n_builds
    d.close()
