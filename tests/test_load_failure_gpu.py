"""A UNet load that fails after its weights were re-laid out must free them.

The weight pack below has every SDXL base tensor but no `alphas_cumprod`, so sdxl_unet_load builds the whole ~5 GB weight
arena and only then fails. One load, then the device's free memory is compared with what it was before the call.
"""
import pytest
import torch

import sdxl_b200
from sdxl_b200 import SDXL_BASE, Diffuser, SdxlError

pytestmark = pytest.mark.gpu


def test_failed_unet_load_frees_weight_arena(ctx):
    w = sdxl_b200.synth_weights(SDXL_BASE, seed=0, device=str(ctx.device))
    del w["alphas_cumprod"]
    pack = sdxl_b200.build_pack(w)
    del w
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free_before, _ = torch.cuda.mem_get_info(ctx.device)
    with pytest.raises(SdxlError, match="alphas_cumprod"):
        Diffuser(ctx, SDXL_BASE, pack)
    torch.cuda.synchronize()
    free_after, _ = torch.cuda.mem_get_info(ctx.device)
    drop = free_before - free_after
    print(f"free device memory dropped by {drop / 2**20:.1f} MiB over a failed load of a {pack.numel() / 2**30:.2f} GiB pack")
    assert drop < pack.numel() // 2
