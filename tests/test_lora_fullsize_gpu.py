"""SDXL base (2.57 B parameters) with a rank-32 synthetic LoRA adapter on every attention, feed-forward and proj_in/out
Linear (722 layers): the 1024x1024 forward of the model merged on the device against a model loaded from host-merged weights,
bit-exact restore, and the apply / restore times."""
import time

import pytest
import torch

import sdxl_b200
from sdxl_b200 import SDXL_BASE, Diffuser
from sdxl_b200.lora import merge_into
from lora_cases import layer_paths, make_adapter
from harness import rel_err

pytestmark = pytest.mark.gpu


def test_base_1024_rank32(ctx):
    w = sdxl_b200.synth_weights(SDXL_BASE, seed=0, device=str(ctx.device))
    d = Diffuser(ctx, SDXL_BASE, sdxl_b200.build_pack(w))
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 128, 128, generator=g)
    c = torch.randn(2, 77, 2048, generator=g).half().float()
    y = torch.randn(2, 2816, generator=g).half().float()
    base = d.unet_forward(x, [749], c, y)
    paths = [p for p in layer_paths(SDXL_BASE) if "/transformer" in p]
    assert len(paths) == 722
    ad = make_adapter(SDXL_BASE, paths, rank=32, seed=1, dyadic=False, alpha=16.0)
    ad_dev = {k: v.to(ctx.device) for k, v in ad.items()}
    pack = sdxl_b200.build_pack(ad_dev)
    d.set_adapters([(pack, 1.0)])       # first touch: allocates the backups
    d.set_adapters([])
    ctx.synchronize()
    t0 = time.perf_counter()
    d.set_adapters([(pack, 1.0)])
    ctx.synchronize()
    t_apply = time.perf_counter() - t0
    out = d.unet_forward(x, [749])
    t0 = time.perf_counter()
    d.set_adapters([])
    ctx.synchronize()
    t_restore = time.perf_counter() - t0
    restored = d.unet_forward(x, [749])
    assert torch.equal(restored, base)

    touched = {p + "/weight" for p in paths}
    wm = dict(w)
    wm.update({k: v.to(ctx.device) for k, v in merge_into({k: w[k].cpu() for k in touched}, ad, 1.0).items()})
    d.close()
    ref_model = Diffuser(ctx, SDXL_BASE, sdxl_b200.build_pack(wm))
    ref = ref_model.unet_forward(x, [749], c, y)
    ref_model.close()
    e = rel_err(out, ref)
    print(f"SDXL base 1024^2, rank-32 adapter on 722 layers: apply {t_apply * 1e3:.1f} ms (host clock around a synchronised "
          f"call, backups already allocated), restore {t_restore * 1e3:.1f} ms; forward vs host-merged load rel err {e:.2e}, "
          f"adapter moves the forward by {rel_err(out, base):.2e}")
    assert e <= 1e-3 and rel_err(out, base) > 1e-2
