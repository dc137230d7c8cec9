"""T2I-Adapter host side: the diffusers config and key mapping with their rejections, the oracle against a module-structured
restatement of diffusers' FullAdapterXL, the injection points, the timestep window rule and the C ABI."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from sdxl_b200 import (SDXL_BASE, SDXL_REFINER, SDXL_T2I_ADAPTER, TINY, TINY_T2I_ADAPTER, SdxlError, T2IAdapterConfig, _lib, ddim_timesteps,
                       synth_weights, t2i_adapter_tensor_specs, t2i_t_min)
from sdxl_b200.t2i_adapter import config_from_diffusers, from_diffusers, injection_points
from oracle import unet_oracle as O
import t2i_adapter_oracle as TA

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SDXL_JSON = {"_class_name": "T2IAdapter", "adapter_type": "full_adapter_xl", "channels": [320, 640, 1280, 1280], "downscale_factor": 16,
             "in_channels": 3, "num_res_blocks": 2}


def to_diffusers(w):
    """Pack names -> diffusers T2IAdapter keys (the inverse of from_diffusers)."""
    return {"adapter." + k.replace("/", "."): v for k, v in w.items()}


def test_config_accepts_sdxl_full_adapter_xl():
    cfg = config_from_diffusers(SDXL_JSON)
    assert cfg == SDXL_T2I_ADAPTER and cfg.channels == (320, 640, 1280, 1280)
    assert config_from_diffusers(dict(SDXL_JSON, in_channels=1)).in_channels == 1
    assert config_from_diffusers(dict(SDXL_JSON, channels=[64, 128, 256, 256]), TINY) == TINY_T2I_ADAPTER


@pytest.mark.parametrize("change, match", [
    ({"adapter_type": "full_adapter"}, "full_adapter"), ({"adapter_type": "light_adapter"}, "light_adapter"),
    ({"adapter_type": "multi_adapter"}, "multi_adapter"), ({"adapter_type": "coadapter"}, "coadapter"),
    ({"downscale_factor": 8}, "downscale_factor"), ({"channels": [320, 640, 1280]}, "channels")])
def test_config_rejects_other_adapters_by_name(change, match):
    with pytest.raises(SdxlError, match=match):
        config_from_diffusers(dict(SDXL_JSON, **change))


def test_sdxl_adapter_size_and_key_mapping():
    specs = t2i_adapter_tensor_specs(SDXL_T2I_ADAPTER)
    n = sum(int(np.prod(s[1])) for s in specs)
    assert 78e6 < n < 80e6, n                      # TencentARC's SDXL adapters have about 79 M parameters
    # a state dict with every key of the SDXL adapter (zero-stride tensors: shapes without the memory)
    sd = {"adapter." + name.replace("/", "."): torch.zeros(()).expand(*shape) for name, shape, _, _ in specs}
    assert len(sd) == len(specs) == 2 + 4 + 4 * 2 * 4
    cfg, w = from_diffusers(sd, SDXL_JSON)
    assert cfg == SDXL_T2I_ADAPTER and sorted(w) == sorted(s[0] for s in specs)
    assert w["body/2/in_conv/weight"].shape == (1280, 640, 1, 1) and w["conv_in/weight"].shape == (320, 768, 3, 3)
    assert w["body/3/resnets/1/block2/bias"].dtype == torch.float16
    with pytest.raises(SdxlError, match="adapter.body.4.resnets.0.block1.weight"):
        from_diffusers(dict(sd, **{"adapter.body.4.resnets.0.block1.weight": torch.zeros(1)}), SDXL_JSON)
    with pytest.raises(SdxlError, match="adapter.body.0.in_conv.weight"):
        from_diffusers(dict(sd, **{"adapter.body.0.in_conv.weight": torch.zeros(1)}), SDXL_JSON)
    with pytest.raises(SdxlError, match="shape"):
        from_diffusers(dict(sd, **{"adapter.conv_in.weight": torch.zeros(320, 192, 3, 3)}), SDXL_JSON)
    del sd["adapter.body.1.in_conv.bias"]
    with pytest.raises(SdxlError, match="body/1/in_conv/bias"):
        from_diffusers(sd, SDXL_JSON)


def test_pixel_unshuffle_matches_torch():
    x = torch.randn(2, 3, 64, 96, generator=torch.Generator().manual_seed(0))
    assert torch.equal(TA.pixel_unshuffle(x, 16), F.pixel_unshuffle(x, 16))
    y = TA.pixel_unshuffle(x, 16)
    assert y[1, 2 * 256 + 5 * 16 + 7, 3, 4] == x[1, 2, 16 * 3 + 5, 16 * 4 + 7]


class _Resnet(nn.Module):   # diffusers AdapterResnetBlock
    def __init__(self, c):
        super().__init__()
        self.block1, self.act, self.block2 = nn.Conv2d(c, c, 3, padding=1), nn.ReLU(), nn.Conv2d(c, c, 1)

    def forward(self, x):
        return self.block2(self.act(self.block1(x))) + x


class _Block(nn.Module):    # diffusers AdapterBlock
    def __init__(self, ci, co, n, down=False):
        super().__init__()
        self.downsample = nn.AvgPool2d(2, 2, ceil_mode=True) if down else None
        self.in_conv = nn.Conv2d(ci, co, 1) if ci != co else None
        self.resnets = nn.Sequential(*[_Resnet(co) for _ in range(n)])

    def forward(self, x):
        if self.downsample is not None:
            x = self.downsample(x)
        if self.in_conv is not None:
            x = self.in_conv(x)
        return self.resnets(x)


class _FullAdapterXL(nn.Module):
    def __init__(self, in_channels, ch, n):
        super().__init__()
        self.unshuffle = nn.PixelUnshuffle(16)
        self.conv_in = nn.Conv2d(in_channels * 256, ch[0], 3, padding=1)
        self.body = nn.ModuleList([_Block(ch[0], ch[0], n), _Block(ch[0], ch[1], n), _Block(ch[1], ch[2], n, down=True), _Block(ch[2], ch[3], n)])

    def forward(self, x):
        x = self.conv_in(self.unshuffle(x))
        out = []
        for b in self.body:
            x = b(x)
            out.append(x)
        return out


@pytest.mark.parametrize("in_channels", [3, 1])
def test_oracle_matches_module_structure(in_channels):
    acfg = T2IAdapterConfig(TINY, in_channels=in_channels)
    w = O.to_f32(synth_weights(acfg, seed=3))
    m = _FullAdapterXL(in_channels, acfg.channels, acfg.n_res_blocks)
    sd = {k[len("adapter."):]: v for k, v in to_diffusers(w).items()}
    m.load_state_dict(sd, strict=True)
    hint = torch.rand(2, in_channels, 64, 96, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        want = m(hint)
    got = TA.adapter_features(acfg, w, hint)
    assert [tuple(t.shape) for t in got] == [(2, 64, 4, 6), (2, 128, 4, 6), (2, 256, 2, 3), (2, 256, 2, 3)]
    for g, r in zip(got, want):
        assert torch.allclose(g, r, rtol=1e-5, atol=1e-5)


def test_injection_points():
    want = ["input_blocks/3", "input_blocks/5", "input_blocks/8", "middle_block"]
    assert injection_points(SDXL_BASE) == want and injection_points(TINY) == want
    assert O.injection_blocks(SDXL_BASE) == want[:3] and O.injection_blocks(TINY) == want[:3]
    with pytest.raises(SdxlError, match="refiner"):
        injection_points(SDXL_REFINER)


@pytest.mark.parametrize("n_steps, factor", [(30, 1.0), (30, 0.5), (30, 0.0), (31, 0.3), (4, 0.5), (4, 0.2), (50, 0.85), (1, 1.0)])
def test_t_min_window(n_steps, factor):
    ts = ddim_timesteps(n_steps)
    t_min = t2i_t_min(n_steps, factor)
    active = [i for i, t in enumerate(ts) if t >= t_min]
    assert active == list(range(int(len(ts) * factor)))       # diffusers: i < int(num_inference_steps * adapter_conditioning_factor)
    if factor == 0.0:
        assert t_min > max(ts)


def test_t2i_abi_from_c(tmp_path):
    """A C99 program using the T2I-Adapter part of include/sdxl_b200.h compiles, links and sees the struct layouts a binding needs."""
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib_dir = os.path.join(ROOT, "stable-diffusion-xl-burn_b200", "sdxl_b200")
    exe = str(tmp_path / "t2i_adapter_abi_check")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "c_abi", "t2i_adapter_abi_check.c"), "-L", lib_dir, "-lsdxl_b200", "-Wl,-rpath," + lib_dir,
                        "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout.startswith("t2i_adapter_abi_check ok"), (r.returncode, r.stdout, r.stderr)
    n_max, s_ctl, s_cfg = (int(v) for v in r.stdout.split()[-3:])
    assert n_max == _lib.MAX_T2I_ADAPTERS and s_ctl == C.sizeof(_lib.T2IControl) and s_cfg == C.sizeof(_lib.T2IAdapterCfg)
