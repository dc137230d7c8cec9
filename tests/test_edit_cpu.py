"""CPU tests of instruction-based editing (DESIGN.md §21): the oracle's combine against the formula, the layout rules of UNetConfig and
the C cfg, from_diffusers on a synthetic 8-channel config, the refusals that need no GPU, and the C ABI of sdxl_edit_image and the
cfg's edit_layout field against the ctypes mirror."""
import ctypes as C
import json
import os
import shutil
import subprocess

import pytest
import torch

from sdxl_b200 import SDXL_BASE, SDXL_EDIT, TINY, TINY_EDIT, _lib, sample, synth_weights
from sdxl_b200.diffusers_unet import config_from_diffusers, from_diffusers, name_map
from sdxl_b200.engine import _cfg_struct
from sdxl_b200._lib import SdxlError
import edit_oracle as EO
import prediction_oracle as PR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oracle_combine_is_the_formula():
    g = torch.Generator().manual_seed(0)
    c, i, u = (torch.randn(2, 4, 8, 8, generator=g, dtype=torch.float64) for _ in range(3))
    s, s_img = 5.0, 1.5
    want = u + s * (c - i) + s_img * (i - u)
    assert torch.allclose(EO.combine(c, i, u, s, s_img), want, rtol=0, atol=1e-13)
    # s_img = 1: the image rows drop out of the unconditional term, g = i + s (c - i)
    assert torch.allclose(EO.combine(c, i, u, s, 1.0), i + s * (c - i), rtol=0, atol=1e-13)
    # i = u: text guidance alone, and guidance rescale of the combine keeps the conditional rows' std
    assert torch.allclose(EO.combine(c, u, u, s, s_img), u + s * (c - u), rtol=0, atol=1e-13)
    r = PR.rescale_noise_cfg(EO.combine(c, i, u, s, s_img), c, 1.0)
    assert torch.allclose(r.reshape(2, -1).std(dim=1), c.reshape(2, -1).std(dim=1), rtol=1e-12)


def test_layout_rules():
    assert TINY_EDIT.is_edit and TINY_EDIT.latent_channels == 4 and SDXL_EDIT.in_channels == 8
    from dataclasses import replace
    plain8 = replace(TINY, in_channels=8)   # an 8 -> 4 cfg without the flag keeps its 8-channel latent
    assert not plain8.is_edit and not plain8.is_inpaint and plain8.latent_channels == 8
    assert _cfg_struct(plain8).edit_layout == 0 and _cfg_struct(TINY_EDIT).edit_layout == 1
    assert _cfg_struct(SDXL_BASE).edit_layout == 0


def _diffusers_config(in_channels):
    return {"in_channels": in_channels, "out_channels": 4, "block_out_channels": [64, 128, 256], "cross_attention_dim": 24,
            "down_block_types": ["DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"],
            "up_block_types": ["CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"], "attention_head_dim": [1, 2, 4],
            "transformer_layers_per_block": [1, 1, 2], "projection_class_embeddings_input_dim": 8, "addition_embed_type": "text_time",
            "addition_time_embed_dim": 256, "layers_per_block": 2, "use_linear_projection": True}


def test_from_diffusers_takes_eight_channels_as_the_edit_layout():
    cfg = config_from_diffusers(_diffusers_config(8))
    assert cfg.is_edit and cfg.in_channels == 8 and cfg.latent_channels == 4
    assert not config_from_diffusers(_diffusers_config(4)).is_edit and not config_from_diffusers(_diffusers_config(9)).is_edit
    with pytest.raises(SdxlError, match="in_channels = 7"):
        config_from_diffusers(_diffusers_config(7))
    # a synthetic state dict in diffusers' names round-trips to the pack names of TINY_EDIT
    w = synth_weights(TINY_EDIT, seed=0)
    m = name_map(cfg)
    sd = {}
    for dk, (pk, lin) in m.items():
        t = w[pk]
        sd[dk] = t.t().contiguous() if lin else t
    got_cfg, got = from_diffusers(sd, json.dumps(_diffusers_config(8)))
    assert got_cfg == cfg and got_cfg == TINY_EDIT
    assert torch.equal(got["input_blocks/0/weight"], w["input_blocks/0/weight"]) and got["input_blocks/0/weight"].shape[1] == 8


class _Stub:
    def __init__(self, cfg):
        self.cfg = cfg


def test_sample_refusals_without_a_gpu():
    img = torch.zeros(1, 64, 64, 3, dtype=torch.uint8)
    with pytest.raises(SdxlError, match="needs edit_image"):
        sample(None, _Stub(TINY_EDIT), None, "a cat")
    with pytest.raises(SdxlError, match="needs an edit UNet"):
        sample(None, _Stub(TINY), None, "a cat", edit_image=img)
    with pytest.raises(SdxlError, match="refiner"):
        sample(None, _Stub(TINY_EDIT), None, "a cat", refiner=_Stub(TINY), edit_image=img)


def test_burn_record_refuses_the_edit_layout(tmp_path):
    """DiffuserConfig has no field for the edit layout: saving an edit UNet as a burn record is refused before any file is written."""
    from sdxl_b200 import burn_record as BR
    path = str(tmp_path / "diffuser")
    with pytest.raises(BR.BurnRecordError, match="edit layout"):
        BR.save_diffuser(path, TINY_EDIT, synth_weights(TINY_EDIT, seed=0))
    assert not os.listdir(tmp_path)


def test_edit_abi_from_c(tmp_path):
    """A C99 program using the editing part of include/sdxl_b200.h compiles with -pedantic -Werror, links, is refused on a NULL UNet
    and sees the layout of sdxl_edit_image and sdxl_unet_cfg that the ctypes mirror has."""
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib_dir = os.path.join(ROOT, "stable-diffusion-xl-burn_b200", "sdxl_b200")
    exe = str(tmp_path / "edit_abi_check")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "c_abi", "edit_abi_check.c"), "-L", lib_dir, "-lsdxl_b200", "-Wl,-rpath," + lib_dir,
                        "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout.startswith("edit_abi_check ok"), (r.returncode, r.stdout, r.stderr)
    size, off, cfg_size = (int(v) for v in r.stdout.split()[-3:])
    assert size == C.sizeof(_lib.EditImage)
    assert off == _lib.UnetCfg.edit_layout.offset and cfg_size == C.sizeof(_lib.UnetCfg)
