"""Perturbed-attention guidance, host side: diffusers' pag_applied_layers resolved to the engine's self-attention mask, the per-step
scale, the oracle's perturbed rows, and the C ABI."""
import ctypes as C
import os
import shutil
import subprocess

import pytest
import torch

from sdxl_b200 import SDXL_BASE, SDXL_REFINER, TINY, TINY_REFINER, SdxlError, _lib, pag_layer_mask, pag_scale_at, self_attention_names
from sdxl_b200 import synth_weights
from sdxl_b200.diffusers_unet import name_map
from oracle import unet_oracle as O
import pag_oracle as PO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("cfg, n, n_mid", [(SDXL_BASE, 70, 10), (SDXL_REFINER, 44, 4), (TINY, 17, 2), (TINY_REFINER, 11, 1)])
def test_self_attention_count_and_mid(cfg, n, n_mid):
    names = self_attention_names(cfg)
    assert len(names) == n and len(set(names)) == n
    assert all(x.endswith(".attn1") for x in names)
    assert sum(pag_layer_mask(cfg, "mid")) == n_mid
    assert sum(pag_layer_mask(cfg, [".*"])) == n


@pytest.mark.parametrize("cfg", [SDXL_BASE, SDXL_REFINER, TINY, TINY_REFINER])
def test_names_are_in_engine_order(cfg):
    """Entry i of the mask is transformer block i in execution order: the diffusers name maps to the oracle's i-th block path."""
    m = name_map(cfg)
    got = [m[f"{x}.to_q.weight"][0] for x in self_attention_names(cfg)]
    assert got == [f"{p}/attn1/query/weight" for p in PO.self_attention_paths(cfg)]


def test_sdxl_base_selections():
    names = self_attention_names(SDXL_BASE)
    assert names[0] == "down_blocks.1.attentions.0.transformer_blocks.0.attn1"
    assert names[24] == "mid_block.attentions.0.transformer_blocks.0.attn1"
    assert names[-1] == "up_blocks.1.attentions.2.transformer_blocks.1.attn1"
    mid = pag_layer_mask(SDXL_BASE, "mid")
    assert [i for i, m in enumerate(mid) if m] == list(range(24, 34))
    assert sum(pag_layer_mask(SDXL_BASE, "down_blocks.2")) == 20
    sel = pag_layer_mask(SDXL_BASE, "up_blocks.1.attentions.0")
    assert [names[i] for i, m in enumerate(sel) if m] == [f"up_blocks.1.attentions.0.transformer_blocks.{j}.attn1" for j in (0, 1)]
    both = pag_layer_mask(SDXL_BASE, ["mid", "up_blocks.1.attentions.0"])
    assert both == [a | b for a, b in zip(mid, sel)]
    assert pag_layer_mask(SDXL_BASE, r"down_blocks\.1\.attentions\.1\.transformer_blocks\.0") == [int(i == 2) for i in range(70)]


def test_unmatched_ids_raise():
    with pytest.raises(SdxlError, match="matches no self-attention"):
        pag_layer_mask(SDXL_BASE, "down_blocks.0")          # the transformer-free level
    with pytest.raises(SdxlError, match="'mid_blocks'"):
        pag_layer_mask(SDXL_BASE, ["mid", "mid_blocks"])
    with pytest.raises(SdxlError, match="no layer ids"):
        pag_layer_mask(SDXL_BASE, [])


def test_pag_scale_at():
    assert pag_scale_at(999, 3.0) == 3.0 and pag_scale_at(0, 3.0) == 3.0
    assert pag_scale_at(999, 3.0, 0.01) == pytest.approx(2.99)
    assert pag_scale_at(800, 3.0, 0.01) == pytest.approx(1.0)
    assert pag_scale_at(700, 3.0, 0.01) == 0.0                # clamped at 0
    assert pag_scale_at(40, 3.0, 0.1, total=50) == pytest.approx(2.0)
    for t in range(0, 1000, 37):
        assert pag_scale_at(t, 3.0, 0.005) == PO.pag_scale(t, 3.0, 0.005, 1000)


def test_oracle_without_layers_is_unet_oracle():
    w = O.to_f32(synth_weights(TINY, seed=0))
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 4, 16, 16, generator=g)
    ctx, y = torch.randn(2, 7, TINY.context_dim, generator=g), torch.randn(2, TINY.adm_in_channels, generator=g)
    t = torch.tensor([499])
    layers = PO.paths_of_mask(TINY, pag_layer_mask(TINY, "mid"))
    assert layers == ["middle_block/transformer/transformer_0", "middle_block/transformer/transformer_1"]
    ptb = PO.forward_rows(TINY, w, x, t, ctx, y, layers, 1)
    assert torch.equal(ptb[0], O.unet_forward(TINY, w, x[:1], t, ctx[:1], y[:1])[0])
    assert not torch.allclose(ptb[1], O.unet_forward(TINY, w, x[1:], t, ctx[1:], y[1:])[0], atol=1e-3)


def test_pag_abi_from_c(tmp_path):
    """A C99 program using the PAG part of include/sdxl_b200.h compiles with -pedantic -Werror, links and sees the layout."""
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib_dir = os.path.join(ROOT, "stable-diffusion-xl-burn_b200", "sdxl_b200")
    exe = str(tmp_path / "pag_abi_check")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "c_abi", "pag_abi_check.c"), "-L", lib_dir, "-lsdxl_b200", "-Wl,-rpath," + lib_dir,
                        "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout.startswith("pag_abi_check ok"), (r.returncode, r.stdout, r.stderr)
    assert int(r.stdout.split()[-1]) == C.sizeof(_lib.Pag)
