"""Inpainting UNet, host side: the diffusers UNet2DConditionModel config and key map, their refusals, the condition's preparation
against the oracle's restatement, and the C ABI."""
import ctypes as C
import os
import shutil
import subprocess
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from sdxl_b200 import SDXL_BASE, SDXL_INPAINT, TINY, TINY_INPAINT, SdxlError, _lib, make_inpaint_mask, prepare_inpaint_condition, synth_weights
from sdxl_b200 import unet_tensor_specs
from sdxl_b200.diffusers_unet import config_from_diffusers, from_diffusers, name_map
import inpaint_oracle as IO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the fields of the published SDXL inpainting UNet's config.json (diffusers/stable-diffusion-xl-1.0-inpainting-0.1, unet/)
SDXL_INPAINT_JSON = {
    "_class_name": "UNet2DConditionModel", "act_fn": "silu", "addition_embed_type": "text_time", "addition_embed_type_num_heads": 64,
    "addition_time_embed_dim": 256, "attention_head_dim": [5, 10, 20], "block_out_channels": [320, 640, 1280], "center_input_sample": False,
    "class_embed_type": None, "class_embeddings_concat": False, "conv_in_kernel": 3, "conv_out_kernel": 3, "cross_attention_dim": 2048,
    "cross_attention_norm": None, "down_block_types": ["DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"], "downsample_padding": 1,
    "dual_cross_attention": False, "encoder_hid_dim": None, "encoder_hid_dim_type": None, "flip_sin_to_cos": True, "freq_shift": 0,
    "in_channels": 9, "layers_per_block": 2, "mid_block_only_cross_attention": None, "mid_block_scale_factor": 1,
    "mid_block_type": "UNetMidBlock2DCrossAttn", "norm_eps": 1e-05, "norm_num_groups": 32, "num_attention_heads": None, "num_class_embeds": None,
    "only_cross_attention": False, "out_channels": 4, "projection_class_embeddings_input_dim": 2816, "resnet_out_scale_factor": 1.0,
    "resnet_skip_time_act": False, "resnet_time_scale_shift": "default", "sample_size": 128, "time_cond_proj_dim": None,
    "time_embedding_act_fn": None, "time_embedding_dim": None, "time_embedding_type": "positional", "timestep_post_act": None,
    "transformer_layers_per_block": [1, 2, 10], "up_block_types": ["CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"],
    "upcast_attention": None, "use_linear_projection": True}
TINY_JSON = dict(SDXL_INPAINT_JSON, attention_head_dim=[1, 2, 4], block_out_channels=[64, 128, 256], cross_attention_dim=24,
                 projection_class_embeddings_input_dim=8, transformer_layers_per_block=[1, 1, 2], in_channels=4)


def to_diffusers(cfg, w):
    """Inverse of from_diffusers on pack-named weights."""
    return {src: (w[dst].t().contiguous() if lin else w[dst]) for src, (dst, lin) in name_map(cfg).items()}


def test_config_of_the_published_files():
    assert config_from_diffusers(SDXL_INPAINT_JSON) == SDXL_INPAINT
    assert config_from_diffusers(dict(SDXL_INPAINT_JSON, in_channels=4)) == SDXL_BASE
    assert config_from_diffusers(TINY_JSON) == TINY and config_from_diffusers(dict(TINY_JSON, in_channels=9)) == TINY_INPAINT
    assert SDXL_INPAINT.is_inpaint and SDXL_INPAINT.latent_channels == 4 and not SDXL_BASE.is_inpaint and SDXL_BASE.latent_channels == 4


@pytest.mark.parametrize("cfg", [SDXL_INPAINT, SDXL_BASE], ids=["inpaint", "base"])
def test_name_map_covers_every_tensor_once(cfg):
    names = name_map(cfg)
    specs = {n: (shape, kind) for n, shape, kind, _ in unet_tensor_specs(cfg)}
    dst = [d for d, _ in names.values()]
    assert len(dst) == len(set(dst)) and sorted(dst) == sorted(specs)
    for src, (d, lin) in names.items():
        assert lin == (specs[d][1] == "linear"), src      # Linear weights, and only they, are transposed
    assert specs["input_blocks/0/weight"][0] == (320, cfg.in_channels, 3, 3)


def test_name_map_spot_checks():
    m = name_map(SDXL_INPAINT)
    assert m["conv_in.weight"] == ("input_blocks/0/weight", False)
    assert m["up_blocks.0.resnets.0.conv_shortcut.weight"] == ("output_blocks/0/res/skip_connection/weight", False)
    assert m["up_blocks.0.attentions.2.transformer_blocks.9.attn2.to_k.weight"] == \
        ("output_blocks/2/transformer/transformer_9/attn2/key/weight", True)
    assert m["up_blocks.0.upsamplers.0.conv.weight"] == ("output_blocks/2/upsample/conv/weight", False)
    assert m["up_blocks.1.upsamplers.0.conv.bias"] == ("output_blocks/5/upsample/conv/bias", False)
    assert m["up_blocks.2.resnets.2.conv2.weight"] == ("output_blocks/8/conv_out/weight", False)
    assert "up_blocks.2.upsamplers.0.conv.weight" not in m and "up_blocks.2.attentions.0.norm.weight" not in m
    assert m["conv_norm_out.weight"] == ("norm_out/weight", False) and m["conv_out.bias"] == ("conv_out/bias", False)
    assert m["mid_block.attentions.0.proj_in.weight"] == ("middle_block/transformer/proj_in/weight", True)


@pytest.mark.parametrize("cfg,js", [(TINY_INPAINT, dict(TINY_JSON, in_channels=9)), (TINY, TINY_JSON)], ids=["inpaint", "base"])
def test_diffusers_round_trip(cfg, js):
    w = synth_weights(cfg, seed=3)
    got_cfg, back = from_diffusers(to_diffusers(cfg, w), js)
    assert got_cfg == cfg and set(back) == set(w)
    assert all(torch.equal(back[k], w[k]) for k in w)


@pytest.mark.parametrize("field,value", [
    ("up_block_types", ["UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D"]),
    ("down_block_types", ["DownBlock2D", "DownBlock2D", "CrossAttnDownBlock2D"]), ("attention_head_dim", [1, 1, 1]),
    ("addition_embed_type", "text"), ("class_embed_type", "timestep"), ("use_linear_projection", False), ("in_channels", 5),
    ("out_channels", 8), ("layers_per_block", 3), ("time_cond_proj_dim", 256)])
def test_unsupported_config_names_the_field(field, value):
    with pytest.raises(SdxlError, match=field):
        config_from_diffusers(dict(TINY_JSON, **{field: value}))


def test_keys_and_shapes_are_named():
    sd = to_diffusers(TINY_INPAINT, synth_weights(TINY_INPAINT, seed=0))
    js = dict(TINY_JSON, in_channels=9)
    bad = dict(sd, **{"up_blocks.2.attentions.0.norm.weight": torch.zeros(64, dtype=torch.float16)})
    with pytest.raises(SdxlError, match=r"unexpected key 'up_blocks\.2\.attentions\.0\.norm\.weight'"):
        from_diffusers(bad, js)
    bad = {k: v for k, v in sd.items() if k != "up_blocks.1.upsamplers.0.conv.bias"}
    with pytest.raises(SdxlError, match=r"up_blocks\.1\.upsamplers\.0\.conv\.bias' is missing"):
        from_diffusers(bad, js)
    bad = dict(sd, **{"conv_in.weight": sd["conv_in.weight"][:, :4].contiguous()})   # a 4-channel conv_in under a 9-channel config
    with pytest.raises(SdxlError, match=r"conv_in\.weight' has shape \(64, 4, 3, 3\), expected \(64, 9, 3, 3\)"):
        from_diffusers(bad, js)
    bad = dict(sd, **{"time_embedding.linear_1.weight": sd["time_embedding.linear_1.weight"].t().contiguous()})
    with pytest.raises(SdxlError, match=r"time_embedding\.linear_1\.weight' has shape"):
        from_diffusers(bad, js)


class FakeDecoder:
    """A CPU stand-in for LatentDecoder.encode_image (8x average pool), so the preparation can be checked without a GPU."""
    ctx = SimpleNamespace(device=torch.device("cpu"))

    @staticmethod
    def encode_image(x):
        return F.avg_pool2d(x, 8) * 0.5


@pytest.mark.parametrize("crop,crop_out", [((5, 27, 3, 19), False), ((5, 27, 3, 19), True), ((None, 13, 9, None), False),
                                           ((0, 40, 0, 24), True)])
def test_prepare_matches_the_oracle(crop, crop_out):
    H, W = 24, 40
    rgb = torch.randint(0, 256, (2, H, W, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(1))
    mask = make_inpaint_mask((H, W), (H, W), *crop, crop_out=crop_out, n_channels=1)
    want = IO.pixel_mask(H, W, *crop, crop_out)
    assert torch.equal(mask, want)
    mask = mask.expand(2, 1, H, W)
    got = prepare_inpaint_condition(FakeDecoder, rgb, mask)
    ref = IO.condition(rgb, mask, FakeDecoder.encode_image, 8)
    assert got.shape == (2, 4, H // 8, W // 8) and torch.equal(got[:, :1], ref[:, :1])
    assert torch.allclose(got, ref, rtol=0, atol=1e-6)
    # repaint pixels are zero in the masked image, kept ones are the image in [-1, 1]
    _, masked = IO.prepare(rgb, mask, 8)
    assert bool((masked[mask.expand(2, 3, H, W)] == 0).all())


def test_prepare_refuses_bad_shapes():
    rgb = torch.zeros(1, 16, 16, 3, dtype=torch.uint8)
    with pytest.raises(SdxlError, match="mask"):
        prepare_inpaint_condition(FakeDecoder, rgb, torch.zeros(1, 1, 8, 16, dtype=torch.bool))
    with pytest.raises(SdxlError, match="u8"):
        prepare_inpaint_condition(FakeDecoder, rgb.float(), torch.zeros(1, 1, 16, 16, dtype=torch.bool))


def test_inpaint_abi_from_c(tmp_path):
    """A C99 program using the inpainting part of include/sdxl_b200.h compiles with -pedantic -Werror, links and sees the layout."""
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib_dir = os.path.join(ROOT, "stable-diffusion-xl-burn_b200", "sdxl_b200")
    exe = str(tmp_path / "inpaint_abi_check")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "c_abi", "inpaint_abi_check.c"), "-L", lib_dir, "-lsdxl_b200", "-Wl,-rpath," + lib_dir,
                        "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout.startswith("inpaint_abi_check ok"), (r.returncode, r.stdout, r.stderr)
    assert int(r.stdout.split()[-1]) == C.sizeof(_lib.InpaintCondition)
