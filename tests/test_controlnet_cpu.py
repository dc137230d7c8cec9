"""ControlNet host side: the diffusers name map, its rejections, the oracle's identities and the C ABI."""
import ctypes as C
import os
import shutil
import subprocess
from types import SimpleNamespace

import pytest
import torch

from sdxl_b200 import SDXL_CONTROLNET, TINY, TINY_CONTROLNET, SdxlError, _lib, controlnet_tensor_specs, synth_weights
from sdxl_b200.controlnet import diffusers_name_map, from_diffusers
from oracle import unet_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TINY_JSON = {"block_out_channels": [64, 128, 256], "down_block_types": ["DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"],
             "attention_head_dim": [1, 2, 4], "transformer_layers_per_block": [1, 1, 2], "cross_attention_dim": 24,
             "projection_class_embeddings_input_dim": 8, "conditioning_embedding_out_channels": [8, 16, 24, 32], "in_channels": 4,
             "conditioning_channels": 3, "global_pool_conditions": False, "controlnet_conditioning_channel_order": "rgb"}


def to_diffusers(cfg, w):
    """Inverse of from_diffusers on pack-named weights."""
    sd = {}
    for src, (dst, lin) in diffusers_name_map(cfg).items():
        sd[src] = w[dst].t().contiguous() if lin else w[dst]
    return sd


def test_name_map_covers_every_tensor_once():
    names = diffusers_name_map(SDXL_CONTROLNET)
    dst = [d for d, _ in names.values()]
    specs = [s[0] for s in controlnet_tensor_specs(SDXL_CONTROLNET)]
    assert len(dst) == len(set(dst)) and sorted(dst) == sorted(specs)
    assert len(specs) == len(set(specs))


def test_name_map_spot_checks():
    names = diffusers_name_map(SDXL_CONTROLNET)
    assert names["down_blocks.1.attentions.0.transformer_blocks.0.attn1.to_q.weight"] == \
        ("input_blocks/4/transformer/transformer_0/attn1/query/weight", True)
    assert names["controlnet_cond_embedding.blocks.5.weight"] == ("input_hint_block/12/weight", False)
    assert names["controlnet_cond_embedding.conv_out.bias"] == ("input_hint_block/14/bias", False)
    assert names["down_blocks.0.resnets.1.conv2.weight"] == ("input_blocks/2/conv_out/weight", False)
    assert names["down_blocks.1.resnets.0.conv_shortcut.weight"] == ("input_blocks/4/res/skip_connection/weight", False)
    assert names["down_blocks.1.downsamplers.0.conv.weight"] == ("input_blocks/6/weight", False)
    assert names["controlnet_down_blocks.8.weight"] == ("zero_convs/8/weight", False)
    assert names["controlnet_mid_block.weight"] == ("middle_block_out/weight", False)
    assert names["mid_block.attentions.0.transformer_blocks.9.ff.net.0.proj.weight"] == \
        ("middle_block/transformer/transformer_9/mlp/geglu/proj/weight", True)
    assert names["add_embedding.linear_2.weight"] == ("lin2_label_embed/weight", True)


def test_diffusers_round_trip():
    w = synth_weights(TINY_CONTROLNET, seed=3)
    cfg, back = from_diffusers(to_diffusers(TINY_CONTROLNET, w), dict(TINY_JSON))
    assert cfg == TINY_CONTROLNET
    assert set(back) == set(w)
    assert all(torch.equal(back[k], w[k]) for k in w)
    # "bgr": the first hint conv takes its input channels reversed
    _, bgr = from_diffusers(to_diffusers(TINY_CONTROLNET, w), dict(TINY_JSON, controlnet_conditioning_channel_order="bgr"))
    assert torch.equal(bgr["input_hint_block/0/weight"], w["input_hint_block/0/weight"].flip(1))


@pytest.mark.parametrize("key", ["control_model.input_blocks.0.0.weight", "task_embedding", "control_type_proj.weight",
                                 "lora_controlnet", "adapter.body.0.resnets.0.block1.weight"])
def test_foreign_formats_name_the_key(key):
    sd = to_diffusers(TINY_CONTROLNET, synth_weights(TINY_CONTROLNET, seed=0))
    sd[key] = torch.zeros(1, dtype=torch.float16)
    with pytest.raises(SdxlError, match=key.replace(".", r"\.")):
        from_diffusers(sd, dict(TINY_JSON))


@pytest.mark.parametrize("field,value", [("global_pool_conditions", True), ("attention_head_dim", [1, 1, 1]),
                                         ("down_block_types", ["DownBlock2D", "DownBlock2D", "CrossAttnDownBlock2D"])])
def test_unsupported_config_names_the_field(field, value):
    sd = to_diffusers(TINY_CONTROLNET, synth_weights(TINY_CONTROLNET, seed=0))
    with pytest.raises(SdxlError, match=field):
        from_diffusers(sd, dict(TINY_JSON, **{field: value}))


def test_unknown_key_is_named():
    sd = to_diffusers(TINY_CONTROLNET, synth_weights(TINY_CONTROLNET, seed=0))
    sd["down_blocks.0.resnets.2.conv1.weight"] = torch.zeros(1, dtype=torch.float16)
    with pytest.raises(SdxlError, match=r"down_blocks\.0\.resnets\.2\.conv1\.weight"):
        from_diffusers(sd, dict(TINY_JSON))


def test_synthetic_zero_convs_are_not_zero():
    w = synth_weights(TINY_CONTROLNET, seed=0)
    assert all(float(w[k].float().abs().max()) > 0 for k in w if k.startswith(("zero_convs/", "middle_block_out/")))


def small_inputs(n_hint=2):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 16, 16, generator=g)
    c = torch.randn(2, 7, TINY.context_dim, generator=g)
    y = torch.randn(2, TINY.adm_in_channels, generator=g)
    hint = torch.rand(n_hint, 3, 128, 128, generator=g)
    return x, c, y, hint


def test_oracle_zero_convs_leave_unet_unchanged():
    wu = O.to_f32(synth_weights(TINY, seed=0))
    wc = O.to_f32(synth_weights(TINY_CONTROLNET, seed=1))
    for k in wc:
        if k.startswith(("zero_convs/", "middle_block_out/")):
            wc[k] = torch.zeros_like(wc[k])
    x, c, y, hint = small_inputs()
    t = torch.tensor([499])
    att = O.Attach(controls=[(TINY_CONTROLNET, wc, hint, 1.0)])
    assert torch.equal(O.unet_forward(TINY, wu, x, t, c, y, att), O.unet_forward(TINY, wu, x, t, c, y))


def test_oracle_hint_embedding_shape():
    wc = O.to_f32(synth_weights(TINY_CONTROLNET, seed=1))
    e = O.hint_embedding(TINY_CONTROLNET, wc, torch.rand(3, 3, 64, 96))
    assert e.shape == (3, TINY.model_channels, 8, 12) and e.is_contiguous()
    res, mid = O.controlnet_forward(TINY_CONTROLNET, wc, torch.randn(2, 4, 8, 12), torch.tensor([9]), torch.randn(2, 5, 24),
                                    torch.randn(2, 8), e[:1])
    assert [tuple(r.shape[1:]) for r in res] == ([(64, 8, 12)] * 3 + [(64, 4, 6)] + [(128, 4, 6)] * 2 + [(128, 2, 3)] +
                                                 [(256, 2, 3)] * 2)
    assert tuple(mid.shape) == (2, 256, 2, 3)


def test_controlnet_symbols_exported():
    lib = _lib.load()
    for s in ("sdxl_controlnet_load", "sdxl_controlnet_destroy", "sdxl_unet_set_controls", "sdxl_controlnet_embed_hint"):
        assert hasattr(lib, s) and s in _lib.PROTOTYPES


def test_controlnet_abi_from_c(tmp_path):
    """A C99 program using the ControlNet part of include/sdxl_b200.h compiles, links and sees the struct layouts a binding needs."""
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib_dir = os.path.join(ROOT, "stable-diffusion-xl-burn_b200", "sdxl_b200")
    exe = str(tmp_path / "controlnet_abi_check")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "c_abi", "controlnet_abi_check.c"), "-L", lib_dir, "-lsdxl_b200", "-Wl,-rpath," + lib_dir,
                        "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout.startswith("controlnet_abi_check ok"), (r.returncode, r.stdout, r.stderr)
    n_max, s_ctl, s_cfg = (int(v) for v in r.stdout.split()[-3:])
    assert n_max == _lib.MAX_CONTROLS and s_ctl == C.sizeof(_lib.Control) and s_cfg == C.sizeof(_lib.ControlNetCfg)


class _NoLibrary:
    """Stands in for the library: any call fails the test."""
    def __getattr__(self, name):
        raise AssertionError(f"library call {name} made")


def _fake_net():
    from sdxl_b200.controlnet import ControlNet
    net = ControlNet.__new__(ControlNet)
    net.ctx = SimpleNamespace(lib=_NoLibrary(), device=torch.device("cpu"))
    net.cfg, net.h, net.attached = TINY_CONTROLNET, C.c_void_p(1), 0
    return net


@pytest.mark.parametrize("hint", [torch.rand(1, 1, 64, 64), torch.rand(1, 4, 64, 64), torch.rand(3, 64, 64),
                                  torch.zeros(1, 64, 64, 1, dtype=torch.uint8)])
def test_hint_shape_is_checked_before_any_library_call(hint):
    """The engine reads n * hint_in_channels * H * W floats from the hint pointer: a single-channel depth map must be refused."""
    from sdxl_b200.controlnet import set_controls
    net = _fake_net()
    diffuser = SimpleNamespace(ctx=net.ctx, h=C.c_void_p(2))
    with pytest.raises(SdxlError, match="control image"):
        set_controls(diffuser, [(net, hint, 1.0)])
    with pytest.raises(SdxlError, match="control image"):
        net.embed_hint(hint)


def test_close_is_refused_while_attached():
    net = _fake_net()
    net.attached = 1
    with pytest.raises(SdxlError, match="still attached"):
        net.close()
    assert net.h is not None

