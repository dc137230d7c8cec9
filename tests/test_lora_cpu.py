"""CPU tests of the LoRA host side: the `.safetensors` reader, the kohya -> reference name map, rejection of unsupported
formats, the host merge formula and the C ABI of the adapter entry points."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from sdxl_b200 import (SDXL_BASE, SDXL_CLIP_L, SDXL_OPEN_CLIP_G, SDXL_REFINER, TINY, TINY_CLIP, TINY_OPEN_CLIP, TINY_REFINER,
                       _lib, synth_weights)
from sdxl_b200.lora import clip_lora_modules, from_kohya, load_kohya, merge_into, read_safetensors, unet_lora_modules
from lora_cases import layer_paths, make_adapter, numpy_merge, to_kohya, write_safetensors

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_safetensors_hand_written(tmp_path):
    a = torch.arange(6, dtype=torch.float32).reshape(2, 3) / 7
    b = torch.tensor([[1.5, -2.25]], dtype=torch.float16)
    c = torch.tensor([0.1, 3.0, -7.5], dtype=torch.bfloat16)
    s = torch.tensor(4.0)
    p = tmp_path / "x.safetensors"
    write_safetensors(p, {"a": a, "b": b, "c": c, "s": s}, metadata={"ss_network_dim": "4"})
    got = read_safetensors(str(p))
    assert set(got) == {"a", "b", "c", "s"}
    for k, t in (("a", a), ("b", b), ("c", c), ("s", s)):
        assert got[k].dtype == t.dtype and got[k].shape == t.shape and torch.equal(got[k], t)
    assert read_safetensors(p.read_bytes())["b"].tolist() == [[1.5, -2.25]]


def test_safetensors_rejects_bad_files(tmp_path):
    with pytest.raises(ValueError, match="dtype"):
        hdr = b'{"x": {"dtype": "I64", "shape": [1], "data_offsets": [0, 8]}}'
        read_safetensors(len(hdr).to_bytes(8, "little") + hdr + bytes(8))
    with pytest.raises(ValueError, match="data_offsets"):
        hdr = b'{"x": {"dtype": "F16", "shape": [4], "data_offsets": [0, 6]}}'
        read_safetensors(len(hdr).to_bytes(8, "little") + hdr + bytes(6))
    with pytest.raises(ValueError, match="truncated"):
        read_safetensors((1000).to_bytes(8, "little") + b"{}")


def test_safetensors_matches_package(tmp_path):
    st = pytest.importorskip("safetensors.torch")
    g = torch.Generator().manual_seed(0)
    t = {"lora_unet_out_2.lora_down.weight": torch.randn(4, 320, 3, 3, generator=g).half(),
         "lora_unet_out_2.lora_up.weight": torch.randn(4, 4, 1, 1, generator=g).to(torch.bfloat16),
         "lora_unet_out_2.alpha": torch.tensor(2.0)}
    p = str(tmp_path / "pkg.safetensors")
    st.save_file(t, p)
    ours, theirs = read_safetensors(p), st.load_file(p)
    assert set(ours) == set(theirs)
    for k in ours:
        assert ours[k].dtype == theirs[k].dtype and torch.equal(ours[k], theirs[k])


@pytest.mark.parametrize("cfg,total,attn", [(TINY, 264, 192), (TINY_REFINER, 204, 132), (SDXL_BASE, 794, 722), (SDXL_REFINER, 554, 462)])
def test_unet_map_covers_every_module(cfg, total, attn):
    """Every Linear and conv of the UNet weight tree has exactly one kohya name. 722 is the count kohya's sd-scripts reports for
    SDXL base's transformer Linears (attention, FF, proj_in/out)."""
    mods = unet_lora_modules(cfg)
    refs = [r for _, r, _ in mods]
    assert len(mods) == total and len(set(refs)) == total and len({k for k, _, _ in mods}) == total
    assert sum("/transformer" in r for r in refs) == attn
    from lora_cases import weight_shapes
    shapes = weight_shapes(cfg)
    assert set(refs) == set(shapes), "map and weight tree disagree"
    for _, r, kind in mods:
        assert (len(shapes[r]) == 2) == (kind == "linear")


def test_unet_map_names():
    m = {r: k for k, r, _ in unet_lora_modules(SDXL_BASE)}
    assert m["input_blocks/4/transformer/transformer_0/attn1/query"] == "lora_unet_input_blocks_4_1_transformer_blocks_0_attn1_to_q"
    assert m["input_blocks/4/transformer/transformer_0/attn2/out"] == "lora_unet_input_blocks_4_1_transformer_blocks_0_attn2_to_out_0"
    assert m["input_blocks/4/transformer/transformer_0/mlp/geglu/proj"] == "lora_unet_input_blocks_4_1_transformer_blocks_0_ff_net_0_proj"
    assert m["input_blocks/4/transformer/transformer_0/mlp/lin"] == "lora_unet_input_blocks_4_1_transformer_blocks_0_ff_net_2"
    assert m["input_blocks/4/res/conv_in"] == "lora_unet_input_blocks_4_0_in_layers_2"
    assert m["input_blocks/4/res/lin_embed"] == "lora_unet_input_blocks_4_0_emb_layers_1"
    assert m["input_blocks/4/res/skip_connection"] == "lora_unet_input_blocks_4_0_skip_connection"
    assert m["input_blocks/1/conv_out"] == "lora_unet_input_blocks_1_0_out_layers_3"
    assert m["input_blocks/3"] == "lora_unet_input_blocks_3_0_op"
    assert m["input_blocks/0"] == "lora_unet_input_blocks_0_0"
    assert m["middle_block/transformer/proj_in"] == "lora_unet_middle_block_1_proj_in"
    assert m["middle_block/res2/conv_out"] == "lora_unet_middle_block_2_out_layers_3"
    assert m["output_blocks/2/upsample/conv"] == "lora_unet_output_blocks_2_2_conv"
    assert m["lin1_time_embed"] == "lora_unet_time_embed_0" and m["lin2_label_embed"] == "lora_unet_label_emb_0_2"
    assert m["conv_out"] == "lora_unet_out_2"
    r = {r: k for k, r, _ in unet_lora_modules(SDXL_REFINER)}
    assert r["output_blocks/2/upsample/conv"] == "lora_unet_output_blocks_2_1_conv"   # non-transformer level: Upsample is block[1]


@pytest.mark.parametrize("cfg,n", [(SDXL_CLIP_L, 72), (SDXL_OPEN_CLIP_G, 192), (TINY_CLIP, 18), (TINY_OPEN_CLIP, 24)])
def test_clip_map_covers_every_module(cfg, n):
    mods = clip_lora_modules(cfg, "lora_te2")
    from lora_cases import weight_shapes
    shapes = weight_shapes(cfg, clip=True)
    assert len(mods) == n and len({r for _, r, _ in mods}) == n
    assert {r for _, r, _ in mods} == set(shapes) - {"token_embedding", "position_embedding"}
    m = {r: k for k, r, _ in mods}
    assert m["blocks/0/attn/query"] == "lora_te2_text_model_encoder_layers_0_self_attn_q_proj"
    assert m["blocks/1/attn/out"] == "lora_te2_text_model_encoder_layers_1_self_attn_out_proj"
    assert m["blocks/1/mlp/fc2"] == "lora_te2_text_model_encoder_layers_1_mlp_fc2"


def test_from_kohya_roundtrip(tmp_path):
    ad = make_adapter(TINY, layer_paths(TINY)[:20], rank=4, seed=0, alpha=2.0)
    te = make_adapter(TINY_CLIP, ["blocks/0/attn/query", "blocks/2/mlp/fc1"], rank=2, seed=1, clip=True)
    k = to_kohya(ad, unet_lora_modules(TINY))
    k.update(to_kohya(te, clip_lora_modules(TINY_CLIP, "lora_te1")))
    k = {n: (t.float() if n.endswith("lora_up.weight") else t) for n, t in k.items()}   # f32 factors are converted to f16
    p = tmp_path / "k.safetensors"
    write_safetensors(p, k)
    out = load_kohya(str(p), TINY, TINY_CLIP, TINY_OPEN_CLIP)
    assert set(out["unet"]) == set(ad) and set(out["te1"]) == set(te) and out["te2"] == {}
    for n in ad:
        assert out["unet"][n].dtype == (torch.float32 if n.endswith("alpha") else torch.float16) and torch.equal(out["unet"][n].float(), ad[n].float())


@pytest.mark.parametrize("key,what", [
    ("lora_unet_down_blocks_1_attentions_0_transformer_blocks_0_attn1_to_q.lora_down.weight", "diffusers"),
    ("unet.down_blocks.1.attentions.0.transformer_blocks.0.attn1.to_q.lora.down.weight", "diffusers"),
    ("lora_unet_input_blocks_4_1_transformer_blocks_0_attn1_to_q.hada_w1_a", "LyCORIS"),
    ("lora_unet_input_blocks_4_1_transformer_blocks_0_attn1_to_q.lokr_w1", "LyCORIS"),
    ("lora_unet_input_blocks_4_1_transformer_blocks_0_attn1_to_q.dora_scale", "DoRA"),
    ("lora_unet_input_blocks_4_1_transformer_blocks_0_norm1.diff", "norm or bias"),
    ("lora_unet_input_blocks_4_1_proj_in.diff_b", "norm or bias"),
    ("lora_unet_not_a_module.lora_up.weight", "known module"),
])
def test_unsupported_formats_name_the_key(key, what):
    good = to_kohya(make_adapter(SDXL_BASE, ["conv_out"], rank=1, seed=0), unet_lora_modules(SDXL_BASE))
    good[key] = torch.zeros(1, dtype=torch.float16)
    with pytest.raises(ValueError) as e:
        from_kohya(good, SDXL_BASE, SDXL_CLIP_L, SDXL_OPEN_CLIP_G)
    assert key in str(e.value) and what in str(e.value)


def test_text_encoder_keys_need_their_config():
    k = to_kohya(make_adapter(TINY_CLIP, ["blocks/0/mlp/fc1"], rank=1, seed=0, clip=True), clip_lora_modules(TINY_CLIP, "lora_te1"))
    with pytest.raises(ValueError, match="lora_te1_text_model_encoder_layers_0_mlp_fc1"):
        from_kohya(k, TINY)


def test_merge_into_matches_numpy_formula():
    w = synth_weights(TINY, seed=0)
    paths = ["input_blocks/4/transformer/transformer_0/attn1/key", "input_blocks/4/res/skip_connection", "input_blocks/0",
             "output_blocks/2/upsample/conv", "lin1_label_embed"]
    for dyadic, scale, alpha in ((True, 0.5, None), (False, 0.8, 3.0)):
        ad = make_adapter(TINY, paths, rank=3, seed=7, dyadic=dyadic, alpha=alpha)
        m = merge_into(w, ad, scale)
        assert set(m) == set(w)
        for p in paths:
            ref = numpy_merge(w[p + "/weight"].numpy(), ad[p + "/lora_down"].numpy(), ad[p + "/lora_up"].numpy(), scale,
                              3.0 if alpha is None else alpha)
            assert np.array_equal(m[p + "/weight"].numpy().view(np.uint16), ref.astype(np.float16).view(np.uint16)), p
            assert not torch.equal(m[p + "/weight"], w[p + "/weight"])
        untouched = [k for k in w if k.rsplit("/", 1)[0] not in paths]
        assert all(m[k] is w[k] for k in untouched)
    # up = 0: bit-identical weights
    z = merge_into(w, make_adapter(TINY, paths, rank=2, seed=1, zero_up=True), 1.0)
    assert all(torch.equal(z[k].view(torch.int16), w[k].view(torch.int16)) for k in w)


def test_adapter_symbols_exported():
    lib = _lib.load()
    for s in ("sdxl_unet_set_adapters", "sdxl_clip_set_adapters"):
        assert hasattr(lib, s) and s in _lib.PROTOTYPES


def test_adapter_abi_from_c(tmp_path):
    """A C99 program using the adapter part of include/sdxl_b200.h compiles, links and sees the struct layout a binding needs."""
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib_dir = os.path.join(ROOT, "stable-diffusion-xl-burn_b200", "sdxl_b200")
    exe = str(tmp_path / "lora_abi_check")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "c_abi", "lora_abi_check.c"), "-L", lib_dir, "-lsdxl_b200", "-Wl,-rpath," + lib_dir, "-o", exe],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout.startswith("lora_abi_check ok"), (r.returncode, r.stdout, r.stderr)
    import ctypes as C
    assert C.sizeof(_lib.Adapter) == int(r.stdout.split()[-1])
