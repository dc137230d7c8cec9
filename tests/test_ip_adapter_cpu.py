"""CPU tests of IP-Adapter support: the h94 key map (flat and nested files, the odd attn2 indices, rejections by name), the
oracle's decoupled attention against two scaled_dot_product_attention calls, the oracle at scale 0 against no prompt, the
embedding-shape checks made before any library call, and a C program against the header."""
import ctypes as C
import os
import shutil
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from sdxl_b200 import SDXL_BASE, SDXL_REFINER, TINY, SdxlError, synth_weights
from sdxl_b200 import _lib
from sdxl_b200.ip_adapter import from_h94, ip_index_map, ip_tensor_specs, set_image_prompt, transformer_block_paths
from oracle import unet_oracle as O
import ip_adapter_oracle as IPO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def h94_state_dict(cfg, D, nested=False, tokens=4, seed=0):
    """A synthetic h94-layout IP-Adapter (diffusers [out, in] Linears) for `cfg`."""
    g = torch.Generator().manual_seed(seed)
    ctx = cfg.context_dim
    proj = {"proj.weight": torch.randn(tokens * ctx, D, generator=g).half(), "proj.bias": torch.randn(tokens * ctx, generator=g).half(),
            "norm.weight": torch.randn(ctx, generator=g).half(), "norm.bias": torch.randn(ctx, generator=g).half()}
    specs = dict(ip_tensor_specs(cfg, D))
    ip = {}
    for i, path in ip_index_map(cfg).items():
        c = specs[f"{path}/attn2/ip_key/weight"][1]
        ip[f"{i}.to_k_ip.weight"] = torch.randn(c, ctx, generator=g).half()
        ip[f"{i}.to_v_ip.weight"] = torch.randn(c, ctx, generator=g).half()
    if nested:
        return {"image_proj": proj, "ip_adapter": ip}
    return {**{f"image_proj.{k}": v for k, v in proj.items()}, **{f"ip_adapter.{k}": v for k, v in ip.items()}}


def test_index_map_sdxl_base():
    m = ip_index_map(SDXL_BASE)
    assert sorted(m) == list(range(1, 140, 2))   # 70 cross-attentions, attn2 at the odd indices
    assert sorted(m.values()) == sorted(transformer_block_paths(SDXL_BASE))
    # down_blocks.1 (4), down_blocks.2 (20), up_blocks.0 (30), up_blocks.1 (6), mid_block (10)
    assert m[1] == "input_blocks/4/transformer/transformer_0"
    assert m[7] == "input_blocks/5/transformer/transformer_1"
    assert m[9] == "input_blocks/7/transformer/transformer_0"
    assert m[47] == "input_blocks/8/transformer/transformer_9"
    assert m[49] == "output_blocks/0/transformer/transformer_0"
    assert m[107] == "output_blocks/2/transformer/transformer_9"
    assert m[109] == "output_blocks/3/transformer/transformer_0"
    assert m[119] == "output_blocks/5/transformer/transformer_1"
    assert m[121] == "middle_block/transformer/transformer_0"
    assert m[139] == "middle_block/transformer/transformer_9"


@pytest.mark.parametrize("nested", [False, True])
def test_from_h94_round_trip(nested):
    sd = h94_state_dict(TINY, 16, nested)
    D, w = from_h94(sd, TINY)
    assert D == 16
    assert sorted(w) == sorted(n for n, _ in ip_tensor_specs(TINY, 16))
    for n, shape in ip_tensor_specs(TINY, 16):
        assert tuple(w[n].shape) == shape, n
    flat = h94_state_dict(TINY, 16)
    assert torch.equal(w["image_proj/proj/weight"], flat["image_proj.proj.weight"].t())
    i, path = next(iter(ip_index_map(TINY).items()))
    assert torch.equal(w[f"{path}/attn2/ip_value/weight"], flat[f"ip_adapter.{i}.to_v_ip.weight"].t())


@pytest.mark.parametrize("key,match", [("image_proj.latents", "Plus"), ("image_proj.layers.0.0.to_q.weight", "Plus"),
                                       ("image_proj.proj_in.weight", "Plus"), ("image_proj.proj.0.weight", "FaceID"),
                                       ("ip_adapter.1.to_k_lora.down.weight", "FaceID")])
def test_foreign_files_rejected_by_name(key, match):
    sd = h94_state_dict(TINY, 16)
    sd[key] = torch.zeros(4, 4)
    with pytest.raises(SdxlError, match=match) as e:
        from_h94(sd, TINY)
    assert key in str(e.value)


def test_other_token_count_and_missing_or_extra_keys_rejected():
    with pytest.raises(SdxlError, match="16 tokens per image"):
        from_h94(h94_state_dict(TINY, 16, tokens=16), TINY)
    sd = h94_state_dict(TINY, 16)
    del sd["ip_adapter.3.to_v_ip.weight"]
    with pytest.raises(SdxlError, match="ip_adapter.3.to_v_ip.weight"):
        from_h94(sd, TINY)
    sd = h94_state_dict(TINY, 16)
    sd["ip_adapter.35.to_k_ip.weight"] = sd["ip_adapter.1.to_k_ip.weight"]
    with pytest.raises(SdxlError, match="ip_adapter.35"):
        from_h94(sd, TINY)
    with pytest.raises(SdxlError, match="refiner"):
        from_h94(h94_state_dict(TINY, 16), SDXL_REFINER)


@pytest.mark.parametrize("S_ip", [4, 16, 129])
def test_oracle_ip_attention_is_two_sdpa_calls(S_ip):
    g = torch.Generator().manual_seed(S_ip)
    B, T, S, nh = 2, 50, 77, 3
    q, k, v = (torch.randn(B, n, 64 * nh, generator=g) for n in (T, S, S))
    kip, vip = (torch.randn(B, S_ip, 64 * nh, generator=g) for _ in range(2))
    heads = lambda t: t.reshape(B, -1, nh, 64).transpose(1, 2)  # noqa: E731
    want = (F.scaled_dot_product_attention(heads(q), heads(k), heads(v))
            + 0.6 * F.scaled_dot_product_attention(heads(q), heads(kip), heads(vip))).transpose(1, 2).reshape(B, T, -1)
    got = IPO.ip_attention(q, k, v, kip, vip, nh, 0.6)
    assert float((got - want).norm() / want.norm()) < 1e-5


def test_oracle_zero_scale_is_no_prompt():
    from sdxl_b200.ip_adapter import synth_ip_adapter
    w = O.to_f32(synth_weights(TINY, seed=0))
    wa = O.to_f32(synth_ip_adapter(TINY, 16, seed=1))
    x = torch.randn(1, 4, 16, 16, generator=torch.Generator().manual_seed(1))
    c, y = torch.randn(1, 7, TINY.context_dim), torch.randn(1, TINY.adm_in_channels)
    tok = IPO.prompt_tokens(wa, torch.randn(1, 2, 16))
    t = torch.tensor([499])
    base = O.unet_forward(TINY, w, x, t, c, y)
    prompt = lambda s: O.Attach(prompts=[(wa, tok, IPO.uniform_scales(TINY, s), None)])  # noqa: E731
    assert torch.allclose(O.unet_forward(TINY, w, x, t, c, y, prompt(0.0)), base, atol=1e-6)
    assert not torch.allclose(O.unet_forward(TINY, w, x, t, c, y, prompt(1.0)), base, atol=1e-3)


class _NoLibrary:
    """Stands in for the library: any call fails the test."""
    def __getattr__(self, name):
        raise AssertionError(f"library call {name} made")


@pytest.mark.parametrize("embeds,scale", [(torch.zeros(2, 1, 15), 1.0), (torch.zeros(16), 1.0), (torch.zeros(2, 16), [1.0, 2.0])])
def test_prompt_checked_before_any_library_call(embeds, scale):
    """The engine reads n_batch * n_images * D floats from the pointer and n_tblocks per-block scales."""
    from sdxl_b200.ip_adapter import IPAdapter
    ad = IPAdapter.__new__(IPAdapter)
    ad.ctx = SimpleNamespace(lib=_NoLibrary(), device=torch.device("cpu"))
    ad.cfg, ad.image_embed_dim, ad.h, ad.attached = TINY, 16, C.c_void_p(1), 0
    diffuser = SimpleNamespace(ctx=ad.ctx, h=C.c_void_p(2), cfg=TINY)
    with pytest.raises(SdxlError):
        set_image_prompt(diffuser, ad, embeds, scale)
    assert ad.attached == 0


def test_ip_adapter_abi_check_compiles_and_runs(tmp_path):
    gcc = shutil.which("gcc") or shutil.which("cc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib_dir = os.path.join(ROOT, "stable-diffusion-xl-burn_b200", "sdxl_b200")
    exe = str(tmp_path / "ip_adapter_abi_check")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "c_abi", "ip_adapter_abi_check.c"), "-L", lib_dir, "-lsdxl_b200", "-Wl,-rpath," + lib_dir,
                        "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout.startswith("ip_adapter_abi_check ok"), (r.returncode, r.stdout, r.stderr)
    s_vcfg, s_prompt, s_cfg = (int(v) for v in r.stdout.split()[-3:])
    assert s_vcfg == C.sizeof(_lib.ClipVisionCfg) and s_prompt == C.sizeof(_lib.ImagePrompt) and s_cfg == C.sizeof(_lib.IpAdapterCfg)


def test_vision_hf_name_map_round_trip_and_config():
    from sdxl_b200.clip_vision import (SDXL_VIT_BIGG, SDXL_VIT_H, TINY_VIT_80, config_from_hf, from_hf, hf_name_map, synth_vision_weights,
                                       to_hf, vision_tensor_specs)
    w = synth_vision_weights(TINY_VIT_80, seed=0)
    assert sorted(w) == sorted(n for n, _, _ in vision_tensor_specs(TINY_VIT_80))
    hf = to_hf(w, TINY_VIT_80)
    hf["vision_model.embeddings.position_ids"] = torch.arange(TINY_VIT_80.n_tokens)[None]
    cfg, back = from_hf(hf, TINY_VIT_80)
    assert all(torch.equal(back[k], w[k]) for k in w)
    assert hf["visual_projection.weight"].shape == (TINY_VIT_80.proj_dim, TINY_VIT_80.n_state)   # HF [out, in]
    assert len(hf_name_map(SDXL_VIT_H)) == 8 + 32 * 16
    hf["vision_model.encoder.layers.0.self_attn.qkv.weight"] = torch.zeros(1)
    with pytest.raises(SdxlError, match="qkv"):
        from_hf(hf, TINY_VIT_80)
    vit_h = {"hidden_size": 1280, "num_attention_heads": 16, "num_hidden_layers": 32, "intermediate_size": 5120, "projection_dim": 1024,
             "image_size": 224, "patch_size": 14, "hidden_act": "gelu"}
    assert config_from_hf(vit_h) == SDXL_VIT_H
    assert config_from_hf({"vision_config": {**vit_h, "hidden_size": 1664, "num_hidden_layers": 48, "intermediate_size": 8192,
                                             "projection_dim": 1280}}) == SDXL_VIT_BIGG
    assert SDXL_VIT_H.n_tokens == 257 and SDXL_VIT_H.n_state // SDXL_VIT_H.n_head == 80 and SDXL_VIT_BIGG.n_state // SDXL_VIT_BIGG.n_head == 104


def test_clip_preprocess_against_clip_image_processor():
    """Bound: torch's antialiased bicubic and PIL's bicubic filter differ by a few u8 levels on sharp edges; on a smooth image
    the normalised pixels agree within 0.05 (about 3 u8 levels / std) and on average within 0.01."""
    transformers = pytest.importorskip("transformers")
    from sdxl_b200.clip_vision import clip_preprocess
    yy, xx = torch.meshgrid(torch.linspace(0, 1, 300), torch.linspace(0, 1, 400), indexing="ij")
    img = torch.stack([128 + 100 * torch.sin(6 * xx), 128 + 100 * torch.cos(5 * yy), 255 * xx * yy], -1).round().clamp(0, 255).to(torch.uint8)
    proc = transformers.CLIPImageProcessor()
    want = torch.from_numpy(np.asarray(proc(images=img.numpy(), return_tensors="np")["pixel_values"]))
    got = clip_preprocess(img)
    assert got.shape == want.shape == (1, 3, 224, 224)
    d = (got - want).abs()
    assert float(d.max()) < 0.05 and float(d.mean()) < 0.01
