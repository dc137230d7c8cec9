"""CPU tests of IP-Adapter Plus support: the h94 Resampler key map (flat and nested files, transposes, inferred depth / heads /
tokens), its rejections by key, the oracle's perceiver attention against scaled_dot_product_attention, the Plus shape checks made
before any library call, and a C program against the header's Plus entry points."""
import ctypes as C
import os
import shutil
import subprocess
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from sdxl_b200 import TINY, SdxlError
from sdxl_b200 import _lib
from sdxl_b200.ip_adapter import (SDXL_PLUS, ResamplerConfig, from_h94, ip_index_map, ip_tensor_specs, resampler_of, set_image_prompt,
                                  synth_ip_adapter)
import ip_adapter_plus_oracle as PO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = ResamplerConfig(depth=2, heads=2, tokens=16)
D = 40


def h94_plus_state_dict(cfg, D, r, nested=False, seed=0):
    """A synthetic h94-layout IP-Adapter Plus (Resampler with [out, in] Linears, latents [1, Q, W]) for `cfg`."""
    g = torch.Generator().manual_seed(seed)
    W, ctx = r.width, cfg.context_dim
    rnd = lambda *s: torch.randn(*s, generator=g).half()  # noqa: E731
    proj = {"latents": rnd(1, r.tokens, W), "proj_in.weight": rnd(W, D), "proj_in.bias": rnd(W), "proj_out.weight": rnd(ctx, W),
            "proj_out.bias": rnd(ctx), "norm_out.weight": rnd(ctx), "norm_out.bias": rnd(ctx)}
    for i in range(r.depth):
        for n in ("norm1", "norm2"):
            proj[f"layers.{i}.0.{n}.weight"], proj[f"layers.{i}.0.{n}.bias"] = rnd(W), rnd(W)
        proj[f"layers.{i}.0.to_q.weight"], proj[f"layers.{i}.0.to_kv.weight"], proj[f"layers.{i}.0.to_out.weight"] = rnd(W, W), rnd(2 * W, W), rnd(W, W)
        proj[f"layers.{i}.1.0.weight"], proj[f"layers.{i}.1.0.bias"] = rnd(W), rnd(W)
        proj[f"layers.{i}.1.1.weight"], proj[f"layers.{i}.1.3.weight"] = rnd(4 * W, W), rnd(W, 4 * W)
    specs = dict(ip_tensor_specs(cfg, D, resampler=r))
    ip = {}
    for i, path in ip_index_map(cfg).items():
        c = specs[f"{path}/attn2/ip_key/weight"][1]
        ip[f"{i}.to_k_ip.weight"] = rnd(c, ctx)
        ip[f"{i}.to_v_ip.weight"] = rnd(c, ctx)
    if nested:
        return {"image_proj": proj, "ip_adapter": ip}
    return {**{f"image_proj.{k}": v for k, v in proj.items()}, **{f"ip_adapter.{k}": v for k, v in ip.items()}}


@pytest.mark.parametrize("nested", [False, True])
def test_from_h94_plus_names_transposes_and_dims(nested):
    sd = h94_plus_state_dict(TINY, D, R, nested)
    dim, w = from_h94(sd, TINY)
    assert dim == D and resampler_of(w) == R
    specs = ip_tensor_specs(TINY, D, resampler=R)
    assert sorted(w) == sorted(n for n, _ in specs)
    for n, shape in specs:
        assert tuple(w[n].shape) == shape and w[n].dtype == torch.float16, n
    flat = h94_plus_state_dict(TINY, D, R)
    assert torch.equal(w["image_proj/latents"], flat["image_proj.latents"][0])
    assert torch.equal(w["image_proj/proj_in/weight"], flat["image_proj.proj_in.weight"].t())
    assert torch.equal(w["image_proj/layers/1/attn/to_kv/weight"], flat["image_proj.layers.1.0.to_kv.weight"].t())
    assert torch.equal(w["image_proj/layers/0/ff/fc1/weight"], flat["image_proj.layers.0.1.1.weight"].t())
    assert torch.equal(w["image_proj/layers/0/ff/fc2/weight"], flat["image_proj.layers.0.1.3.weight"].t())
    assert torch.equal(w["image_proj/layers/1/ff/norm/bias"], flat["image_proj.layers.1.1.0.bias"])
    assert torch.equal(w["image_proj/norm_out/weight"], flat["image_proj.norm_out.weight"])
    i, path = next(iter(ip_index_map(TINY).items()))
    assert torch.equal(w[f"{path}/attn2/ip_key/weight"], flat[f"ip_adapter.{i}.to_k_ip.weight"].t())


def test_sdxl_plus_shapes():
    from sdxl_b200 import SDXL_BASE
    specs = dict(ip_tensor_specs(SDXL_BASE, 1280, resampler=SDXL_PLUS))
    assert specs["image_proj/latents"] == (16, 1280) and specs["image_proj/proj_in/weight"] == (1280, 1280)
    assert specs["image_proj/layers/3/attn/to_kv/weight"] == (1280, 2560) and specs["image_proj/layers/3/ff/fc1/weight"] == (1280, 5120)
    assert specs["image_proj/proj_out/weight"] == (1280, 2048) and "image_proj/layers/4/attn/to_q/weight" not in specs
    assert resampler_of(synth_ip_adapter(TINY, D, seed=0, resampler=R)) == R
    assert resampler_of(synth_ip_adapter(TINY, D, seed=0)) is None


@pytest.mark.parametrize("key", ["image_proj.pos_emb.weight", "image_proj.to_latents_from_mean_pooled_seq.1.weight"])
def test_unsupported_resampler_options_rejected_by_key(key):
    sd = h94_plus_state_dict(TINY, D, R)
    sd[key] = torch.zeros(4, 4)
    with pytest.raises(SdxlError, match="not supported") as e:
        from_h94(sd, TINY)
    assert key in str(e.value)


@pytest.mark.parametrize("key", ["image_proj.layers.1.0.norm2.bias", "image_proj.layers.0.1.3.weight", "image_proj.proj_in.bias",
                                 "image_proj.norm_out.weight", "ip_adapter.3.to_v_ip.weight"])
def test_missing_tensor_rejected_by_key(key):
    sd = h94_plus_state_dict(TINY, D, R)
    del sd[key]
    with pytest.raises(SdxlError, match="missing") as e:
        from_h94(sd, TINY)
    assert key in str(e.value)


def test_wrong_widths_and_foreign_keys_rejected_by_key():
    sd = h94_plus_state_dict(TINY, D, R)
    sd["image_proj.proj_out.weight"] = torch.zeros(TINY.context_dim + 8, R.width).half()
    with pytest.raises(SdxlError, match="context_dim") as e:
        from_h94(sd, TINY)
    assert "image_proj.proj_out.weight" in str(e.value)
    sd = h94_plus_state_dict(TINY, D, R)
    sd["image_proj.layers.1.1.1.weight"] = torch.zeros(3 * R.width, R.width).half()   # ff_mult 3
    with pytest.raises(SdxlError, match="image_proj.layers.1.1.1.weight"):
        from_h94(sd, TINY)
    sd = h94_plus_state_dict(TINY, D, R)
    sd["image_proj.layers.0.0.to_q.weight"] = torch.zeros(64, R.width).half()          # attention width != latent width
    with pytest.raises(SdxlError, match="image_proj.layers.0.0.to_q.weight"):
        from_h94(sd, TINY)
    sd = h94_plus_state_dict(TINY, D, R)
    sd["image_proj.layers.0.2.weight"] = torch.zeros(4)
    with pytest.raises(SdxlError, match="image_proj.layers.0.2.weight"):
        from_h94(sd, TINY)
    sd = h94_plus_state_dict(TINY, D, R)
    sd["image_proj.perceiver_resampler.latents"] = torch.zeros(4)                       # FaceID Plus
    with pytest.raises(SdxlError, match="FaceID"):
        from_h94(sd, TINY)


def test_oracle_perceiver_attention_is_sdpa_over_concatenation():
    g = torch.Generator().manual_seed(0)
    wa = {k: v.float() for k, v in synth_ip_adapter(TINY, D, seed=2, resampler=R).items()}
    p = "image_proj/layers/0/attn"
    x, lat = torch.randn(19, R.width, generator=g), torch.randn(R.tokens, R.width, generator=g)
    ln = lambda t, n: F.layer_norm(t, (R.width,), wa[f"{p}/{n}/weight"], wa[f"{p}/{n}/bias"], 1e-5)  # noqa: E731
    kv = torch.cat([ln(x, "norm1"), ln(lat, "norm2")]) @ wa[f"{p}/to_kv/weight"]
    heads = lambda t: t.reshape(-1, R.heads, 64).transpose(0, 1)  # noqa: E731
    q = ln(lat, "norm2") @ wa[f"{p}/to_q/weight"]
    o = F.scaled_dot_product_attention(heads(q), heads(kv[:, :R.width]), heads(kv[:, R.width:])).transpose(0, 1).reshape(R.tokens, -1)
    want = o @ wa[f"{p}/to_out/weight"]
    got = PO.perceiver_attention(x, lat, wa, p, R.heads)
    assert float((got - want).norm() / want.norm()) < 1e-5
    tok = PO.plus_prompt_tokens(wa, torch.randn(2, 3, 19, D, generator=g))
    assert tok.shape == (2, 3 * R.tokens, TINY.context_dim)


class _NoLibrary:
    """Stands in for the library: any call fails the test."""
    def __getattr__(self, name):
        raise AssertionError(f"library call {name} made")


@pytest.mark.parametrize("embeds,negative", [(torch.zeros(2, 1, 19, D), None),                       # Plus needs a negative
                                             (torch.zeros(2, 1, 19, D + 8), torch.zeros(2, 1, 19, D + 8)),
                                             (torch.zeros(2, D), torch.zeros(2, D)),              # base-shaped embeddings
                                             (torch.zeros(2, 1, 19, D), torch.zeros(2, 1, 18, D)),
                                             (torch.zeros(2, 0, 19, D), torch.zeros(2, 0, 19, D))])
def test_plus_prompt_checked_before_any_library_call(embeds, negative):
    """The engine reads n_batch * n_images * seq_len * D floats from each pointer."""
    from sdxl_b200.ip_adapter import IPAdapter
    ad = IPAdapter.__new__(IPAdapter)
    ad.ctx = SimpleNamespace(lib=_NoLibrary(), device=torch.device("cpu"))
    ad.cfg, ad.image_embed_dim, ad.h, ad.attached, ad.resampler = TINY, D, C.c_void_p(1), 0, R
    diffuser = SimpleNamespace(ctx=ad.ctx, h=C.c_void_p(2), cfg=TINY)
    with pytest.raises(SdxlError):
        set_image_prompt(diffuser, ad, embeds, 1.0, negative=negative)
    assert ad.attached == 0


def test_ip_adapter_plus_abi_check_compiles_and_runs(tmp_path):
    gcc = shutil.which("gcc") or shutil.which("cc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib_dir = os.path.join(ROOT, "stable-diffusion-xl-burn_b200", "sdxl_b200")
    exe = str(tmp_path / "ip_adapter_plus_abi_check")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "c_abi", "ip_adapter_plus_abi_check.c"), "-L", lib_dir, "-lsdxl_b200",
                        "-Wl,-rpath," + lib_dir, "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout.startswith("ip_adapter_plus_abi_check ok"), (r.returncode, r.stdout, r.stderr)
    s_prompt, s_cfg = (int(v) for v in r.stdout.split()[-2:])
    assert s_prompt == C.sizeof(_lib.ImagePrompt) and s_cfg == C.sizeof(_lib.IpAdapterCfg)
