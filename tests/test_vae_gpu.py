"""GPU parity of the latent decoder (LatentDecoder::{decode_latent, latent_to_image}) against the CPU f32 oracle,
through the C ABI (sdxl_b200.LatentDecoder -> libsdxl_b200.so).

Tolerance statement. The reference runs the autoencoder in f32. The engine keeps the residual stream, GroupNorm
statistics, the attention scores and the softmax in f32 but rounds every tensor-core operand (normalised activations,
weights, attention probabilities) to f16, as on the UNet path; weights are the same f16-stored values in both. The
difference is operand rounding (2^-11 relative per GEMM input), measured as relative L2 error ||a-b|| / ||b||:
  * decode_latent:        <= 2e-3
  * latent_to_image (u8): |a-b| <= 1 everywhere, equal on >= 95 % of the bytes (an f32 error of ~1e-3 * 127.5 moves
    a value across a truncation boundary with that probability; measured 97.6 %)
"""
import os

import numpy as np
import pytest
import torch

from sdxl_b200 import SDXL_VAE, TINY_VAE, LatentDecoder, synth_weights
from oracle import unet_oracle as O
from oracle import vae_oracle as VO
from harness import rel_err

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 2e-3


@pytest.fixture(scope="module")
def tiny(ctx):
    w = synth_weights(TINY_VAE, seed=0)
    d = LatentDecoder(ctx, TINY_VAE, w)
    yield d, O.to_f32(w)
    d.close()


def test_golden_fixture(tiny):
    d, _ = tiny
    g = np.load(os.path.join(GOLD, "tiny_vae_decode.npz"))
    lat = torch.from_numpy(g["latent"])
    img = d.decode_latent(lat)                       # host in -> host out
    assert not img.is_cuda
    e = rel_err(img, torch.from_numpy(g["image"]))
    print("golden decode rel err", e)
    assert e <= TOL
    u8 = d.latent_to_image(lat.cuda()).cpu().numpy().astype(np.int32)   # device in -> device out
    diff = np.abs(u8 - g["u8"].astype(np.int32))
    assert diff.max() <= 1 and (diff == 0).mean() >= 0.95


@pytest.mark.parametrize("B,h,w", [(1, 8, 8), (2, 8, 16), (3, 16, 16), (1, 24, 8)])
def test_decode_vs_oracle(tiny, B, h, w):
    d, wf = tiny
    lat = torch.randn(B, 4, h, w, generator=torch.Generator().manual_seed(10 * B + h)) * TINY_VAE.scale_factor * 1.5
    got = d.decode_latent(lat.cuda())
    want = VO.decode_latent(TINY_VAE, wf, lat)
    e = rel_err(got, want)
    print(f"tiny decode B={B} {h}x{w}: rel err {e:.2e}")
    assert got.shape == (B, 3, 4 * h, 4 * w) and e <= TOL
    assert abs(d.plan_flops / VO.decoder_flops(TINY_VAE, h, w, B) - 1) < 1e-9


def test_bad_shape_is_an_error(tiny):
    d, _ = tiny
    with pytest.raises(Exception, match="multiple of 64"):
        d.decode_latent(torch.zeros(1, 4, 4, 4))


def test_batch_invariance_and_determinism(tiny):
    d, _ = tiny
    lat = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(5)).cuda() * 0.2
    a = d.decode_latent(lat)
    b = d.decode_latent(torch.cat([lat, lat * 0.5, lat]))
    assert torch.equal(a[0], b[0]) and torch.equal(b[0], b[2])
    assert torch.equal(a, d.decode_latent(lat))


@pytest.fixture(scope="module")
def full(ctx):
    w = synth_weights(SDXL_VAE, seed=7)
    d = LatentDecoder(ctx, SDXL_VAE, w)
    yield d, w
    d.close()


def test_sdxl_vae_256_vs_oracle(full):
    """Real widths (512/512/256/128) at a 256^2 image (latent 32^2, T=1024): the oracle finishes in seconds."""
    d, w = full
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    lat = torch.randn(1, 4, 32, 32, generator=torch.Generator().manual_seed(0)) * SDXL_VAE.scale_factor
    got = d.decode_latent(lat.cuda())
    want = VO.decode_latent(SDXL_VAE, O.to_f32(w), lat)
    e = rel_err(got, want)
    print("SDXL VAE 256^2 decode rel err", e)
    assert e <= TOL
    u8 = d.latent_to_image(lat.cuda()).cpu().numpy().astype(np.int32)
    ref = VO.latent_to_image(SDXL_VAE, O.to_f32(w), lat).numpy().astype(np.int32)
    diff = np.abs(u8 - ref)
    assert diff.max() <= 1 and (diff == 0).mean() >= 0.95


def test_sdxl_vae_1024_properties(full):
    """Full size (latent 128^2, T=16384, 1.07 GB score matrix): size-independent properties — determinism, finiteness,
    the FLOP total of SURVEY.md §8(f), u8 conversion consistent with the f32 image, batch invariance."""
    d, _ = full
    lat = torch.randn(1, 4, 128, 128, generator=torch.Generator().manual_seed(1)).cuda() * SDXL_VAE.scale_factor
    a = d.decode_latent(lat)
    assert a.shape == (1, 3, 1024, 1024) and torch.isfinite(a).all()
    assert abs(d.plan_flops / 10.470392594432e12 - 1) < 1e-9
    assert torch.equal(a, d.decode_latent(lat))
    u8 = d.latent_to_image(lat)
    ref = (((a.permute(0, 2, 3, 1) + 1.0) / 2.0) * 255.0).clamp(0, 255).to(torch.uint8)
    assert torch.equal(u8, ref)
    b = d.decode_latent(torch.cat([lat, lat]))
    assert torch.equal(b[0], a[0]) and torch.equal(b[1], a[0])


def test_sdxl_vae_1024_vs_golden(full):
    """Full size against the CPU f32 oracle (committed digests, tests/golden/make_fullsize_golden.py --only vae): the decoded 1024^2
    image through its 8x8 block means (every pixel contributes) and one raw pixel per block; the encoded latent in full."""
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import fullsize_cases as FC
    d, _ = full
    g = np.load(os.path.join(GOLD, "vae_1024.npz"))
    lat, rgb = FC.vae_1024_inputs(SDXL_VAE.scale_factor)
    img = d.decode_latent(lat.cuda()).cpu()
    pool, samp = FC.vae_image_digest(img)
    e_pool, e_samp = rel_err(pool, torch.from_numpy(g["pool"])), rel_err(samp, torch.from_numpy(g["samp"]))
    e_norm = abs(float(img.double().norm()) / float(g["norm"]) - 1.0)
    print(f"SDXL VAE 1024^2 decode vs oracle: block means rel err {e_pool:.2e}, raw samples rel err {e_samp:.2e}, |image| rel {e_norm:.1e}")
    assert e_pool <= TOL and e_samp <= TOL and e_norm <= 1e-3
    enc = d.image_to_latent(rgb.cuda()).cpu()
    e_enc = rel_err(enc, torch.from_numpy(g["latent"]))
    print(f"SDXL VAE 1024^2 image_to_latent vs oracle: rel err {e_enc:.2e}")
    assert enc.shape == (1, 4, 128, 128) and e_enc <= TOL


# ---- encoder half (LatentDecoder::{encode_image, image_to_latent}) ---------------------------------------------------
def test_encode_golden_fixture(tiny):
    d, _ = tiny
    g = np.load(os.path.join(GOLD, "tiny_vae_encode.npz"))
    lat = d.image_to_latent(torch.from_numpy(g["rgb"]))          # host u8 in -> host latent out
    e = rel_err(lat, torch.from_numpy(g["latent"]))
    print("golden encode rel err", e)
    assert not lat.is_cuda and e <= TOL


@pytest.mark.parametrize("B,H,W", [(1, 32, 32), (2, 64, 32), (1, 96, 64)])
def test_encode_vs_oracle(tiny, B, H, W):
    d, wf = tiny
    img = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(H + W)) * 2 - 1
    got = d.encode_image(img.cuda())
    want = VO.encode_image(TINY_VAE, wf, img)
    e = rel_err(got, want)
    print(f"tiny encode B={B} {H}x{W}: rel err {e:.2e}")
    assert got.shape == (B, 4, H // 4, W // 4) and e <= TOL
    assert abs(d.encode_plan_flops / VO.encoder_flops(TINY_VAE, H, W, B) - 1) < 1e-9
    rgb = torch.randint(0, 256, (B, H, W, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(3))
    assert rel_err(d.image_to_latent(rgb.cuda()), VO.image_to_latent(TINY_VAE, wf, rgb)) <= TOL


def test_sdxl_vae_encode_256_vs_oracle(full):
    d, w = full
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    img = torch.rand(1, 3, 256, 256, generator=torch.Generator().manual_seed(2)) * 2 - 1
    got = d.encode_image(img.cuda())
    want = VO.encode_image(SDXL_VAE, O.to_f32(w), img)
    e = rel_err(got, want)
    print("SDXL VAE 256^2 encode rel err", e)
    assert got.shape == (1, 4, 32, 32) and e <= TOL


def test_sdxl_vae_encode_1024_properties(full):
    d, _ = full
    rgb = torch.randint(0, 256, (1, 1024, 1024, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(6)).cuda()
    a = d.image_to_latent(rgb)
    assert a.shape == (1, 4, 128, 128) and torch.isfinite(a).all()
    assert abs(d.encode_plan_flops / VO.encoder_flops(SDXL_VAE, 1024, 1024) - 1) < 1e-9
    assert torch.equal(a, d.image_to_latent(rgb))                                       # deterministic
    img = (rgb.float() / 255.0).permute(0, 3, 1, 2) * 2.0 - 1.0
    # u8 front end == f32 entry point, up to torch's own CUDA `x / 255` (multiplies by the reciprocal: 1 ulp off true division)
    assert rel_err(a, d.encode_image(img.contiguous())) <= TOL      # 1-ulp input changes flip f16 operand roundings: same noise floor
    # encode -> decode round trip runs and stays finite (synthetic weights: no reconstruction claim)
    assert torch.isfinite(d.decode_latent(a)).all()
