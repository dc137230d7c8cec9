"""CPU tests (no GPU): pin the oracle.

The reference ships no numeric vectors for the UNet/sampler path (parity unpinned, see the oracle header), so
each oracle primitive is checked against an INDEPENDENT implementation of the same published op in PyTorch —
including F.scaled_dot_product_attention, which is the libtorch call the reference's own backend issues
(src/backend.rs:66-74) — and the block program against the parameter / FLOP totals SURVEY.md derives from the
reference source. Committed goldens must be reproduced bit-for-bit by the oracle on this machine.
"""
import math
import os

import numpy as np
import torch
import torch.nn.functional as F

from oracle import philox
from oracle import unet_oracle as O
from sdxl_b200.config import SDXL_BASE, SDXL_REFINER, TINY
from sdxl_b200.weights import alphas_cumprod, n_params, synth_weights, unet_tensor_specs
from harness import arb

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def test_group_norm_vs_torch():
    x = torch.randn(2, 64, 5, 7)
    g, b = torch.randn(64), torch.randn(64)
    assert torch.allclose(O.group_norm(x, g, b), F.group_norm(x, 32, g, b, eps=1e-5), atol=2e-5)


def test_layer_norm_vs_torch():
    x = torch.randn(9, 128)
    g, b = torch.randn(128), torch.randn(128)
    assert torch.allclose(O.layer_norm(x, g, b), F.layer_norm(x, (128,), g, b, eps=1e-5), atol=2e-5)


def test_attention_vs_libtorch_sdpa():
    # the reference's libtorch backend: SDPA(q,k,v, zeros mask, dropout 0, not causal)  (src/backend.rs:32-79)
    B, T, S, nh = 2, 33, 77, 3
    q, k, v = torch.randn(B, T, nh * 64), torch.randn(B, S, nh * 64), torch.randn(B, S, nh * 64)
    sp = lambda t: t.reshape(B, -1, nh, 64).transpose(1, 2)  # noqa: E731
    ref = F.scaled_dot_product_attention(sp(q), sp(k), sp(v), attn_mask=torch.zeros(T, S), dropout_p=0.0, is_causal=False)
    ref = ref.transpose(1, 2).flatten(2, 3)
    assert torch.allclose(O.qkv_attention(q, k, v, None, nh), ref, atol=2e-5)


def test_gelu_silu_vs_torch():
    x = torch.linspace(-6, 6, 101)
    assert torch.allclose(O.gelu_erf(x), F.gelu(x), atol=1e-6)
    assert torch.allclose(O.silu(x), F.silu(x), atol=1e-6)


def test_upsample_is_nearest():
    w = {"u/conv/weight": torch.zeros(3, 3, 3, 3), "u/conv/bias": torch.zeros(3)}
    for c in range(3):
        w["u/conv/weight"][c, c, 1, 1] = 1.0  # identity conv
    x = torch.randn(1, 3, 4, 5)
    assert torch.equal(O.upsample(x, w, "u"), F.interpolate(x, scale_factor=2, mode="nearest"))


def test_timestep_embedding_layout():
    e = O.timestep_embedding(torch.tensor([3]), 8)
    f = torch.exp(-math.log(10000) * torch.arange(4) / 4)
    assert torch.allclose(e[0, :4], torch.cos(3 * f)) and torch.allclose(e[0, 4:], torch.sin(3 * f))  # cos first
    ce = O.conditioning_embedding(torch.zeros(1, 1280), 256, torch.tensor([[1024, 1024]]), torch.tensor([[0, 0]]),
                                  torch.tensor([[1024, 1024]]))
    assert ce.shape == (1, 2816)  # SURVEY appendix A: 1280 + 6*256


def test_block_program_matches_survey_totals():
    for cfg, params, fl1024, fl256 in ((SDXL_BASE, 2.5675e9, 6.7612e12, 0.4278e12), (SDXL_REFINER, 2.2595e9, 7.2860e12, None)):
        shapes = {s[0]: s[1] for s in unet_tensor_specs(cfg)}
        assert abs(n_params(cfg) / params - 1) < 1e-4
        assert abs(O.unet_flops(cfg, shapes, 128, 128) / fl1024 - 1) < 1e-4
        if fl256:
            assert abs(O.unet_flops(cfg, shapes, 32, 32) / fl256 - 1) < 1e-4
    ins, mid, outs = O.unet_blocks(SDXL_BASE)
    assert [k for k, *_ in ins] == ["conv", "resnet", "resnet", "downsample", "resnet_transformer", "resnet_transformer",
                                    "downsample", "resnet_transformer", "resnet_transformer"]
    assert [k for k, *_ in outs] == ["resnet_transformer"] * 2 + ["resnet_transformer_upsample"] + ["resnet_transformer"] * 2 + \
        ["resnet_transformer_upsample"] + ["resnet"] * 3
    assert sum(d for _, _, _, d in ins + outs) + mid[3] == 70  # 70 TransformerBlocks (SURVEY 3.2)


def test_iteration_counts():
    assert [O.n_iterations(n) for n in (30, 50, 100, 4)] == [31, 50, 100, 4]
    assert O.n_iterations(30, 800) == 7 and O.n_iterations(50, 800) == 10


def test_ddim_update_algebra():
    """One DDIM step with eps == true noise recovers x0 exactly at a_prev = 1 (last step), and CFG with s=1 is the
    conditional branch: checks the restated update order (mod.rs:423-428, 539-540) on a model-free case."""
    a = 0.37
    x0, eps = torch.randn(4, 4), torch.randn(4, 4)
    x = x0 * math.sqrt(a) + eps * math.sqrt(1 - a)
    predx0 = (x - eps * math.sqrt(1 - a)) / math.sqrt(a)
    assert torch.allclose(predx0 * math.sqrt(1.0) + eps * math.sqrt(0.0), x0, atol=1e-5)
    u, c = torch.randn(5), torch.randn(5)
    assert torch.allclose(u + (c - u) * 1.0, c, atol=1e-6)


def test_alphas_schedule():
    a = alphas_cumprod().double()
    assert a.shape == (1000,) and a[0] > 0.999 and 0.004 < a[-1] < 0.006 and (a[1:] <= a[:-1]).all()


def test_goldens_reproduce():
    w = O.to_f32(synth_weights(TINY, seed=0))
    g = np.load(os.path.join(GOLD, "tiny_unet_forward.npz"))
    out = O.unet_forward(TINY, w, torch.from_numpy(g["x"]), torch.tensor([int(g["t"])]), torch.from_numpy(g["context"]),
                         torch.from_numpy(g["y"]))
    assert np.allclose(out.numpy(), g["out"], atol=1e-5)
    p = np.load(os.path.join(GOLD, "primitives.npz"))
    assert np.allclose(O.gelu_erf(arb(16)).numpy(), p["gelu"], atol=1e-7)
    q, k, v = arb(1, 6, 128), arb(1, 3, 128).cos(), arb(1, 3, 128) * 0.5
    assert np.allclose(O.qkv_attention(q, k, v, None, 2).numpy(), p["attn"], atol=1e-6)


def test_sampler_tiny_runs_and_inpaint_mask_semantics():
    w = O.to_f32(synth_weights(TINY, seed=0))
    c = O.OracleConditioning(context_full=arb(1, 2, 24), unconditional_context_full=arb(2, 24).cos(), channel_context=arb(1, 8),
                             unconditional_channel_context=arb(8).cos(), resolution=(32, 32))
    noise = torch.randn(1, 4, 4, 4, generator=torch.Generator().manual_seed(0))
    out = O.sample_latent(TINY, w, alphas_cumprod(), noise, c, 7.5, 4)
    assert out.shape == (1, 4, 4, 4) and torch.isfinite(out).all()
    # mask all-true => reference never enters: identical to plain sampling (mask_where keeps latent where true)
    mask = torch.ones(1, 4, 4, 4, dtype=torch.bool)
    out2 = O.sample_latent_with_inpainting(TINY, w, alphas_cumprod(), noise, c, 7.5, 4, torch.randn(1, 4, 4, 4), mask,
                                           [torch.randn(1, 4, 4, 4) for _ in range(4)])
    assert torch.allclose(out, out2)


def test_philox_known_answers():
    # Random123 kat_vectors for philox4x32-10
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, out in kat:
        r = philox.philox4x32_10(np.array([ctr], dtype=np.uint32), np.array(key, dtype=np.uint32))
        assert tuple(int(x) for x in r[0]) == out
    z = philox.randn(200000, 7, 1)
    assert abs(z.mean()) < 0.01 and abs(z.std() - 1) < 0.01
