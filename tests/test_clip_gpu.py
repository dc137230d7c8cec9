"""GPU parity of the text encoders and the Embedder glue (CLIP::forward_hidden / forward_hidden_pooled,
Embedder::text_to_conditioning) against the CPU f32 oracle, through the C ABI.

Tolerance statement. The reference runs the Embedder in f32. The engine keeps the residual stream, LayerNorm, softmax and
the pooled projection input in f32 and rounds GEMM operands to f16 (weights are the same f16-stored values on both sides):
relative L2 error <= 2e-3 on hidden states and pooled features (measured values are printed).
"""
import os

import numpy as np
import pytest
import torch

from sdxl_b200 import (TINY, TINY_CLIP, TINY_OPEN_CLIP, SDXL_CLIP_L, SDXL_OPEN_CLIP_G, ClipTextEncoder, Diffuser, Embedder,
                       OpenClipTokenizer, synth_weights)
from oracle import clip_oracle as CO
from oracle import tokenizer_oracle as TO
from oracle import unet_oracle as O
from harness import rel_err

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
MINI = os.path.join(GOLD, "mini_bpe")
TOL = 2e-3


@pytest.fixture(scope="module")
def enc(ctx):
    w1, w2 = synth_weights(TINY_CLIP, seed=1), synth_weights(TINY_OPEN_CLIP, seed=2)
    e1, e2 = ClipTextEncoder(ctx, TINY_CLIP, w1), ClipTextEncoder(ctx, TINY_OPEN_CLIP, w2)
    yield e1, e2, O.to_f32(w1), O.to_f32(w2)
    e1.close()
    e2.close()


def test_golden_fixture(enc):
    e1, e2, _, _ = enc
    g = np.load(os.path.join(GOLD, "tiny_clip.npz"))
    h1 = e1.forward_hidden(g["tokens_clip"], TINY_CLIP.n_layer - 1)
    h2, p2 = e2.forward_hidden_pooled(g["tokens_open_clip"], TINY_OPEN_CLIP.n_layer - 1)
    errs = rel_err(h1, torch.from_numpy(g["hidden_clip"])), rel_err(h2, torch.from_numpy(g["hidden_open_clip"])), \
        rel_err(p2, torch.from_numpy(g["pooled_open_clip"]))
    print("tiny clip golden rel errs", errs)
    assert max(errs) <= TOL


@pytest.mark.parametrize("B,hidden_idx", [(1, 0), (1, 3), (3, 2), (2, 4)])
def test_forward_hidden_vs_oracle(enc, B, hidden_idx):
    _, e2, _, w2 = enc
    g = torch.Generator().manual_seed(B * 10 + hidden_idx)
    tok = torch.randint(1, 49405, (B, 77), generator=g, dtype=torch.int32)
    tok[:, 0] = 49406
    for b in range(B):
        tok[b, 5 + 9 * b] = 49407
        tok[b, 6 + 9 * b:] = 0
    got = e2.forward_hidden(tok, hidden_idx)
    want = CO.forward_hidden(TINY_OPEN_CLIP, w2, tok, hidden_idx)
    e = rel_err(got, want)
    print(f"forward_hidden B={B} idx={hidden_idx}: rel err {e:.2e}")
    assert e <= TOL
    if hidden_idx < TINY_OPEN_CLIP.n_layer:
        h, p = e2.forward_hidden_pooled(tok, hidden_idx)
        hw, pw = CO.forward_hidden_pooled(TINY_OPEN_CLIP, w2, tok, hidden_idx)
        assert rel_err(h, hw) <= TOL and rel_err(p, pw) <= TOL


def test_errors(enc):
    e1, _, _, _ = enc
    bad = torch.zeros(1, 77, dtype=torch.int32)
    bad[0, 3] = 60000
    with pytest.raises(Exception, match="token id outside"):
        e1.forward_hidden(bad, 1)
    with pytest.raises(Exception, match="out of range"):
        e1.forward_hidden(torch.zeros(1, 77, dtype=torch.int32), 99)


def test_masked_qkv_attention_op(ctx):
    """Backend::qkv_attention with the decoder mask (src/backend.rs:4-21) through the public op."""
    g = torch.Generator().manual_seed(3)
    q, k, v = (torch.randn(2, 77, 128, generator=g).half() for _ in range(3))
    mask = CO.attn_decoder_mask(77)
    got = ctx.qkv_attention(q.cuda(), k.cuda(), v.cuda(), mask.half().cuda(), 2)
    want = O.qkv_attention(q.float(), k.float(), v.float(), mask, 2)
    assert rel_err(got.float(), want) <= 1e-3


def test_embedder_text_to_conditioning(ctx, enc):
    """End to end: text -> tokenizers -> encoders -> Conditioning, then one UNet forward consumes it."""
    e1, e2, w1, w2 = enc
    tok = OpenClipTokenizer(os.path.join(MINI, "mini_merges.txt"), os.path.join(MINI, "mini_vocab.txt"))
    otok = TO.OpenClipTokenizer(os.path.join(MINI, "mini_merges.txt"), os.path.join(MINI, "mini_vocab.txt"))
    emb = Embedder(ctx, e1, e2, tok, tok)
    text = "An astronaut riding a horse on Mars, 4k"
    size, crop, ar = (1024, 1024), (0, 0), (1024, 1024)
    cond = emb.text_to_conditioning(text, size, crop, ar)
    want = CO.text_to_conditioning(TINY_CLIP, w1, TINY_OPEN_CLIP, w2, otok, otok, TO.tokenize_text, text, size, crop, ar)
    assert cond.context_full.shape == (1, 77, 128 + 192) and cond.channel_context.shape == (1, 64 + 6 * 256)
    assert cond.channel_context_refiner.shape == (1, 64 + 5 * 256) and cond.unconditional_context_full.shape == (77, 320)
    assert tuple(cond.resolution) == (1024, 1024)
    for f in cond._fields():
        e = rel_err(getattr(cond, f).float(), want[f])
        assert e <= TOL + 5e-4, (f, e)    # + f16 rounding of Conditioning::convert


def test_sdxl_text_encoders_full_size(ctx):
    """Real widths (CLIP-L 12x768, OpenCLIP-bigG 32x1280): parity with the oracle on one prompt-sized batch."""
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    tok = torch.zeros(1, 77, dtype=torch.int32)
    tok[0, :8] = torch.tensor([49406, 320, 1125, 539, 320, 2368, 269, 49407])
    for cfg, seed in ((SDXL_CLIP_L, 11), (SDXL_OPEN_CLIP_G, 12)):
        w = synth_weights(cfg, seed=seed)
        e = ClipTextEncoder(ctx, cfg, w)
        wf = O.to_f32(w)
        h, p = e.forward_hidden_pooled(tok, cfg.n_layer - 1)
        hw, pw = CO.forward_hidden_pooled(cfg, wf, tok, cfg.n_layer - 1)
        print(cfg.n_state, "hidden rel err", rel_err(h, hw), "pooled rel err", rel_err(p, pw))
        assert rel_err(h, hw) <= TOL and rel_err(p, pw) <= TOL
        e.close()
        del w, wf
