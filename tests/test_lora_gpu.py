"""GPU tests of LoRA adapters merged on the device (sdxl_unet_set_adapters / sdxl_clip_set_adapters), tiny configs.

Exactness. The adapters of the exact tests have factors in {-1, 0, 1} / 16, no alpha (alpha / r = 1) and a power-of-two scale,
so every f32 product and sum of the merge is exact and independent of its order: the device merge must then give the same
bits as `merge_into` on the host, and a model merged in place must compute exactly what a model loaded from the host-merged
weights computes. The upsample convs are the one documented exception (their 3x3 weights are stored as four phase kernels
and the delta is added after the phase sums were rounded): those are checked against the f32 oracle on host-merged weights
with the bounds of tests/test_unet_gpu.py.
"""
import pytest
import torch

import sdxl_b200
from sdxl_b200 import (TINY, TINY_CLIP, TINY_OPEN_CLIP, TINY_REFINER, TINY_VAE, ClipTextEncoder, Conditioning, Diffuser, Embedder,
                       LatentDecoder, OpenClipTokenizer, SdxlError, UNetConfig, synth_weights)
from sdxl_b200.lora import clip_lora_modules, merge_into, unet_lora_modules
from sdxl_b200.pipeline import sample
from oracle import clip_oracle as CO
from oracle import unet_oracle as O
from lora_cases import layer_paths, make_adapter, to_kohya, write_safetensors
from harness import arb, h16f, rel_err, tiny_conditioning

pytestmark = pytest.mark.gpu
FWD_TOL = 2e-3
SAMPLE_TOL = 5e-3


def exact_paths(cfg):
    """Every LoRA-able layer except the upsample convs: fused QKV slices, KV2, GEGLU, FF down, proj_in/out, attention out,
    ResBlock conv_in / conv_out, skip segment, downsample, lin_embed rows, time / label MLPs, first conv, head conv."""
    return [p for p in layer_paths(cfg) if "/upsample/" not in p]


X = arb(2, 4, 16, 16)
T = 499


class Tiny:
    def __init__(self, ctx, cfg=TINY, seed=0):
        self.ctx, self.cfg = ctx, cfg
        self.w = synth_weights(cfg, seed=seed)
        self.d = Diffuser(ctx, cfg, self.w)
        self.c = h16f(arb(2, 7, cfg.context_dim))
        self.y = h16f(arb(2, cfg.adm_in_channels))
        self.noise = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(0))

    def fwd(self, d=None, set_cond=True):
        d = d or self.d
        return d.unet_forward(X, [T], self.c, self.y) if set_cond else d.unet_forward(X, [T])

    def smp(self, d=None):
        return (d or self.d).sample_latent(Conditioning(**tiny_conditioning(cfg=self.cfg)), 7.5, 4, noise=self.noise)

    def loaded(self, weights):
        return Diffuser(self.ctx, self.cfg, weights)


@pytest.fixture(scope="module")
def tiny(ctx):
    t = Tiny(ctx)
    t.base_fwd = t.fwd()
    t.base_smp = t.smp()
    yield t
    t.d.close()


def test_zero_up_is_bit_identical(tiny):
    tiny.d.set_adapters([(make_adapter(TINY, layer_paths(TINY), rank=4, seed=1, zero_up=True), 1.0)])
    assert torch.equal(tiny.fwd(), tiny.base_fwd)
    tiny.d.set_adapters([])


def test_exact_layout_with_live_plan_graph_and_conditioning(tiny):
    t = tiny
    t.fwd()
    t.fwd()                                   # plan built, graph captured, conditioning hoisted
    n_ops = t.d.plan_num_ops
    ad = make_adapter(TINY, exact_paths(TINY), rank=4, seed=3)
    t.d.set_adapters([(ad, 0.5)])
    got = t.fwd(set_cond=False)               # the conditioning set before the merge is re-projected
    assert t.d.plan_num_ops == n_ops
    ref_model = t.loaded(merge_into(t.w, ad, 0.5))
    want = t.fwd(ref_model)
    assert not torch.equal(want, t.base_fwd)
    assert torch.equal(got, want)
    assert torch.equal(t.fwd(), want)          # and with conditioning set again
    assert torch.equal(t.smp(), t.smp(ref_model))
    ref_model.close()
    t.d.set_adapters([])
    assert torch.equal(t.fwd(), t.base_fwd)


def test_upsample_convs_vs_oracle(tiny):
    t = tiny
    ad = make_adapter(TINY, layer_paths(TINY), rank=4, seed=5)
    assert any("/upsample/" in k for k in ad)
    t.d.set_adapters([(ad, 0.5)])
    wf = O.to_f32(merge_into(t.w, ad, 0.5))
    out = t.fwd()
    ref = O.unet_forward(TINY, wf, X, torch.tensor([T]), t.c, t.y)
    e = rel_err(out, ref)
    print(f"tiny forward with every layer merged vs oracle on merged weights: rel err {e:.3e} (adapter moves it {rel_err(out, t.base_fwd):.3e})")
    assert e < FWD_TOL and rel_err(out, t.base_fwd) > 10 * FWD_TOL
    s = t.smp()
    sref = O.sample_latent(TINY, wf, sdxl_b200.alphas_cumprod(), t.noise, O.OracleConditioning(**tiny_conditioning()), 7.5, 4)
    e = rel_err(s, sref)
    print(f"tiny 4-step CFG sample with every layer merged vs oracle: rel err {e:.3e}")
    assert e < SAMPLE_TOL
    t.d.set_adapters([])


def test_restore_cycles_are_bit_exact(tiny):
    t = tiny
    ad = make_adapter(TINY, layer_paths(TINY), rank=8, seed=9, dyadic=False, alpha=4.0)
    merged = None
    for _ in range(3):
        t.d.set_adapters([(ad, 0.7)])
        m = t.fwd()
        merged = m if merged is None else merged
        assert torch.equal(m, merged)
        t.d.set_adapters([])
        assert torch.equal(t.fwd(), t.base_fwd)
        assert torch.equal(t.smp(), t.base_smp)


def test_stacking_equals_concatenated_ranks_and_rescale_equals_fresh_apply(tiny):
    t = tiny
    paths = exact_paths(TINY)
    a1 = make_adapter(TINY, paths, rank=2, seed=11)
    a2 = make_adapter(TINY, paths, rank=3, seed=12)
    cat = {}
    for p in paths:
        cat[f"{p}/lora_down"] = torch.cat([a1[f"{p}/lora_down"], a2[f"{p}/lora_down"]], 0)
        cat[f"{p}/lora_up"] = torch.cat([a1[f"{p}/lora_up"], a2[f"{p}/lora_up"]], 1)
    t.d.set_adapters([(a1, 0.5), (a2, 0.5)])
    two = t.fwd()
    t.d.set_adapters([(cat, 0.5)])
    assert torch.equal(t.fwd(), two)
    # changing a scale re-derives from the loaded weights: equal to applying it to a freshly loaded model
    g = make_adapter(TINY, layer_paths(TINY), rank=5, seed=13, dyadic=False)
    t.d.set_adapters([(g, 1.0)])
    t.d.set_adapters([(g, 0.3)])
    again = t.fwd()
    fresh = t.loaded(t.w)
    fresh.set_adapters([(g, 0.3)])
    assert torch.equal(again, t.fwd(fresh))
    fresh.close()
    # a layer touched before but not now is restored
    t.d.set_adapters([(make_adapter(TINY, paths[:40], rank=2, seed=14), 0.5)])
    t.d.set_adapters([(make_adapter(TINY, paths[40:], rank=2, seed=15), 0.5)])
    only = t.loaded(merge_into(t.w, make_adapter(TINY, paths[40:], rank=2, seed=15), 0.5))
    assert torch.equal(t.fwd(), t.fwd(only))
    only.close()
    t.d.set_adapters([])
    assert torch.equal(t.fwd(), t.base_fwd)


def test_invalid_adapter_leaves_the_model_unchanged(tiny):
    t = tiny
    p = "input_blocks/4/transformer/transformer_0/attn1/value"
    good = make_adapter(TINY, exact_paths(TINY)[:30], rank=2, seed=21)
    t.d.set_adapters([(good, 0.5)])
    before = t.fwd()
    bad = make_adapter(TINY, [p, "conv_out"], rank=2, seed=22)
    cases = []
    b1 = dict(bad); b1[f"{p}/lora_up"] = torch.zeros(129, 2, dtype=torch.float16); cases.append((b1, f"{p}/lora_up"))
    b2 = dict(bad); b2[f"{p}/lora_up"] = torch.zeros(128, 3, dtype=torch.float16); cases.append((b2, p))
    b3 = dict(bad); b3["no/such/layer/lora_down"] = torch.zeros(2, 4, dtype=torch.float16); cases.append((b3, "no/such/layer"))
    b4 = dict(bad); b4[f"{p}/lora_down"] = b4[f"{p}/lora_down"].float(); cases.append((b4, f"{p}/lora_down"))
    b5 = dict(bad); del b5["conv_out/lora_up"]; cases.append((b5, "conv_out/lora_up"))
    b6 = dict(bad); b6["conv_out/lora_down"] = torch.zeros(2, 64, 1, 1, dtype=torch.float16); cases.append((b6, "conv_out/lora_down"))
    for b, name in cases:
        with pytest.raises(SdxlError, match=name):
            t.d.set_adapters([(make_adapter(TINY, exact_paths(TINY)[:5], rank=2, seed=23), 1.0), (b, 1.0)])
        assert torch.equal(t.fwd(), before)
    with pytest.raises(SdxlError, match="at most"):
        t.d.set_adapters([(good, 0.1)] * 17)
    t.d.set_adapters([])
    assert torch.equal(t.fwd(), t.base_fwd)


def test_refiner(ctx):
    t = Tiny(ctx, TINY_REFINER, seed=1)
    base = t.fwd()
    ad = make_adapter(TINY_REFINER, exact_paths(TINY_REFINER), rank=4, seed=31)
    t.d.set_adapters([(ad, 0.5)])
    ref_model = t.loaded(merge_into(t.w, ad, 0.5))
    assert torch.equal(t.fwd(set_cond=False), t.fwd(ref_model))
    lat = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(2))
    c = Conditioning(context_open_clip=h16f(arb(2, 6, 40)), channel_context_refiner=h16f(arb(2, 16)), resolution=(128, 128))
    assert torch.equal(t.d.refine_latent(lat, c, 7.5, 800, 50, noise=t.noise), ref_model.refine_latent(lat, c, 7.5, 800, 50, noise=t.noise))
    t.d.set_adapters([])
    assert torch.equal(t.fwd(), base)
    ref_model.close()
    t.d.close()


def test_clip_adapters(ctx):
    w = synth_weights(TINY_OPEN_CLIP, seed=2)
    e = ClipTextEncoder(ctx, TINY_OPEN_CLIP, w)
    g = torch.Generator().manual_seed(4)
    tok = torch.randint(1, 49405, (2, 77), generator=g, dtype=torch.int32)
    tok[:, 0] = 49406
    tok[0, 9] = tok[1, 20] = 49407
    idx = TINY_OPEN_CLIP.n_layer - 1
    h0, p0 = e.forward_hidden_pooled(tok, idx)
    ad = make_adapter(TINY_OPEN_CLIP, layer_paths(TINY_OPEN_CLIP, clip=True), rank=4, seed=41, clip=True)
    e.set_adapters([(ad, 0.5)])
    h, p = e.forward_hidden_pooled(tok, idx)
    wm = merge_into(w, ad, 0.5)
    hw, pw = CO.forward_hidden_pooled(TINY_OPEN_CLIP, O.to_f32(wm), tok, idx)
    print(f"tiny CLIP with adapters vs oracle: hidden {rel_err(h, hw):.2e} pooled {rel_err(p, pw):.2e}")
    assert rel_err(h, hw) <= FWD_TOL and rel_err(p, pw) <= FWD_TOL and rel_err(h, h0) > 10 * FWD_TOL
    em = ClipTextEncoder(ctx, TINY_OPEN_CLIP, wm)
    hm, pm = em.forward_hidden_pooled(tok, idx)
    assert torch.equal(h, hm) and torch.equal(p, pm)
    e.set_adapters([])
    h1, p1 = e.forward_hidden_pooled(tok, idx)
    assert torch.equal(h1, h0) and torch.equal(p1, p0)
    em.close()
    e.close()


def test_pipeline_sample_with_kohya_file(ctx, tmp_path):
    import os
    mini = os.path.join(os.path.dirname(__file__), "golden", "mini_bpe")
    ca, cb = TINY_CLIP, TINY_OPEN_CLIP
    ucfg = UNetConfig(adm_in_channels=cb.embed_dim + 6 * 256, model_channels=64, channel_mults=(1, 2, 4), transformer_depths=(0, 1, 1),
                      context_dim=ca.n_state + cb.n_state)
    wa, wb, wu, wv = (synth_weights(c, seed=s) for c, s in ((ca, 1), (cb, 2), (ucfg, 3), (TINY_VAE, 0)))
    tok = OpenClipTokenizer(os.path.join(mini, "mini_merges.txt"), os.path.join(mini, "mini_vocab.txt"))
    vae = LatentDecoder(ctx, TINY_VAE, wv)

    def models(a, b, u):
        return Embedder(ctx, ClipTextEncoder(ctx, ca, a), ClipTextEncoder(ctx, cb, b), tok, tok), Diffuser(ctx, ucfg, u)

    au = make_adapter(ucfg, exact_paths(ucfg), rank=4, seed=51)
    a1 = make_adapter(ca, layer_paths(ca, clip=True), rank=2, seed=52, clip=True)
    a2 = make_adapter(cb, layer_paths(cb, clip=True), rank=2, seed=53, clip=True)
    k = to_kohya(au, unet_lora_modules(ucfg))
    k.update(to_kohya(a1, clip_lora_modules(ca, "lora_te1")))
    k.update(to_kohya(a2, clip_lora_modules(cb, "lora_te2")))
    path = str(tmp_path / "style.safetensors")
    write_safetensors(path, k)

    emb, dif = models(wa, wb, wu)
    kw = dict(guidance=5.0, n_steps=4, resolution=(64, 64), seed=0)
    base = sample(emb, dif, vae, "a photo of a cat", **kw)
    got = sample(emb, dif, vae, "a photo of a cat", loras=[(path, 0.5)], **kw)
    emb_m, dif_m = models(merge_into(wa, a1, 0.5), merge_into(wb, a2, 0.5), merge_into(wu, au, 0.5))
    want = sample(emb_m, dif_m, vae, "a photo of a cat", **kw)
    assert torch.equal(got, want) and not torch.equal(got, base)
    assert torch.equal(sample(emb, dif, vae, "a photo of a cat", **kw), base)   # the adapters are gone after the call
