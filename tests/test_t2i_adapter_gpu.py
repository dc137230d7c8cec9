"""GPU tests of T2I-Adapter conditioning (sdxl_t2i_adapter_load, sdxl_unet_set_t2i_adapters), tiny configs, against the f32 oracle
(oracle/unet_oracle.py) with the bounds of tests/test_unet_gpu.py, plus the bit-exact identities of detach, scale 0, the timestep
window and in-place rewrites, and the refusals that leave the previous set attached."""
import pytest
import torch

import sdxl_b200
from sdxl_b200 import (TINY, TINY_CONTROLNET, TINY_T2I_ADAPTER, Conditioning, ControlNet, Diffuser, SdxlError, T2IAdapter, T2IAdapterConfig,
                       UNetConfig, synth_weights, t2i_t_min)
from sdxl_b200 import _lib
from oracle import unet_oracle as O
import t2i_adapter_oracle as TA
from harness import arb, h16f, plan_builds, rel_err, tiny_conditioning

pytestmark = pytest.mark.gpu
FWD_TOL = 2e-3
SAMPLE_TOL = 5e-3
T = 499


def hint(n, seed, c=3, size=128):
    return torch.rand(n, c, size, size, generator=torch.Generator().manual_seed(seed))


X = arb(2, 4, 16, 16)


class Setup:
    def __init__(self, ctx):
        self.ctx = ctx
        self.w = synth_weights(TINY, seed=0)
        self.wf = O.to_f32(self.w)
        self.d = Diffuser(ctx, TINY, self.w)
        self.wa = [synth_weights(TINY_T2I_ADAPTER, seed=s) for s in (1, 2)]
        self.waf = [O.to_f32(w) for w in self.wa]
        self.ads = [T2IAdapter(ctx, TINY_T2I_ADAPTER, w) for w in self.wa]
        self.c = h16f(arb(2, 7, TINY.context_dim))
        self.y = h16f(arb(2, TINY.adm_in_channels))
        self.h = [hint(2, 10), hint(1, 11)]
        self.noise = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(0))

    def fwd(self, t=T):
        return self.d.unet_forward(X, [t], self.c, self.y)

    def oracle_fwd(self, items, t=T, t_min=0, controls=()):
        feats = TA.summed_features([(TINY_T2I_ADAPTER, self.waf[i], self.h[j], s) for i, j, s in items])
        return O.unet_forward(TINY, self.wf, X, torch.tensor([t]), self.c, self.y, O.Attach(t2i=(feats, t_min), controls=controls))


@pytest.fixture(scope="module")
def S(ctx):
    s = Setup(ctx)
    s.base = s.fwd()
    s.base_ops, s.base_flops = s.d.plan_num_ops, s.d.plan_flops
    yield s
    s.d.set_t2i_adapters([])
    for a in s.ads:
        a.close()
    s.d.close()


@pytest.mark.parametrize("in_channels, n_hint", [(3, 1), (3, 2), (1, 1), (1, 2)])
def test_features_vs_oracle(ctx, in_channels, n_hint):
    acfg = T2IAdapterConfig(TINY, in_channels=in_channels)
    w = synth_weights(acfg, seed=5)
    ad = T2IAdapter(ctx, acfg, w)
    hh = hint(n_hint, 20, c=in_channels)
    got = ad.features(hh)
    ref = TA.adapter_features(acfg, O.to_f32(w), hh)
    ad.close()
    assert [g.shape for g in got] == [r.shape for r in ref]
    errs = [rel_err(g, r) for g, r in zip(got, ref)]
    print(f"in_channels {in_channels}, n_hint {n_hint}: feature rel errs {['%.2e' % e for e in errs]}")
    assert max(errs) <= FWD_TOL


def test_forward_one_adapter_vs_oracle(S):
    S.d.set_t2i_adapters([(S.ads[0], S.h[0], 1.0)])
    got = S.fwd()
    ref = S.oracle_fwd([(0, 0, 1.0)])
    S.d.set_t2i_adapters([])
    e, moved = rel_err(got, ref), rel_err(got, S.base)
    print(f"one adapter: forward rel err vs oracle {e:.2e}; the adapter moves the output by {moved:.2e}")
    assert e <= FWD_TOL and moved > 0.05


def test_forward_two_adapters_vs_oracle(S):
    S.d.set_t2i_adapters([(S.ads[0], S.h[1], 0.6), (S.ads[1], S.h[1], 1.4)])
    got = S.fwd()
    S.d.set_t2i_adapters([])
    assert rel_err(got, S.oracle_fwd([(0, 1, 0.6), (1, 1, 1.4)])) <= FWD_TOL


def test_forward_adapter_and_controlnet_vs_oracle(S, ctx):
    wc = synth_weights(TINY_CONTROLNET, seed=7)
    net = ControlNet(ctx, TINY_CONTROLNET, wc)
    S.d.set_controls([(net, S.h[1], 0.8)])
    S.d.set_t2i_adapters([(S.ads[0], S.h[0], 1.0)])
    got = S.fwd()
    S.d.set_t2i_adapters([])
    S.d.set_controls([])
    net.close()
    ref = S.oracle_fwd([(0, 0, 1.0)], controls=[(TINY_CONTROLNET, O.to_f32(wc), S.h[1], 0.8)])
    assert rel_err(got, ref) <= FWD_TOL


@pytest.mark.parametrize("factor", [1.0, 0.5])
def test_sample_cfg_vs_oracle(S, factor):
    t_min = t2i_t_min(4, factor)
    S.d.set_t2i_adapters([(S.ads[0], S.h[0], 1.0)], t_min=t_min)
    got = S.d.sample_latent(Conditioning(**tiny_conditioning()), 7.5, 4, noise=S.noise)
    S.d.set_t2i_adapters([])
    alphas = sdxl_b200.alphas_cumprod(TINY.n_steps)
    att = O.Attach(t2i=(TA.summed_features([(TINY_T2I_ADAPTER, S.waf[0], S.h[0], 1.0)]), t_min))
    ref = O.sample_latent(TINY, S.wf, alphas, S.noise, O.OracleConditioning(**tiny_conditioning()), 7.5, 4, att=att)
    assert rel_err(got, ref) <= SAMPLE_TOL


def test_detach_scale_zero_and_window_are_bit_identical(S):
    S.d.set_t2i_adapters([(S.ads[0], S.h[0], 1.0)])
    adapted = S.fwd()
    assert S.d.plan_num_ops == S.base_ops + 4 and not torch.equal(adapted, S.base)
    S.d.set_t2i_adapters([])
    assert torch.equal(S.fwd(), S.base)
    assert S.d.plan_num_ops == S.base_ops and S.d.plan_flops == S.base_flops   # the same plan as before any attach
    fresh = Diffuser(S.ctx, TINY, S.w)
    assert torch.equal(fresh.unet_forward(X, [T], S.c, S.y), S.base)
    fresh.close()
    S.d.set_t2i_adapters([(S.ads[0], S.h[0], 0.0)])
    assert torch.equal(S.fwd(), S.base)
    S.d.set_t2i_adapters([(S.ads[0], S.h[0], 1.0)], t_min=T + 1)
    assert torch.equal(S.fwd(), S.base)                     # t < t_min: nothing added
    S.d.set_t2i_adapters([(S.ads[0], S.h[0], 1.0)], t_min=T)
    assert torch.equal(S.fwd(), adapted)                    # t >= t_min
    S.d.set_t2i_adapters([])


def test_rewrite_in_place_matches_fresh_attach(S):
    S.d.set_t2i_adapters([(S.ads[0], S.h[0], 0.5)])
    S.fwd()
    S.fwd()                                                 # plan built and graph captured
    n = plan_builds(S.d)
    results = []
    for items, t_min in (([(S.ads[0], S.h[0], 1.3)], 0), ([(S.ads[0], S.h[0].flip(3), 1.3)], 0), ([(S.ads[0], S.h[0], 1.3)], T + 1),
                         ([(S.ads[1], S.h[0], 0.7)], 0)):
        S.d.set_t2i_adapters(items, t_min=t_min)            # same n_hint and size: features and t_min rewritten in place
        results.append(S.fwd())
        assert plan_builds(S.d) == n
    for (items, t_min), want in zip((([(S.ads[0], S.h[0], 1.3)], 0), ([(S.ads[0], S.h[0].flip(3), 1.3)], 0),
                                     ([(S.ads[0], S.h[0], 1.3)], T + 1), ([(S.ads[1], S.h[0], 0.7)], 0)), results):
        S.d.set_t2i_adapters([])
        S.d.set_t2i_adapters(items, t_min=t_min)
        assert torch.equal(S.fwd(), want)
    assert torch.equal(results[2], S.base)
    S.d.set_t2i_adapters([])


def test_batch_rows_use_their_own_features(S):
    h0, h1 = S.h[0][:1], S.h[0][1:]
    S.d.set_t2i_adapters([(S.ads[0], torch.cat([h0, h1]), 1.0)])
    mixed = S.fwd()
    S.d.set_t2i_adapters([(S.ads[0], h0, 1.0)])
    only0 = S.fwd()
    S.d.set_t2i_adapters([(S.ads[0], h1, 1.0)])
    only1 = S.fwd()
    S.d.set_t2i_adapters([])
    assert torch.equal(mixed[0], only0[0]) and torch.equal(mixed[1], only1[1]) and not torch.equal(mixed[0], only1[0])


def test_refusals_leave_the_previous_set(S, ctx):
    S.d.set_t2i_adapters([(S.ads[0], S.h[0], 1.0)])
    want = S.fwd()
    n = plan_builds(S.d)

    def unchanged():
        assert torch.equal(S.fwd(), want) and plan_builds(S.d) == n

    with pytest.raises(SdxlError, match="multiples of 32"):
        S.d.set_t2i_adapters([(S.ads[0], hint(2, 1, size=112), 1.0)])
    unchanged()
    with pytest.raises(SdxlError, match="differ from item 0"):
        S.d.set_t2i_adapters([(S.ads[0], S.h[0], 1.0), (S.ads[1], S.h[1], 1.0)])
    unchanged()
    with pytest.raises(SdxlError, match="differ from item 0"):
        S.d.set_t2i_adapters([(S.ads[0], S.h[0], 1.0), (S.ads[1], hint(2, 3, size=96), 1.0)])
    unchanged()
    with pytest.raises(SdxlError, match="at most 4"):
        S.d.set_t2i_adapters([(S.ads[0], S.h[0], 1.0)] * 5)
    arr = (_lib.T2IControl * 5)()
    for i in range(5):
        arr[i].adapter, arr[i].hint, arr[i].n_hint, arr[i].height, arr[i].width, arr[i].scale = S.ads[0].h.value, 1, 1, 128, 128, 1.0
    assert S.d.ctx.lib.sdxl_unet_set_t2i_adapters(S.d.h, 5, arr, 0) != 0
    unchanged()
    with pytest.raises(SdxlError, match="not finite"):
        S.d.set_t2i_adapters([(S.ads[0], S.h[0], float("nan"))])
    unchanged()
    other_cfg = T2IAdapterConfig(UNetConfig(adm_in_channels=16, model_channels=64, channel_mults=(1, 2, 4), transformer_depths=(0, 1, 2),
                                            context_dim=24))
    other = T2IAdapter(ctx, other_cfg, synth_weights(other_cfg, seed=4))
    with pytest.raises(SdxlError, match="adm_in_channels"):
        S.d.set_t2i_adapters([(other, S.h[0], 1.0)])
    unchanged()
    other.close()
    with pytest.raises(SdxlError, match="still attached"):
        S.ads[0].close()
    # forwards the attached set cannot serve
    with pytest.raises(SdxlError, match="latent"):
        S.d.unet_forward(arb(2, 4, 8, 8), [T], S.c, S.y)
    S.d.set_t2i_adapters([(S.ads[0], S.h[0], 1.0)])          # n_hint = 2
    with pytest.raises(SdxlError, match="multiple of n_hint"):
        S.d.unet_forward(X[:1], [T], S.c[:1], S.y[:1])
    with pytest.raises(SdxlError, match="multiple of n_hint"):
        S.d.sample_latent(Conditioning(**tiny_conditioning(B=1)), 7.5, 2, noise=S.noise[:1])
    assert torch.equal(S.fwd(), want)
    S.d.set_t2i_adapters([])


def test_refiner_and_foreign_cfgs_refused(ctx):
    from sdxl_b200 import TINY_REFINER
    with pytest.raises(SdxlError, match="refiner"):
        T2IAdapter(ctx, T2IAdapterConfig(TINY_REFINER), synth_weights(T2IAdapterConfig(TINY_REFINER), seed=0))
    four = UNetConfig(adm_in_channels=8, model_channels=64, channel_mults=(1, 2, 4, 4), transformer_depths=(0, 1, 1, 1), context_dim=24)
    with pytest.raises(SdxlError, match="3 levels"):
        T2IAdapter(ctx, T2IAdapterConfig(four), synth_weights(T2IAdapterConfig(four), seed=0))


def test_pipeline_t2i_adapters_attach_for_the_call(ctx):
    import os
    from sdxl_b200 import TINY_CLIP, TINY_OPEN_CLIP, TINY_VAE, ClipTextEncoder, Embedder, LatentDecoder, OpenClipTokenizer
    from sdxl_b200.pipeline import sample
    mini = os.path.join(os.path.dirname(__file__), "golden", "mini_bpe")
    ca, cb = TINY_CLIP, TINY_OPEN_CLIP
    ucfg = UNetConfig(adm_in_channels=cb.embed_dim + 6 * 256, model_channels=64, channel_mults=(1, 2, 4), transformer_depths=(0, 1, 1),
                      context_dim=ca.n_state + cb.n_state)
    acfg = T2IAdapterConfig(ucfg)
    tok = OpenClipTokenizer(os.path.join(mini, "mini_merges.txt"), os.path.join(mini, "mini_vocab.txt"))
    emb = Embedder(ctx, ClipTextEncoder(ctx, ca, synth_weights(ca, seed=1)), ClipTextEncoder(ctx, cb, synth_weights(cb, seed=2)), tok, tok)
    dif = Diffuser(ctx, ucfg, synth_weights(ucfg, seed=3))
    vae = LatentDecoder(ctx, TINY_VAE, synth_weights(TINY_VAE, seed=0))
    ad = T2IAdapter(ctx, acfg, synth_weights(acfg, seed=4))
    image = (torch.rand(1, 64, 64, 3, generator=torch.Generator().manual_seed(3)) * 255).to(torch.uint8)
    kw = dict(guidance=5.0, n_steps=4, resolution=(64, 64), seed=0)
    plain = sample(emb, dif, vae, "a photo of a cat", **kw)
    adapted = sample(emb, dif, vae, "a photo of a cat", t2i_adapters=[(ad, image, 1.0)], t2i_factor=0.5, **kw)
    dif.set_t2i_adapters([(ad, image.permute(0, 3, 1, 2).float() / 255.0, 1.0)], t_min=t2i_t_min(4, 0.5))
    same = sample(emb, dif, vae, "a photo of a cat", **kw)
    dif.set_t2i_adapters([])
    assert torch.equal(adapted, same) and not torch.equal(adapted, plain)
    assert torch.equal(sample(emb, dif, vae, "a photo of a cat", **kw), plain)   # detached after the call
    ad.close()
    dif.close()
