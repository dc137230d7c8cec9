"""SDXL base (synthetic weights) at full size with each kind of attachment: one forward against the f32 oracle
(oracle/unet_oracle.py), with the bound of the uncontrolled 1024^2 forward (test_fullsize_gpu).

 * ControlNet (synthetic weights, non-zero zero convs): the hint encoder and one CFG-batched forward.
 * FreeU at the SDXL values the FreeU authors recommend: one CFG-batched forward.
 * A ViT-H-sized IP-Adapter (D = 1024, 4 tokens): one CFG-batched forward with an image prompt.
 * A ViT-H-sized IP-Adapter Plus (image features 257 x 1280, Resampler of depth 4, 20 heads, 16 tokens): one CFG-batched forward.
 * A base and a Plus adapter masked to the left and right halves of the image, at 1024 x 1024 and at 832 x 1216.
 * Perturbed-attention guidance on the 10 mid-block self-attentions: one batched forward of the three row groups
   [cond | uncond | ptb].
 * An SDXL-sized T2I-Adapter (synthetic weights, drawn on the CPU generator): its four features and one CFG-batched forward.

Every test attaches to one SDXL base, drawn, widened for the oracle and loaded once for the module."""
import pytest
import torch

import sdxl_b200
from sdxl_b200 import SDXL_BASE, SDXL_CONTROLNET, SDXL_T2I_ADAPTER, ControlNet, Diffuser, IPAdapter, T2IAdapter, pag_layer_mask
from sdxl_b200.ip_adapter import SDXL_PLUS, synth_ip_adapter
from oracle import unet_oracle as O
import freeu_oracle as FO
import ip_adapter_oracle as IPO
import ip_adapter_plus_oracle as IPPO
import pag_oracle as PO
import t2i_adapter_oracle as TA
from harness import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-3


@pytest.fixture(scope="module")
def base(ctx):
    """(the SDXL base on the device, its weights in f32 for the oracle); the f16 draw is dropped once both are made."""
    w = sdxl_b200.synth_weights(SDXL_BASE, seed=0)
    d = Diffuser(ctx, SDXL_BASE, w)
    wf = O.to_f32(w)
    del w
    yield d, wf
    d.close()


@pytest.fixture(autouse=True)
def detach_all(base):
    """A test that fails with something attached must not leave it on the shared UNet for the next one."""
    yield
    d = base[0]
    d.set_controls([])
    d.set_image_prompts([])
    d.set_t2i_adapters([])
    d.set_pag(None)
    d.set_freeu(None)


def test_controlnet_1024(ctx, base):
    d, wf = base
    wc = sdxl_b200.synth_weights(SDXL_CONTROLNET, seed=1)
    net = ControlNet(ctx, SDXL_CONTROLNET, wc)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 128, 128, generator=g)
    c = torch.randn(2, 77, 2048, generator=g).half().float()
    y = torch.randn(2, 2816, generator=g).half().float()
    hint = torch.rand(1, 3, 1024, 1024, generator=g)
    wcf = O.to_f32(wc)
    emb = net.embed_hint(hint)
    emb_ref = O.hint_embedding(SDXL_CONTROLNET, wcf, hint)
    e_hint = rel_err(emb, emb_ref)
    d.set_controls([(net, hint, 1.0)])          # n_hint = 1: both CFG rows use the image's hint
    got = d.unet_forward(x, [749], c, y)
    d.set_controls([])
    base_out = d.unet_forward(x, [749], c, y)
    net.close()
    ref = O.unet_forward(SDXL_BASE, wf, x, torch.tensor([749]), c, y, O.Attach(controls=[(SDXL_CONTROLNET, wcf, hint, 1.0)]))
    e = rel_err(got, ref)
    print(f"SDXL ControlNet 1024^2: hint_emb rel err {e_hint:.2e}, CFG-batched forward rel err {e:.2e}, "
          f"the control moves the forward by {rel_err(got, base_out):.2e}")
    assert e_hint <= TOL and e <= TOL and rel_err(got, base_out) > 0.05


def test_freeu_1024(base):
    d, wf = base
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1, 4, 128, 128, generator=g).repeat(2, 1, 1, 1)
    c = torch.randn(2, 77, 2048, generator=g).half().float()
    y = torch.randn(2, 2816, generator=g).half().float()
    d.set_freeu(*FO.RECOMMENDED_SDXL)
    got = d.unet_forward(x, [749], c, y).cpu()
    d.set_freeu(None)
    base_out = d.unet_forward(x, [749], c, y).cpu()
    ref = O.unet_forward(SDXL_BASE, wf, x, torch.tensor([749]), c, y, O.Attach(freeu=FO.RECOMMENDED_SDXL))
    err, moved = rel_err(got, ref), rel_err(got, base_out)
    print(f"SDXL FreeU 1024^2: forward rel err {err:.3e}; FreeU moves the forward by {moved:.3e}")
    assert err < TOL and moved > 1e-2


def test_ip_adapter_1024(ctx, base):
    d, wf = base
    wa = synth_ip_adapter(SDXL_BASE, 1024, seed=1)
    ad = IPAdapter(ctx, SDXL_BASE, 1024, wa)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 128, 128, generator=g)
    c = torch.randn(2, 77, 2048, generator=g).half().float()
    y = torch.randn(2, 2816, generator=g).half().float()
    e = torch.randn(1, 1, 1024, generator=g)
    d.set_image_prompt(ad, e, 1.0)              # n_batch = 1: both rows use the image
    got = d.unet_forward(x, [749], c, y)
    d.set_image_prompt(None)
    ad.close()
    waf = O.to_f32(wa)
    tok = IPO.prompt_tokens(waf, e).repeat(2, 1, 1)
    ref = O.unet_forward(SDXL_BASE, wf, x, torch.tensor([749]), c, y, O.Attach(prompts=[(waf, tok, IPO.uniform_scales(SDXL_BASE, 1.0), None)]))
    err = rel_err(got, ref)
    print(f"SDXL base + IP-Adapter 1024^2 forward: rel err {err:.3e}")
    assert err < TOL


def test_ip_adapter_plus_1024(ctx, base):
    d, wf = base
    wa = synth_ip_adapter(SDXL_BASE, 1280, seed=1, resampler=SDXL_PLUS)
    ad = IPAdapter(ctx, SDXL_BASE, 1280, wa)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 128, 128, generator=g)
    c = torch.randn(2, 77, 2048, generator=g).half().float()
    y = torch.randn(2, 2816, generator=g).half().float()
    h = torch.randn(1, 1, 257, 1280, generator=g)
    d.set_image_prompt(ad, h, 1.0, negative=torch.zeros_like(h))   # n_batch = 1: both rows use the image
    got = d.unet_forward(x, [749], c, y)
    d.set_image_prompt(None)
    ad.close()
    waf = O.to_f32(wa)
    tok = IPPO.plus_prompt_tokens(waf, h).repeat(2, 1, 1)
    ref = O.unet_forward(SDXL_BASE, wf, x, torch.tensor([749]), c, y, O.Attach(prompts=[(waf, tok, IPO.uniform_scales(SDXL_BASE, 1.0), None)]))
    err = rel_err(got, ref)
    print(f"SDXL base + IP-Adapter Plus 1024^2 forward: rel err {err:.3e}")
    assert err < TOL


@pytest.mark.parametrize("H,W", [(1024, 1024), (832, 1216)])
def test_base_and_plus_masked_halves(ctx, base, H, W):
    d, wf = base
    wa = synth_ip_adapter(SDXL_BASE, 1024, seed=1)
    wp = synth_ip_adapter(SDXL_BASE, 1280, seed=2, resampler=SDXL_PLUS)
    ad = IPAdapter(ctx, SDXL_BASE, 1024, wa)
    plus = IPAdapter(ctx, SDXL_BASE, 1280, wp)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, H // 8, W // 8, generator=g)
    c = torch.randn(2, 77, 2048, generator=g).half().float()
    y = torch.randn(2, 2816, generator=g).half().float()
    e = torch.randn(1, 1, 1024, generator=g)
    h = torch.randn(1, 1, 257, 1280, generator=g)
    left = torch.zeros(1, H, W)
    left[:, :, :W // 2] = 1
    right = 1 - left
    d.set_image_prompts([(ad, e, 0.8, None, left), (plus, h, 0.7, torch.zeros_like(h), right)])   # n_batch = 1: both rows
    got = d.unet_forward(x, [749], c, y)
    d.set_image_prompts([])
    ad.close()
    plus.close()
    waf, wpf = O.to_f32(wa), O.to_f32(wp)
    prompts = [(waf, IPO.prompt_tokens(waf, e).repeat(2, 1, 1), IPO.uniform_scales(SDXL_BASE, 0.8), left),
               (wpf, IPPO.plus_prompt_tokens(wpf, h).repeat(2, 1, 1), IPO.uniform_scales(SDXL_BASE, 0.7), right)]
    ref = O.unet_forward(SDXL_BASE, wf, x, torch.tensor([749]), c, y, O.Attach(prompts=prompts))
    err = rel_err(got, ref)
    print(f"SDXL base + base and Plus adapters, masked halves, {H}x{W} forward: rel err {err:.3e}")
    assert err < TOL


def test_pag_mid_1024(base):
    d, wf = base
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1, 4, 128, 128, generator=g).repeat(3, 1, 1, 1)     # the sampler broadcasts one latent to every row group
    c = torch.randn(2, 77, 2048, generator=g).half().float()
    y = torch.randn(2, 2816, generator=g).half().float()
    c, y = torch.cat([c, c[:1]]), torch.cat([y, y[:1]])                  # the perturbed row repeats the conditional one
    mask = pag_layer_mask(SDXL_BASE, "mid")
    d.set_pag("mid", 3.0)
    got = d.unet_forward(x, [749], c, y, perturbed_rows=1).cpu()
    d.set_pag(None)
    base_out = d.unet_forward(x, [749], c, y).cpu()
    ref = PO.forward_rows(SDXL_BASE, wf, x, torch.tensor([749]), c, y, PO.paths_of_mask(SDXL_BASE, mask), 1)
    err, moved = rel_err(got, ref), rel_err(got[2], base_out[2])
    print(f"SDXL PAG (mid) 1024^2: forward rel err {err:.3e}; PAG moves the perturbed row by {moved:.3e}; "
          f"attended rows bit-identical to the unperturbed forward: {torch.equal(got[:2], base_out[:2])}")
    assert err < TOL and moved > 1e-2
    assert torch.equal(got[:2], base_out[:2])


def test_t2i_adapter_1024(ctx, base):
    d, wf = base
    wa = sdxl_b200.synth_weights(SDXL_T2I_ADAPTER, seed=1)
    ad = T2IAdapter(ctx, SDXL_T2I_ADAPTER, wa)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 128, 128, generator=g)
    c = torch.randn(2, 77, 2048, generator=g).half().float()
    y = torch.randn(2, 2816, generator=g).half().float()
    hint = torch.rand(1, 3, 1024, 1024, generator=g)
    feats = ad.features(hint)
    d.set_t2i_adapters([(ad, hint, 1.0)])   # n_hint = 1: both rows use the hint
    got = d.unet_forward(x, [749], c, y)
    d.set_t2i_adapters([])
    base_out = d.unet_forward(x, [749], c, y)
    ad.close()
    waf = O.to_f32(wa)
    ref_feats = TA.adapter_features(SDXL_T2I_ADAPTER, waf, hint)
    feat_errs = [rel_err(a, b) for a, b in zip(feats, ref_feats)]
    att = O.Attach(t2i=(TA.summed_features([(SDXL_T2I_ADAPTER, waf, hint, 1.0)]), 0))
    ref = O.unet_forward(SDXL_BASE, wf, x, torch.tensor([749]), c, y, att)
    err, moved = rel_err(got, ref), rel_err(got, base_out)
    print(f"SDXL T2I-Adapter 1024^2: feature rel errs {['%.3e' % e for e in feat_errs]}; forward rel err {err:.3e}; "
          f"the adapter moves the output by {moved:.3e}")
    assert max(feat_errs) < TOL and err < TOL and moved > 1e-2
