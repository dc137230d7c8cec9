"""SDXL base (synthetic weights) with an SDXL-sized T2I-Adapter (synthetic weights, drawn on the CPU generator) at 1024x1024: the
adapter's four features and one CFG-batched forward with the adapter attached, against the f32 oracle, with the bound of the 1024^2
forward (test_fullsize_gpu)."""
import pytest
import torch

import sdxl_b200
from sdxl_b200 import SDXL_BASE, SDXL_T2I_ADAPTER, Diffuser, T2IAdapter
from oracle import unet_oracle as O
import t2i_adapter_oracle as TA

pytestmark = pytest.mark.gpu
TOL = 1e-3


def rel_err(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def test_t2i_adapter_1024(ctx):
    w = sdxl_b200.synth_weights(SDXL_BASE, seed=0)
    wa = sdxl_b200.synth_weights(SDXL_T2I_ADAPTER, seed=1)
    d = Diffuser(ctx, SDXL_BASE, w)
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
    base = d.unet_forward(x, [749], c, y)
    d.close()
    ad.close()
    waf = O.to_f32(wa)
    ref_feats = TA.adapter_features(SDXL_T2I_ADAPTER, waf, hint)
    feat_errs = [rel_err(a, b) for a, b in zip(feats, ref_feats)]
    att = O.Attach(t2i=(TA.summed_features([(SDXL_T2I_ADAPTER, waf, hint, 1.0)]), 0))
    ref = O.unet_forward(SDXL_BASE, O.to_f32(w), x, torch.tensor([749]), c, y, att)
    err, moved = rel_err(got, ref), rel_err(got, base)
    print(f"SDXL T2I-Adapter 1024^2: feature rel errs {['%.3e' % e for e in feat_errs]}; forward rel err {err:.3e}; "
          f"the adapter moves the output by {moved:.3e}")
    assert max(feat_errs) < TOL and err < TOL and moved > 1e-2
