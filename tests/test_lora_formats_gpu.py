"""GPU tests of the adapter families beyond LoRA (LoHa, LoKr, full delta) and of DoRA, merged on the device (DESIGN.md §19), tiny
configs.

Exactness follows tests/test_lora_gpu.py: factors in {-1, 0, 1} / 16 (/ 4 for LoKr's w1), no alpha and a power-of-two scale make every
f32 product and sum exact, so a model merged in place must compute exactly what a model loaded from `merge_into` weights computes
(upsample convs: within the oracle bounds). DoRA divides by a norm, so its merged weights are held to the float64 merge within one
f16 ulp (kernel level) and the forward to the f32 oracle on `merge_into` weights.
"""
import os
import subprocess
import sys

import pytest
import torch

import sdxl_b200
from sdxl_b200 import TINY, TINY_CLIP, TINY_OPEN_CLIP, TINY_VAE, ClipTextEncoder, Embedder, LatentDecoder, OpenClipTokenizer, SdxlError, \
    UNetConfig, _testing, synth_weights
from sdxl_b200.lora import merge_into
from sdxl_b200.pipeline import sample
from oracle import clip_oracle as CO
from oracle import unet_oracle as O
from lora_cases import layer_paths, write_safetensors
from lora_family_cases import add_dora, make_family, to_file
from harness import plan_builds, rel_err
from test_lora_gpu import FWD_TOL, T, X, Tiny, exact_paths

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def tiny(ctx):
    t = Tiny(ctx)
    t.base_fwd = t.fwd()
    t.base_smp = t.smp()
    yield t
    t.d.close()


# ---- exact families -----------------------------------------------------------------------------------------------------------------
CASES = [("loha", None), ("lokr", 0), ("lokr", 1), ("lokr", 2), ("lokr", 3), ("full", None)]


@pytest.mark.parametrize("family,mode", CASES)
def test_exact_families_equal_host_merge(tiny, family, mode):
    t = tiny
    t.fwd()
    n_ops, builds = t.d.plan_num_ops, plan_builds(t.d)
    ad = make_family(TINY, exact_paths(TINY), family, seed=3, lokr_mode=mode)
    t.d.set_adapters([(ad, 0.5)])
    got = t.fwd(set_cond=False)
    assert t.d.plan_num_ops == n_ops and plan_builds(t.d) == builds
    ref_model = t.loaded(merge_into(t.w, ad, 0.5))
    want = t.fwd(ref_model)
    assert not torch.equal(want, t.base_fwd)
    assert torch.equal(got, want)
    assert torch.equal(t.smp(), t.smp(ref_model))
    ref_model.close()
    t.d.set_adapters([])
    assert torch.equal(t.fwd(), t.base_fwd)


def test_exact_families_stacked(tiny):
    t = tiny
    sets = [(make_family(TINY, exact_paths(TINY), f, seed=10 + i), 0.5) for i, f in enumerate(("lora", "loha", "lokr", "full"))]
    t.d.set_adapters(sets)
    ref_model = t.loaded(merge_into(t.w, sets))
    assert torch.equal(t.fwd(), t.fwd(ref_model))
    ref_model.close()
    t.d.set_adapters([])
    assert torch.equal(t.fwd(), t.base_fwd)


@pytest.mark.parametrize("family,mode", [("lora", None), ("loha", None), ("lokr", 1), ("lokr", 3)])
def test_negative_alpha_equals_host_merge(tiny, family, mode):
    """A finite negative alpha is used as given (c = alpha / r < 0), as the LoRA merge always did."""
    t = tiny
    ad = make_family(TINY, exact_paths(TINY), family, seed=30, lokr_mode=mode, alpha=-2.0)   # rank 2: c = -1
    t.d.set_adapters([(ad, 0.5)])
    got = t.fwd()
    ref_model = t.loaded(merge_into(t.w, ad, 0.5))
    assert torch.equal(got, t.fwd(ref_model))
    pos = t.loaded(merge_into(t.w, {k: (-v if k.endswith("/alpha") else v) for k, v in ad.items()}, 0.5))
    assert not torch.equal(got, t.fwd(pos))
    pos.close()
    ref_model.close()
    t.d.set_adapters([])


@pytest.mark.parametrize("family", ("loha", "lokr", "full"))
def test_upsample_convs_vs_oracle(tiny, family):
    t = tiny
    ad = make_family(TINY, layer_paths(TINY), family, seed=5)
    assert any("/upsample/" in k for k in ad)
    t.d.set_adapters([(ad, 0.5)])
    wf = O.to_f32(merge_into(t.w, ad, 0.5))
    out = t.fwd()
    e = rel_err(out, O.unet_forward(TINY, wf, X, torch.tensor([T]), t.c, t.y))
    print(f"tiny forward, {family} on every layer vs oracle on merged weights: rel err {e:.3e}")
    assert e < FWD_TOL and rel_err(out, t.base_fwd) > 10 * FWD_TOL
    t.d.set_adapters([])


# ---- DoRA -----------------------------------------------------------------------------------------------------------------------------
def _dora_sets(w, axis):
    paths = exact_paths(TINY)
    lora = make_family(TINY, paths, "lora", seed=1, dyadic=False, alpha=2.0)
    loha = make_family(TINY, paths, "loha", seed=2, dyadic=False)
    return {"alone": [(add_dora(TINY, lora, w, axis, seed=3), 1.0)],
            "with_lora": [(lora, 0.5), (add_dora(TINY, loha, w, axis, seed=4), 0.7)],
            "with_loha": [(add_dora(TINY, make_family(TINY, paths, "lokr", seed=5, dyadic=False), w, axis, seed=6), 1.3), (loha, 0.5)]}


@pytest.mark.parametrize("axis", (0, 1))
def test_dora_vs_oracle(tiny, axis):
    t = tiny
    t.fwd()
    n_ops, builds = t.d.plan_num_ops, plan_builds(t.d)
    for name, sets in _dora_sets(t.w, axis).items():
        t.d.set_adapters(sets)
        out = t.fwd()
        wm = merge_into(t.w, sets)
        e = rel_err(out, O.unet_forward(TINY, O.to_f32(wm), X, torch.tensor([T]), t.c, t.y))
        moved = rel_err(out, t.base_fwd)
        print(f"DoRA axis {axis} {name}: forward vs oracle on merged weights {e:.3e} (the adapters move it {moved:.3e})")
        assert e < FWD_TOL and moved > 2 * FWD_TOL
        again = t.fwd()
        t.d.set_adapters(sets)
        assert torch.equal(t.fwd(), again)
    assert t.d.plan_num_ops == n_ops and plan_builds(t.d) == builds
    t.d.set_adapters([])
    assert torch.equal(t.fwd(), t.base_fwd) and torch.equal(t.smp(), t.base_smp)


# ---- kernels against float64 ----------------------------------------------------------------------------------------------------------
def _store(W, taps, f32=False, row0=3, col0=5):
    """W [N, Kd] (k = i * taps + tap) scattered into a padded K-major store, as the loader lays out a conv or a fused Linear slice."""
    N, Kd = W.shape
    I = Kd // taps
    Ipad = I + 11
    ld = col0 + taps * Ipad + 3
    k = torch.arange(Kd)
    cols = col0 + (k % taps) * Ipad + k // taps
    st = torch.zeros(row0 + N + 2, ld, dtype=torch.float32 if f32 else torch.float16)
    st[row0:row0 + N, cols] = W.to(st.dtype)
    return st.to(DEV), dict(ld=ld, row0=row0, col0=col0, Ipad=Ipad), cols


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _rand16(shape, seed, s=0.1):
    return (torch.randn(shape, generator=_g(seed)) * s).half()


@pytest.mark.parametrize("N,I,taps", [(100, 77, 1), (100, 35, 9)])
@pytest.mark.parametrize("r", (1, 33, 128))
def test_merge_kinds_kernel(N, I, taps, r):
    Kd = I * taps
    a, b = 10, (7 if I == 77 else 5)
    c, d = N // a, I // b
    up, down = _rand16((N, r), 1), _rand16((r, Kd), 2)
    r2 = 33 if r != 33 else 1
    up2, down2 = _rand16((N, r2), 3), _rand16((r2, Kd), 4)
    w1 = torch.randn(a, b, generator=_g(5)) * 0.3
    w2 = torch.randn(c, d * taps, generator=_g(6)) * 0.3
    diff = _rand16((N, Kd), 7, 0.01)
    dl = [x.to(DEV) for x in (up, down, up2, down2, w1, w2, diff)]
    up_d, down_d, up2_d, down2_d, w1_d, w2_d, diff_d = dl
    W = _rand16((N, Kd), 8, 1.0)
    st, lay, cols = _store(W, taps)
    f64 = {
        "lora": up.double() @ down.double(),
        "loha": (up.double() @ down.double()) * (up2.double() @ down2.double()),
        "lokr": torch.einsum("ip,jqt->ijpqt", w1.double(), w2.double().reshape(c, d, taps)).reshape(N, Kd),
        "full": diff.double(),
    }
    terms = {"lora": ("lora", 0.5, (up_d, down_d)), "loha": ("loha", 0.25, (up_d, down_d, up2_d, down2_d)),
             "lokr": ("lokr", 0.75, (w1_d, w2_d)), "full": ("full", 1.5, (diff_d,))}
    for name, term in list(terms.items()) + [("mixed", None)]:
        ts = list(terms.values()) if name == "mixed" else [term]
        outs = []
        for _ in range(2):
            o = torch.full((N, Kd), float("nan"), device=DEV)
            _testing.lora_merge_kinds(N, Kd, taps, ts, st, st, delta_out=o, **lay)
            outs.append(o.cpu())
        assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), name
        want = sum(cf * f64[k] for k, cf, _ in ts)
        err = float((outs[0].double() - want).abs().max() / want.abs().max())
        assert err < 3e-6, (name, err)
        if name == "lokr":   # one f32 product and one f32 scale per element: bit-exact
            assert torch.equal(outs[0], torch.tensor(0.75, dtype=torch.float32) * (w1.float().repeat_interleave(c, 0).repeat_interleave(d * taps, 1)
                               * w2.float().reshape(c, d * taps).repeat(a, b)))
        if name == "full":
            assert torch.equal(outs[0], torch.tensor(1.5, dtype=torch.float32) * diff.float())
    # a LoRA-only set runs the original kernel: the original binding gives the same bits
    o1, o2 = torch.zeros(N, Kd, device=DEV), torch.zeros(N, Kd, device=DEV)
    _testing.lora_merge_kinds(N, Kd, taps, [terms["lora"]], st, st, delta_out=o1, **lay)
    _testing.lora_merge(N, Kd, taps, [(up_d, down_d, 0.5)], st, st, delta_out=o2, **lay)
    assert torch.equal(o1, o2)


@pytest.mark.parametrize("f32", (False, True))
def test_f32_delta_apply_kernel(f32):
    N, I, taps = 70, 29, 9
    Kd = I * taps
    W = _rand16((N, Kd), 1, 1.0)
    src, lay, cols = _store(W, taps, f32=f32)
    dst = src.clone()
    delta = torch.randn(N, Kd, generator=_g(2)) * 0.01
    delta[:, ::7] = 0
    _testing.lora_merge_kinds(N, Kd, taps, [("f32", 1.0, (delta.to(DEV),))], src, dst, **lay)
    got = dst.cpu()[lay["row0"]:lay["row0"] + N][:, cols]
    want = torch.where(delta == 0, W.float(), (W.float() + delta).half().float()).to(got.dtype)
    assert torch.equal(got, want)
    rest = torch.ones_like(dst.cpu(), dtype=torch.bool)
    rest[lay["row0"]:lay["row0"] + N, cols] = False
    assert torch.equal(dst.cpu()[rest], src.cpu()[rest])   # nothing outside the slot is written


def _dora_f64(W, dw, taps, axis):
    V = W.double() + dw.double()
    N, Kd = V.shape
    if axis == 0:
        return V.pow(2).sum(1).sqrt()
    return V.reshape(N, Kd // taps, taps).pow(2).sum((0, 2)).sqrt()


@pytest.mark.parametrize("axis", (0, 1))
@pytest.mark.parametrize("N,I,taps,f32", [(100, 77, 1, False), (130, 35, 9, False), (66, 4, 9, True)])
def test_dora_norm_and_accum_kernels(axis, N, I, taps, f32):
    Kd = I * taps
    W = _rand16((N, Kd), 1, 0.5)
    dw = torch.randn(N, Kd, generator=_g(2)) * 0.05
    W[0] = 0
    dw[0] = 0
    if axis == 1:
        W[:, :taps] = 0
        dw[:, :taps] = 0
    st, lay, _ = _store(W, taps, f32=f32)
    J = N if axis == 0 else I
    norms = []
    for _ in range(2):
        nrm = torch.full((J,), float("nan"), dtype=torch.float64, device=DEV)
        _testing.dora_norm(N, Kd, taps, st, lay["ld"], dw.to(DEV), axis, nrm, row0=lay["row0"], col0=lay["col0"], Ipad=lay["Ipad"])
        norms.append(nrm.cpu())
    assert torch.equal(norms[0], norms[1])
    want = _dora_f64(W, dw, taps, axis)
    assert norms[0][0] == 0 and float(((norms[0] - want).abs() / want.clamp_min(1e-300)).max()) < 1e-12
    m = (torch.rand(J, generator=_g(3)) + 0.5).float()
    acc0 = torch.randn(N, Kd, generator=_g(4)) * 0.01
    accs = []
    for _ in range(2):
        acc = acc0.clone().to(DEV)
        _testing.dora_accum(N, Kd, taps, st, lay["ld"], dw.to(DEV), m.to(DEV), norms[0].to(DEV), axis, 0.7, acc, row0=lay["row0"],
                            col0=lay["col0"], Ipad=lay["Ipad"])
        accs.append(acc.cpu())
    assert torch.equal(accs[0], accs[1])
    V = W.double() + dw.double()
    mm = m.double()[:, None] if axis == 0 else m.double().repeat_interleave(taps)[None, :]
    nn = want[:, None] if axis == 0 else want.repeat_interleave(taps)[None, :]
    c = torch.where(nn == 0, torch.zeros_like(V), 0.7 * (mm * V / nn - W.double()))
    exp = acc0 + c.float()
    assert torch.allclose(accs[0], exp, rtol=1e-6, atol=1e-8)
    zero = (slice(0, 1), slice(None)) if axis == 0 else (slice(None), slice(0, taps))
    assert torch.equal(accs[0][zero], acc0[zero])   # n = 0: no term


# ---- refusals ---------------------------------------------------------------------------------------------------------------------------
def test_refusals_leave_the_model_unchanged(tiny):
    t = tiny
    good = make_family(TINY, exact_paths(TINY)[:30], "loha", seed=21)
    t.d.set_adapters([(good, 0.5)])
    before = t.fwd()
    p = "input_blocks/4/transformer/transformer_0/attn1/value"
    up_p = "output_blocks/2/upsample/conv"
    loha = make_family(TINY, [p, "conv_out"], "loha", seed=22)
    lokr = make_family(TINY, [p], "lokr", seed=23, lokr_mode=3)
    lora = make_family(TINY, [p], "lora", seed=24)
    N = 128
    lokr_ranks = dict(lokr, **{f"{p}/lokr_w2_a": torch.zeros(lokr[f"{p}/lokr_w2_a"].shape[0], 3, dtype=torch.float16),
                               f"{p}/lokr_w2_b": torch.zeros(3, lokr[f"{p}/lokr_w2_b"].shape[1], dtype=torch.float16)})
    cases = [   # (adapter, status code, what the message names)
        (dict(loha, **{f"{p}/lora_down": lora[f"{p}/lora_down"], f"{p}/lora_up": lora[f"{p}/lora_up"]}), 4615, f"{p}.*two delta families"),
        (dict(lokr, **{f"{p}/lokr_w1": torch.zeros(2, 2, dtype=torch.float16)}), 4615, f"{p}.*lokr_w1"),
        ({k: v for k, v in loha.items() if k != f"{p}/hada_w2_b"}, 4616, f"{p}/hada_w2_b"),
        ({k: v for k, v in lokr.items() if k != f"{p}/lokr_w1_b"}, 4616, f"{p}/lokr_w1_b"),
        (dict(loha, **{f"{p}/hada_w1_a": torch.zeros(N + 1, 2, dtype=torch.float16)}), 4617, f"{p}/hada_w1_a"),
        (dict(loha, **{f"{p}/hada_w1_b": torch.zeros(3, 128, dtype=torch.float16)}), 4618, f"{p}.*hada_w1_a has rank 2 but hada_w1_b"),
        (lokr_ranks, 4618, f"{p}.*lokr_w1_a has rank 2 but lokr_w2_a has rank 3"),
        (dict(lokr, **{f"{p}/lokr_w2_a": torch.zeros(lokr[f"{p}/lokr_w2_a"].shape[0] - 1, 2, dtype=torch.float16)}), 4619, f"{p}.*kron"),
        (dict(lora, **{f"{p}/dora_scale": torch.ones(N + 1)}), 4620, f"{p}/dora_scale"),
        (dict(lora, **{"conv_out/dora_scale": torch.ones(4)}), 4621, "conv_out/dora_scale"),
        (dict(make_family(TINY, [up_p], "lora", seed=25), **{f"{up_p}/dora_scale": torch.ones(TINY.model_channels * 4)}), 4622,
         f"{up_p}/dora_scale"),
        (dict(lora, **{f"{p}/dora_scale": torch.ones(N, dtype=torch.float16)}), 4623, f"{p}/dora_scale"),
    ]
    for bad, code, name in cases:
        with pytest.raises(SdxlError, match=rf"failed \({code}\): .*{name}"):
            t.d.set_adapters([(make_family(TINY, exact_paths(TINY)[:5], "full", seed=26), 1.0), (bad, 1.0)])
        assert torch.equal(t.fwd(), before), name
    t.d.set_adapters([])
    assert torch.equal(t.fwd(), t.base_fwd)


# ---- text encoders, pipeline, fills ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family", ("loha", "lokr", "full", "dora"))
def test_clip_adapters(ctx, family):
    w = synth_weights(TINY_OPEN_CLIP, seed=2)
    e = ClipTextEncoder(ctx, TINY_OPEN_CLIP, w)
    tok = torch.randint(1, 49405, (2, 77), generator=_g(4), dtype=torch.int32)
    tok[:, 0] = 49406
    tok[0, 9] = tok[1, 20] = 49407
    idx = TINY_OPEN_CLIP.n_layer - 1
    h0, p0 = e.forward_hidden_pooled(tok, idx)
    paths = layer_paths(TINY_OPEN_CLIP, clip=True)
    if family == "dora":
        ad = add_dora(TINY_OPEN_CLIP, make_family(TINY_OPEN_CLIP, paths, "loha", seed=41, clip=True, dyadic=False), w, 0, seed=42, clip=True)
    else:
        ad = make_family(TINY_OPEN_CLIP, paths, family, seed=41, clip=True)
    e.set_adapters([(ad, 0.5)])
    h, p = e.forward_hidden_pooled(tok, idx)
    wm = merge_into(w, ad, 0.5)
    hw, pw = CO.forward_hidden_pooled(TINY_OPEN_CLIP, O.to_f32(wm), tok, idx)
    assert rel_err(h, hw) <= FWD_TOL and rel_err(p, pw) <= FWD_TOL and rel_err(h, h0) > 2 * FWD_TOL
    if family != "dora":
        em = ClipTextEncoder(ctx, TINY_OPEN_CLIP, wm)
        hm, pm = em.forward_hidden_pooled(tok, idx)
        assert torch.equal(h, hm) and torch.equal(p, pm)
        em.close()
    e.set_adapters([])
    h1, p1 = e.forward_hidden_pooled(tok, idx)
    assert torch.equal(h1, h0) and torch.equal(p1, p0)
    e.close()


@pytest.mark.parametrize("scheme,family", [("kohya", "loha"), ("kohya_diffusers", "lokr"), ("peft", "lora"), ("diffusers", "full")])
def test_pipeline_sample_with_adapter_files(ctx, tmp_path, scheme, family):
    mini = os.path.join(os.path.dirname(__file__), "golden", "mini_bpe")
    ca, cb = TINY_CLIP, TINY_OPEN_CLIP
    ucfg = UNetConfig(adm_in_channels=cb.embed_dim + 6 * 256, model_channels=64, channel_mults=(1, 2, 4), transformer_depths=(0, 1, 1),
                      context_dim=ca.n_state + cb.n_state)
    wa, wb, wu, wv = (synth_weights(c, seed=s) for c, s in ((ca, 1), (cb, 2), (ucfg, 3), (TINY_VAE, 0)))
    tok = OpenClipTokenizer(os.path.join(mini, "mini_merges.txt"), os.path.join(mini, "mini_vocab.txt"))
    vae = LatentDecoder(ctx, TINY_VAE, wv)

    def models(a, b, u):
        return Embedder(ctx, ClipTextEncoder(ctx, ca, a), ClipTextEncoder(ctx, cb, b), tok, tok), sdxl_b200.Diffuser(ctx, ucfg, u)

    au = make_family(ucfg, exact_paths(ucfg), family, seed=51)
    a1 = make_family(ca, layer_paths(ca, clip=True), family, seed=52, clip=True)
    a2 = make_family(cb, layer_paths(cb, clip=True), family, seed=53, clip=True)
    path = str(tmp_path / "adapter.safetensors")
    write_safetensors(path, to_file(scheme, [("unet", ucfg, au), ("te1", ca, a1), ("te2", cb, a2)]))
    emb, dif = models(wa, wb, wu)
    kw = dict(guidance=5.0, n_steps=4, resolution=(64, 64), seed=0)
    base = sample(emb, dif, vae, "a photo of a cat", **kw)
    got = sample(emb, dif, vae, "a photo of a cat", loras=[(path, 0.5)], **kw)
    emb_m, dif_m = models(merge_into(wa, a1, 0.5), merge_into(wb, a2, 0.5), merge_into(wu, au, 0.5))
    want = sample(emb_m, dif_m, vae, "a photo of a cat", **kw)
    assert torch.equal(got, want) and not torch.equal(got, base)
    assert torch.equal(sample(emb, dif, vae, "a photo of a cat", **kw), base)


WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lora_formats_worker.py")
SWITCHES = ("SDXL_B200_FILL", "SDXL_B200_NO_GRAPH", "SDXL_B200_NO_PDL")


def _run_worker(name, env_extra, out_dir):
    env = {k: v for k, v in os.environ.items() if k not in SWITCHES}
    env.update(env_extra)
    out = os.path.join(out_dir, f"{name}.pt")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [WORKER, out]
    p = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, f"worker [{name}] exited with {p.returncode}:\n{p.stderr[-6000:]}"
    return torch.load(out, weights_only=True)


def test_fills_change_no_merge(tmp_path):
    base = _run_worker("base", {}, str(tmp_path))
    assert all(bool(torch.isfinite(v).all()) for v in base.values())
    for name, fill in (("nan", "0xff"), ("big", "0x7b")):
        got = _run_worker(name, {"SDXL_B200_FILL": fill}, str(tmp_path))
        for k in base:
            assert torch.equal(got[k], base[k]), (name, k)
