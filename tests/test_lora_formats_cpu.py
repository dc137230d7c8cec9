"""CPU tests of the adapter formats beyond kohya LoRA (DESIGN.md §19): the name tables of every naming scheme, load_adapter on
synthetic files of every family and scheme, its refusals, and the host merge (merge_into) against a float64 statement of each
family's delta and of DoRA."""
import numpy as np
import pytest
import torch

from sdxl_b200 import SDXL_BASE, SDXL_CLIP_L, SDXL_OPEN_CLIP_G, TINY, TINY_CLIP, TINY_OPEN_CLIP, synth_weights
from sdxl_b200.lora import adapter_module_table, clip_lora_modules, load_adapter, load_kohya, merge_into, unet_lora_modules
from lora_cases import layer_paths, make_adapter, to_kohya, write_safetensors
from lora_family_cases import FAMILIES, SCHEMES, add_dora, logical, make_family, module_names, to_file
from lora_cases import weight_shapes

MIXED = ["input_blocks/4/transformer/transformer_0/attn1/key", "input_blocks/4/res/skip_connection", "input_blocks/0",
         "input_blocks/4/res/lin_embed", "input_blocks/4/transformer/transformer_0/mlp/geglu/proj", "conv_out", "lin1_label_embed",
         "input_blocks/3"]


@pytest.mark.parametrize("scheme", SCHEMES)
def test_every_module_is_reachable(scheme):
    under, dotted = adapter_module_table(SDXL_BASE, SDXL_CLIP_L, SDXL_OPEN_CLIP_G)
    table = dotted if scheme in ("diffusers", "peft") else under
    for part, cfg, n in (("unet", SDXL_BASE, 794), ("te1", SDXL_CLIP_L, 72), ("te2", SDXL_OPEN_CLIP_G, 192)):
        names = module_names(scheme, part, cfg)
        assert len(names) == n and len(set(names.values())) == n
        assert all(table[m] == (part, r) for r, m in names.items())
    m = module_names(scheme, "unet", SDXL_BASE)
    if scheme == "kohya_diffusers":
        assert m["input_blocks/4/transformer/transformer_0/attn1/query"] == "lora_unet_down_blocks_1_attentions_0_transformer_blocks_0_attn1_to_q"
        assert m["output_blocks/2/upsample/conv"] == "lora_unet_up_blocks_0_upsamplers_0_conv"
    if scheme == "peft":
        assert m["middle_block/res1/conv_in"] == "unet.mid_block.resnets.0.conv1"
        assert module_names(scheme, "te2", SDXL_OPEN_CLIP_G)["blocks/3/mlp/fc2"] == "text_encoder_2.text_model.encoder.layers.3.mlp.fc2"


def _expected(ad):
    return {k: (v.float().reshape(()) if k.endswith("/alpha") else v) for k, v in ad.items()}


@pytest.mark.parametrize("scheme", SCHEMES)
@pytest.mark.parametrize("family", FAMILIES + ("dora",))
def test_files_round_trip(tmp_path, scheme, family):
    paths = MIXED
    w = synth_weights(TINY, seed=0)
    ad = make_family(TINY, paths, "loha" if family == "dora" else family, seed=3, alpha=4.0)
    if family == "dora":
        ad = add_dora(TINY, ad, w, axis=0, seed=4)
    te1 = make_family(TINY_CLIP, ["blocks/0/attn/query", "blocks/1/mlp/fc2"], family if family != "dora" else "lora", seed=5, clip=True)
    te2 = make_family(TINY_OPEN_CLIP, ["blocks/2/attn/out"], "lokr" if family == "lora" else "lora", seed=6, clip=True)
    f = to_file(scheme, [("unet", TINY, ad), ("te1", TINY_CLIP, te1), ("te2", TINY_OPEN_CLIP, te2)])
    f = {k: (t.float() if k.endswith(("lora_up.weight", "lora_B.weight", "diff")) else t) for k, t in f.items()}  # f32 factors -> f16
    p = tmp_path / "a.safetensors"
    write_safetensors(p, f)
    got = load_adapter(str(p), TINY, TINY_CLIP, TINY_OPEN_CLIP)
    for part, want in (("unet", ad), ("te1", te1), ("te2", te2)):
        assert set(got[part]) == set(want), part
        for k, v in _expected(want).items():
            dt = torch.float32 if k.endswith(("/alpha", "/dora_scale")) else torch.float16
            assert got[part][k].dtype == dt and got[part][k].shape == v.shape and torch.equal(got[part][k].float(), v.float()), k


def test_load_adapter_equals_load_kohya(tmp_path):
    ad = make_adapter(TINY, layer_paths(TINY), rank=3, seed=0, alpha=2.0)
    te = make_adapter(TINY_CLIP, layer_paths(TINY_CLIP, clip=True), rank=2, seed=1, clip=True)
    k = to_kohya(ad, unet_lora_modules(TINY))
    k.update(to_kohya(te, clip_lora_modules(TINY_CLIP, "lora_te1")))
    p = tmp_path / "k.safetensors"
    write_safetensors(p, k)
    a, b = load_adapter(str(p), TINY, TINY_CLIP, TINY_OPEN_CLIP), load_kohya(str(p), TINY, TINY_CLIP, TINY_OPEN_CLIP)
    assert a.keys() == b.keys()
    for part in a:
        assert a[part].keys() == b[part].keys()
        for n in a[part]:
            assert a[part][n].dtype == b[part][n].dtype and a[part][n].shape == b[part][n].shape and torch.equal(a[part][n], b[part][n])


@pytest.mark.parametrize("key,what", [
    ("lora_unet_input_blocks_4_1_proj_in.lora_mid.weight", "Tucker"),
    ("lora_unet_input_blocks_4_1_proj_in.hada_t1", "Tucker"),
    ("lora_unet_input_blocks_4_1_proj_in.lokr_t2", "Tucker"),
    ("lora_unet_input_blocks_4_1_proj_in.oft_blocks", "OFT"),
    ("unet.down_blocks.1.attentions.0.proj_in.boft_R", "OFT"),
    ("lora_unet_input_blocks_4_1_proj_in.weight", "IA3"),
    ("lora_unet_input_blocks_4_1_proj_in.on_input", "IA3"),
    ("lora_unet_input_blocks_4_1_proj_in.a1.weight", "GLoRA"),
    ("lora_unet_input_blocks_4_1_transformer_blocks_0_norm1.diff", "norm or bias"),
    ("lora_unet_input_blocks_4_1_proj_in.diff_b", "norm or bias"),
    ("unet.not_a_module.lora_A.weight", "known module"),
])
def test_refusals_name_every_key(key, what):
    good = to_file("kohya", [("unet", SDXL_BASE, make_adapter(SDXL_BASE, ["conv_out"], rank=1, seed=0))])
    good[key] = torch.zeros(1, dtype=torch.float16)
    good["lora_unet_nothing_here.alpha"] = torch.ones(())
    with pytest.raises(ValueError) as e:
        load_adapter(good, SDXL_BASE, SDXL_CLIP_L, SDXL_OPEN_CLIP_G)
    assert key in str(e.value) and what in str(e.value) and "lora_unet_nothing_here.alpha" in str(e.value)


def _f64_merge(w, sets, paths):
    """The table of DESIGN.md §19 written directly in float64 (products of the factors, kron by index, norms by loops over axes)."""
    out = dict(w)
    shapes = {p: tuple(w[p + "/weight"].shape) for p in paths}
    for p in paths:
        N, I, taps, conv = logical(shapes[p])
        W64 = w[p + "/weight"].double().numpy()
        W = W64.T if W64.ndim == 2 else W64.reshape(N, -1)
        plain, dora = np.zeros_like(W), np.zeros_like(W)
        for ad, s in sets:
            g = {k.rsplit("/", 1)[1]: v.double().numpy() for k, v in ad.items() if k.rsplit("/", 1)[0] == p}
            if not g:
                continue
            if "lora_down" in g:
                r = g["lora_down"].shape[0]
                P, c = g["lora_up"].reshape(N, r) @ g["lora_down"].reshape(r, -1), g.get("alpha", r) / r
            elif "hada_w1_a" in g:
                r = g["hada_w1_b"].shape[0]
                P = (g["hada_w1_a"] @ g["hada_w1_b"].reshape(r, -1)) * (g["hada_w2_a"] @ g["hada_w2_b"].reshape(g["hada_w2_b"].shape[0], -1))
                c = g.get("alpha", r) / r
            elif "diff" in g:
                P, c = g["diff"].reshape(N, -1), 1.0
            else:
                r = 0
                fs = []
                for n in ("lokr_w1", "lokr_w2"):
                    if n in g:
                        fs.append(g[n].reshape(g[n].shape[0], -1))
                    else:
                        r = g[n + "_a"].shape[1]
                        fs.append(g[n + "_a"] @ g[n + "_b"].reshape(r, -1))
                w1, w2 = fs
                cc, d = w2.shape[0], w2.shape[1] // taps
                P = np.zeros((N, I * taps))
                for i in range(w1.shape[0]):
                    for j in range(cc):
                        for pp in range(w1.shape[1]):
                            for q in range(d):
                                P[i * cc + j, (pp * d + q) * taps:(pp * d + q + 1) * taps] = w1[i, pp] * w2[j, q * taps:(q + 1) * taps]
                c = (g.get("alpha", r) / r) if r else 1.0
            if "dora_scale" not in g:
                plain += s * c * P
                continue
            V = W + c * P
            m = g["dora_scale"]
            if m.shape[0] == N and m.size == N:
                n = np.sqrt((V ** 2).sum(1, keepdims=True))
                mm = m.reshape(N, 1)
            else:
                n = np.sqrt(np.array([(V[:, i * taps:(i + 1) * taps] ** 2).sum() for i in range(I)])).repeat(taps)[None]
                mm = m.reshape(-1).repeat(taps)[None]
            dora += s * (mm * V / n - W)
        t = plain + dora
        M = W + t
        M = M.T if W64.ndim == 2 else M.reshape(W64.shape)
        t = t.T if W64.ndim == 2 else t.reshape(W64.shape)
        out[p + "/weight"] = torch.where(torch.from_numpy(t == 0), w[p + "/weight"], torch.from_numpy(M).half())
    return out


def _ulps(a, b):
    ia, ib = a.view(torch.int16).int(), b.view(torch.int16).int()
    ia = torch.where(ia < 0, -32768 - ia, ia)
    ib = torch.where(ib < 0, -32768 - ib, ib)
    return int((ia - ib).abs().max())


@pytest.mark.parametrize("family", FAMILIES)
def test_merge_into_exact_families(family):
    w = synth_weights(TINY, seed=0)
    for mode in (0, 1, 2, 3):
        ad = make_family(TINY, MIXED, family, seed=7 + mode, lokr_mode=mode if family == "lokr" else None)
        m = merge_into(w, ad, 0.5)
        ref = _f64_merge(w, [(ad, 0.5)], MIXED)
        for p in MIXED:
            assert torch.equal(m[p + "/weight"].view(torch.int16), ref[p + "/weight"].view(torch.int16)), (family, mode, p)
            assert not torch.equal(m[p + "/weight"], w[p + "/weight"])
        if family != "lokr":
            break


@pytest.mark.parametrize("axis", (0, 1))
def test_merge_into_dora(axis):
    w = synth_weights(TINY, seed=0)
    lora = make_family(TINY, MIXED, "lora", seed=1, dyadic=False, alpha=3.0)
    loha = make_family(TINY, MIXED, "loha", seed=2, dyadic=False)
    lokr = make_family(TINY, MIXED, "lokr", seed=3, dyadic=False)
    for base, s in ((lora, 1.0), (loha, 0.7), (lokr, 1.3)):
        d = add_dora(TINY, base, w, axis, seed=11)
        for sets in ([(d, s)], [(lora, 0.5), (d, s)], [(d, s), (make_family(TINY, MIXED, "loha", seed=4, dyadic=False), 0.8)]):
            m = merge_into(w, sets)
            ref = _f64_merge(w, sets, MIXED)
            for p in MIXED:
                assert _ulps(m[p + "/weight"], ref[p + "/weight"]) <= 1, p
                assert not torch.equal(m[p + "/weight"], w[p + "/weight"])


def test_merge_into_stacking_exact():
    w = synth_weights(TINY, seed=0)
    sets = [(make_family(TINY, MIXED, f, seed=20 + i), 0.5) for i, f in enumerate(FAMILIES)]
    m, ref = merge_into(w, sets), _f64_merge(w, sets, MIXED)
    for p in MIXED:
        assert torch.equal(m[p + "/weight"].view(torch.int16), ref[p + "/weight"].view(torch.int16)), p
