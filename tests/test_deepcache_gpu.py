"""GPU tests of DeepCache (sdxl_unet_set_deepcache, DESIGN.md §17), tiny configs: interval 1 and detaching are bit-identical to the
plain calls, a full forward with DeepCache attached is the plain forward, the cached forward right after a full one on the same
inputs is that forward bit for bit for every branch and with every attachment (FreeU's in-place scale does not compound), cached
forwards at new inputs and interval-3 samples against the f32 oracle (tests/deepcache_oracle.py), the sampler's evaluation count,
the plan builds, the refusals, the pipeline's per-call attach, and bit-identity under fresh-memory fills, eager launches and no PDL
(tests/deepcache_invariance_worker.py, one subprocess per configuration)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import sdxl_b200
from sdxl_b200 import (TINY, TINY_CONTROLNET, TINY_INPAINT, TINY_REFINER, TINY_T2I_ADAPTER, Conditioning, ControlNet, Diffuser, IPAdapter,
                       SdxlError, T2IAdapter, _lib, pag_layer_mask, synth_weights)
from sdxl_b200.ip_adapter import synth_ip_adapter
from sdxl_b200.schedulers import SAMPLERS, Schedule
from oracle import unet_oracle as O
import deepcache_oracle as DO
import freeu_oracle as FO
import pag_oracle as PO
import scheduler_oracle as SO
from harness import first_difference, h16f, plan_builds, rel_err, tiny_conditioning

pytestmark = pytest.mark.gpu
FWD_TOL = 2e-3
SAMPLE_TOL = 5e-3
T = 499
FV = FO.RECOMMENDED_SDXL
N_BRANCH = 9   # 3 * n_levels of TINY and TINY_REFINER


def gen(seed):
    return torch.Generator().manual_seed(seed)


class Setup:
    def __init__(self, ctx):
        self.ctx = ctx
        self.w = synth_weights(TINY, seed=0)
        self.wf = O.to_f32(self.w)
        self.d = Diffuser(ctx, TINY, self.w)
        g = gen(1)
        self.x = torch.randn(3, 4, 16, 16, generator=g)
        self.c = h16f(torch.randn(3, 7, TINY.context_dim, generator=g))
        self.y = h16f(torch.randn(3, TINY.adm_in_channels, generator=g))
        self.noise = torch.randn(2, 4, 16, 16, generator=gen(0))
        self.cond = Conditioning(**tiny_conditioning(refiner=True))
        self.oc = O.OracleConditioning(**tiny_conditioning(refiner=True))
        self.alphas = sdxl_b200.alphas_cumprod(TINY.n_steps)
        self.a64 = np.array([O.get_alpha(self.alphas, i) for i in range(TINY.n_steps)])


@pytest.fixture(scope="module")
def S(ctx):
    s = Setup(ctx)
    yield s
    s.d.close()


@pytest.fixture(autouse=True)
def detach(S):
    yield
    S.d.set_deepcache(None)
    S.d.set_controls([])
    S.d.set_pag(None)
    S.d.set_freeu(None)


def _fwd(d, x, c, y, cached=None, t=T, perturbed_rows=None):
    return d.unet_forward(x, [t], c, y, perturbed_rows=perturbed_rows, cached=cached).cpu()


def _equal(got, want, what):
    assert torch.equal(got, want), f"{what}: {first_difference(want, got)}"


# ---- 1. interval 1 and detaching are the plain calls -------------------------------------------------------------------------------
SAMPLE_CASES = ["ddim", "inpainting", "pag"] + [f"{s}/{m}" for s in SAMPLERS for m in ("cfg", "no_cfg")]


def _sample(S, case):
    if case == "ddim":
        return S.d.sample_latent(S.cond, 7.5, 4, noise=S.noise).cpu()
    if case == "pag":
        return S.d.sample_latent(S.cond, 7.5, 4, noise=S.noise, schedule=Schedule("dpmpp_2m", "karras", 4)).cpu()
    if case == "inpainting":
        mask = torch.zeros(2, 4, 16, 16, dtype=torch.bool)
        mask[:, :, :6] = True
        ref = torch.randn(2, 4, 16, 16, generator=gen(3))
        return S.d.sample_latent_with_inpainting(S.cond, 7.5, 4, ref, mask, init_noise=S.noise, seed=4).cpu()
    sampler, mode = case.split("/")
    sch = Schedule(sampler, "karras" if sampler != "lcm" else "lcm", 4, no_cfg=mode == "no_cfg")
    return S.d.sample_latent(S.cond, 7.5, 4, noise=S.noise, seed=5, schedule=sch).cpu()


@pytest.mark.parametrize("case", SAMPLE_CASES)
def test_interval_1_and_detach_are_bit_identical(S, case):
    if case == "pag":
        S.d.set_pag("mid", 3.0)
    plain = _sample(S, case)
    S.d.set_deepcache(1, 4)
    _equal(_sample(S, case), plain, f"{case}, interval 1")
    S.d.set_deepcache(3, 4)
    moved = _sample(S, case)
    S.d.set_deepcache(None)
    _equal(_sample(S, case), plain, f"{case}, detached")
    assert not torch.equal(moved, plain)


def test_interval_1_inpainting_unet_and_refiner(ctx):
    w = synth_weights(TINY_INPAINT, seed=0)
    d = Diffuser(ctx, TINY_INPAINT, w)
    d.set_inpaint_condition(torch.rand(1, 5, 16, 16, generator=gen(6)))
    cond, noise = Conditioning(**tiny_conditioning(refiner=True)), torch.randn(2, 4, 16, 16, generator=gen(0))
    plain = d.sample_latent(cond, 7.5, 4, noise=noise).cpu()
    d.set_deepcache(1, 2)
    _equal(d.sample_latent(cond, 7.5, 4, noise=noise).cpu(), plain, "inpainting UNet, interval 1")
    d.set_deepcache(None)
    _equal(d.sample_latent(cond, 7.5, 4, noise=noise).cpu(), plain, "inpainting UNet, detached")
    d.close()
    r = Diffuser(ctx, TINY_REFINER, synth_weights(TINY_REFINER, seed=1))
    latent, rn = torch.randn(2, 4, 16, 16, generator=gen(5)), torch.randn(2, 4, 16, 16, generator=gen(7))
    plain = r.refine_latent(latent, cond, 7.5, 800, 50, noise=rn).cpu()
    r.set_deepcache(1, 6)
    _equal(r.refine_latent(latent, cond, 7.5, 800, 50, noise=rn).cpu(), plain, "refiner, interval 1")
    r.set_deepcache(None)
    _equal(r.refine_latent(latent, cond, 7.5, 800, 50, noise=rn).cpu(), plain, "refiner, detached")
    r.close()


# ---- 2. a full forward with DeepCache attached is the plain forward ------------------------------------------------------------------
def test_full_forward_is_the_plain_forward(S):
    S.d.set_freeu(*FV)
    plain = _fwd(S.d, S.x[:2], S.c[:2], S.y[:2])
    n_ops = S.d.plan_num_ops
    for b in range(N_BRANCH):
        S.d.set_deepcache(3, b)
        _equal(_fwd(S.d, S.x[:2], S.c[:2], S.y[:2], cached=False), plain, f"branch {b}")
        assert S.d.plan_num_ops == n_ops + (b >= 3)   # output block 8 - b is a FreeU block: the copy of the feature it scales


# ---- 3. cached right after full, same inputs, is the full output bit for bit ----------------------------------------------------------
ATTACHMENTS = ["none", "controlnet", "t2i", "image_prompt", "ip_masked", "pag", "freeu", "inpainting", "refiner", "refiner_freeu"]


def _attached(S, ctx, kind):
    """(diffuser, x, c, y, perturbed_rows, closers) with the attachment on."""
    x, c, y, rows, closers = S.x[:2], S.c[:2], S.y[:2], None, []
    d = S.d
    if kind == "controlnet":
        net = ControlNet(ctx, TINY_CONTROLNET, synth_weights(TINY_CONTROLNET, seed=7))
        d.set_controls([(net, torch.rand(1, 3, 128, 128, generator=gen(4)), 0.8)])
        closers = [lambda: d.set_controls([]), net.close]
    elif kind == "t2i":
        ad = T2IAdapter(ctx, TINY_T2I_ADAPTER, synth_weights(TINY_T2I_ADAPTER, seed=1))
        d.set_t2i_adapters([(ad, torch.rand(1, 3, 128, 128, generator=gen(2)), 1.5)])
        closers = [lambda: d.set_t2i_adapters([]), ad.close]
    elif kind in ("image_prompt", "ip_masked"):
        ad = IPAdapter(ctx, TINY, 32, synth_ip_adapter(TINY, 32, seed=3))
        if kind == "image_prompt":
            d.set_image_prompt(ad, torch.randn(1, 1, 32, generator=gen(2)), 0.8)
        else:
            mask = torch.zeros(2, 128, 128)
            mask[0, :, :64], mask[1, :, 64:] = 1, 1
            two = torch.randn(1, 2, 32, generator=gen(4))
            d.set_image_prompts([(ad, two, 0.8, None, mask), (ad, two.flip(1), 0.5, None, mask.flip(0))])
        closers = [lambda: d.set_image_prompts([]), ad.close]
    elif kind == "pag":
        d.set_pag(".*", 3.0)
        x, c, y, rows = S.x, S.c, S.y, 1
    elif kind == "freeu":
        d.set_freeu(*FV)
    elif kind == "inpainting":
        d = Diffuser(ctx, TINY_INPAINT, synth_weights(TINY_INPAINT, seed=0))
        d.set_inpaint_condition(torch.rand(1, 5, 16, 16, generator=gen(6)))
        closers = [d.close]
    elif kind.startswith("refiner"):
        d = Diffuser(ctx, TINY_REFINER, synth_weights(TINY_REFINER, seed=1))
        g = gen(5)
        x, c, y = torch.randn(2, 4, 8, 16, generator=g), h16f(torch.randn(2, 6, 40, generator=g)), h16f(torch.randn(2, 16, generator=g))
        if kind == "refiner_freeu":
            d.set_freeu(*FV)
        closers = [d.close]
    return d, x, c, y, rows, closers


@pytest.mark.parametrize("kind", ATTACHMENTS)
def test_cached_after_full_is_the_full_forward(S, ctx, kind):
    d, x, c, y, rows, closers = _attached(S, ctx, kind)
    try:
        for b in range(N_BRANCH):
            d.set_deepcache(2, b)
            full = _fwd(d, x, c, y, cached=False, perturbed_rows=rows)
            _equal(_fwd(d, x, c, y, cached=True, perturbed_rows=rows), full, f"{kind}, branch {b}, cached")
            if "freeu" in kind and b >= 3:   # FreeU scales the block's input in place: the feature must not compound
                _equal(_fwd(d, x, c, y, cached=True, perturbed_rows=rows), full, f"{kind}, branch {b}, second cached")
            assert not torch.equal(_fwd(d, x * 0.5, c, y, cached=True, perturbed_rows=rows), full)
    finally:
        d.set_deepcache(None)
        for f in closers:
            f()


# ---- 4. cached forwards at new inputs against the oracle ----------------------------------------------------------------------------
@pytest.mark.parametrize("b", [0, 3])
@pytest.mark.parametrize("control", [False, True], ids=["plain", "controlnet"])
def test_cached_forward_vs_oracle(S, ctx, b, control):
    att, net = O.NOTHING, None
    if control:
        wc = synth_weights(TINY_CONTROLNET, seed=7)
        net = ControlNet(ctx, TINY_CONTROLNET, wc)
        hint = torch.rand(1, 3, 128, 128, generator=gen(4))
        S.d.set_controls([(net, hint, 0.8)])
        att = O.Attach(controls=[(TINY_CONTROLNET, O.to_f32(wc), hint, 0.8)])
    S.d.set_deepcache(3, b)
    x0, c, y = S.x[:2], S.c[:2], S.y[:2]
    x1 = x0 + 0.3 * torch.randn(2, 4, 16, 16, generator=gen(9))
    _fwd(S.d, x0, c, y, cached=False, t=T)
    got = _fwd(S.d, x1, c, y, cached=True, t=T - 40)
    if net:
        S.d.set_controls([])
        net.close()
    _, feature = DO.unet_forward(TINY, S.wf, x0, torch.tensor([T]), c, y, att, b)
    ref, _ = DO.unet_forward(TINY, S.wf, x1, torch.tensor([T - 40]), c, y, att, b, feature)
    full = O.unet_forward(TINY, S.wf, x1, torch.tensor([T - 40]), c, y, att)
    e = rel_err(got, ref)
    print(f"cached forward, branch {b}{' + ControlNet' if control else ''}: rel err vs oracle {e:.2e}; "
          f"the cached oracle is {rel_err(ref, full):.2e} from the full one")
    assert e <= FWD_TOL


# ---- 5. interval-3 samples against the oracle chains -----------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["ddim", "dpmpp_2m", "dpmpp_2m_pag", "dpmpp_2m_controlnet"])
def test_interval_3_sample_vs_oracle(S, ctx, case):
    b, att, net = 2, O.NOTHING, None
    if case == "dpmpp_2m_pag":
        S.d.set_pag("mid", 3.0)
        att = PO.attach(TINY, PO.paths_of_mask(TINY, pag_layer_mask(TINY, "mid")), 3.0)
    if case == "dpmpp_2m_controlnet":
        wc = synth_weights(TINY_CONTROLNET, seed=7)
        net = ControlNet(ctx, TINY_CONTROLNET, wc)
        hint = torch.rand(1, 3, 128, 128, generator=gen(4))
        S.d.set_controls([(net, hint, 0.8)])
        att = O.Attach(controls=[(TINY_CONTROLNET, O.to_f32(wc), hint, 0.8)])
    S.d.set_deepcache(3, b)
    if case == "ddim":
        got = S.d.sample_latent(S.cond, 7.5, 5, noise=S.noise).cpu()
        ref = DO.sample_latent(TINY, S.wf, S.alphas, S.noise, S.oc, 7.5, 5, 3, b, att)
        plain = O.sample_latent(TINY, S.wf, S.alphas, S.noise, S.oc, 7.5, 5, att=att)
    else:
        sch = Schedule("dpmpp_2m", "karras", 5)
        got = S.d.sample_latent(S.cond, 7.5, 5, noise=S.noise, schedule=sch).cpu()
        t, sig = SO.schedule("karras", 5, S.a64)
        x = S.noise * (sig[0] ** 2 + 1) ** 0.5
        ref = SO.sample(DO.eps_fn(TINY, S.wf, S.oc, 7.5, 3, b, att), "dpmpp_2m", t, sig, x, None, 0, None, 1.0, 1.0, None, torch.where)
        plain = SO.sample(DO.eps_fn(TINY, S.wf, S.oc, 7.5, 1, b, att), "dpmpp_2m", t, sig, x, None, 0, None, 1.0, 1.0, None, torch.where)
    if net:
        S.d.set_controls([])
        net.close()
    e = rel_err(got, ref)
    print(f"interval-3 {case}: rel err vs oracle {e:.2e}; DeepCache moves the oracle by {rel_err(ref, plain):.2e}")
    assert e <= SAMPLE_TOL


def test_interval_3_refine_vs_oracle(ctx):
    w = synth_weights(TINY_REFINER, seed=1)
    d = Diffuser(ctx, TINY_REFINER, w)
    g = gen(5)
    latent, noise = torch.randn(2, 4, 8, 16, generator=g), torch.randn(2, 4, 8, 16, generator=g)
    c = tiny_conditioning(2, 6, (64, 128), refiner=True)
    d.set_deepcache(3, 4)
    got = d.refine_latent(latent, Conditioning(**c), 7.5, 800, 50, noise=noise).cpu()
    d.close()
    ref = DO.refine_latent(TINY_REFINER, O.to_f32(w), sdxl_b200.alphas_cumprod(), latent, O.OracleConditioning(**c), 7.5, 800, 50,
                           noise, 3, 4)
    e = rel_err(got, ref)
    print(f"interval-3 TINY_REFINER refine: rel err vs oracle {e:.2e}")
    assert e <= SAMPLE_TOL


# ---- 6. the sampler counts from sampler_begin ----------------------------------------------------------------------------------------
def test_hand_driven_steps_are_sample_latent(S):
    S.d.set_deepcache(2, 1)
    want = S.d.sample_latent(S.cond, 7.5, 5, noise=S.noise).cpu()
    for _ in range(2):   # the second begin restarts the count
        S.d.sampler_begin(S.cond, 7.5)
        S.d.sampler_set_latent(S.noise)
        ts = list(range(999, -1, -200))
        for t in ts:
            S.d.sampler_step(t, t - 200 if t >= 200 else -1)
        _equal(S.d.sampler_get_latent(S.noise).cpu(), want, "hand-driven loop")
    host = S.noise.clone()
    S.d.sampler_begin(S.cond, 7.5)
    for t in ts:
        S.d.sampler_step_host(t, t - 200 if t >= 200 else -1, host)
    _equal(host, want, "hand-driven host loop")


# ---- 7. plan builds --------------------------------------------------------------------------------------------------------------------
def test_plan_builds(S):
    fwd = lambda cached=None: _fwd(S.d, S.x[:2], S.c[:2], S.y[:2], cached=cached)   # noqa: E731
    fwd()
    n = plan_builds(S.d)
    S.d.set_deepcache(2, 1)                     # attach: one rebuild
    fwd(False)
    assert plan_builds(S.d) == n + 1
    S.d.set_deepcache(5, 1)                     # interval only: kept, and so is the feature
    fwd(True)
    S.d.sample_latent(S.cond, 7.5, 3, noise=S.noise)
    fwd(False)
    assert plan_builds(S.d) == n + 3            # the sampler's batch of 4 rows, then back to 2
    S.d.set_deepcache(5, 2)                     # a new branch: one rebuild
    fwd(False)
    assert plan_builds(S.d) == n + 4
    S.d.set_deepcache(None)                     # detach: one rebuild
    fwd()
    assert plan_builds(S.d) == n + 5


# ---- 8. refusals -----------------------------------------------------------------------------------------------------------------------
def _set(S, interval, branch, cached=0):
    s = _lib.Deepcache()
    s.interval, s.branch, s.forward_cached = interval, branch, cached
    return S.ctx.lib.sdxl_unet_set_deepcache(S.d.h, C.byref(s))


def test_refusals_leave_the_previous_state(S):
    S.d.set_deepcache(2, 3)
    full = _fwd(S.d, S.x[:2], S.c[:2], S.y[:2], cached=False)
    n = plan_builds(S.d)
    for (interval, branch, cached), field in (((0, 3, 0), "interval"), ((-2, 3, 0), "interval"), ((2, -1, 0), "branch"),
                                              ((2, N_BRANCH, 0), "branch"), ((2, 3, 2), "forward_cached")):
        assert _set(S, interval, branch, cached) != 0
        assert field in S.ctx.lib.sdxl_last_error(S.ctx.h).decode()
        _equal(_fwd(S.d, S.x[:2], S.c[:2], S.y[:2], cached=True), full, f"after refusing {field}")
        assert plan_builds(S.d) == n
    # a cached forward before any full forward of the plan, and after a rebuild, is refused and keeps the previous state
    S.d.set_deepcache(2, 4)
    with pytest.raises(SdxlError, match="DeepCache"):
        _fwd(S.d, S.x[:2], S.c[:2], S.y[:2], cached=True)
    full = _fwd(S.d, S.x[:2], S.c[:2], S.y[:2], cached=False)
    _equal(_fwd(S.d, S.x[:2], S.c[:2], S.y[:2], cached=True), full, "after the refusal")
    with pytest.raises(SdxlError, match="DeepCache"):
        _fwd(S.d, S.x[:1], S.c[:1], S.y[:1], cached=True)    # another batch: a rebuilt plan
    with pytest.raises(SdxlError, match="set_deepcache"):
        S.d.set_deepcache(None)
        _fwd(S.d, S.x[:2], S.c[:2], S.y[:2], cached=True)


def test_sampler_needs_a_new_begin_after_attach(S):
    s, keep = S.cond.to_struct(S.ctx.device)
    lib = S.ctx.lib
    assert lib.sdxl_sampler_begin(S.d.h, C.byref(s), C.c_double(7.5)) == 0
    S.d.set_deepcache(3, 0)
    assert lib.sdxl_sampler_step(S.d.h, 999, 749) != 0
    assert "sampler_begin" in lib.sdxl_last_error(S.ctx.h).decode()
    torch.cuda.synchronize()


# ---- pipeline ----------------------------------------------------------------------------------------------------------------------
def test_pipeline_deepcache_attaches_for_the_call(ctx):
    from sdxl_b200 import TINY_CLIP, TINY_OPEN_CLIP, TINY_VAE, ClipTextEncoder, Embedder, LatentDecoder, OpenClipTokenizer, UNetConfig
    from sdxl_b200.pipeline import sample
    mini = os.path.join(os.path.dirname(__file__), "golden", "mini_bpe")
    ca, cb = TINY_CLIP, TINY_OPEN_CLIP
    ucfg = UNetConfig(adm_in_channels=cb.embed_dim + 6 * 256, model_channels=64, channel_mults=(1, 2, 4), transformer_depths=(0, 1, 1),
                      context_dim=ca.n_state + cb.n_state)
    tok = OpenClipTokenizer(os.path.join(mini, "mini_merges.txt"), os.path.join(mini, "mini_vocab.txt"))
    emb = Embedder(ctx, ClipTextEncoder(ctx, ca, synth_weights(ca, seed=1)), ClipTextEncoder(ctx, cb, synth_weights(cb, seed=2)), tok, tok)
    dif = Diffuser(ctx, ucfg, synth_weights(ucfg, seed=3))
    vae = LatentDecoder(ctx, TINY_VAE, synth_weights(TINY_VAE, seed=0))
    kw = dict(guidance=5.0, n_steps=4, resolution=(64, 64), seed=0)
    plain = sample(emb, dif, vae, "a photo of a cat", **kw)
    with_dc = sample(emb, dif, vae, "a photo of a cat", deepcache=(3, 1), **kw)
    dif.set_deepcache(3, 1)
    same = sample(emb, dif, vae, "a photo of a cat", **kw)
    dif.set_deepcache(None)
    assert torch.equal(with_dc, same) and not torch.equal(with_dc, plain)
    assert torch.equal(sample(emb, dif, vae, "a photo of a cat", **kw), plain)   # detached after the call
    both = sample(emb, dif, vae, "a photo of a cat", deepcache=(3, 1), freeu=FV, sampler="dpmpp_2m", spacing="karras", **kw)
    assert both.shape == plain.shape
    assert torch.equal(sample(emb, dif, vae, "a photo of a cat", **kw), plain)
    dif.close()


# ---- 9. fresh-memory fills, graphs and PDL ---------------------------------------------------------------------------------------------
WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "deepcache_invariance_worker.py")
SWITCHES = ("SDXL_B200_FILL", "SDXL_B200_NO_GRAPH", "SDXL_B200_NO_PDL")
CONFIGS = {"base": {}, "nan": {"SDXL_B200_FILL": "0xff"}, "big": {"SDXL_B200_FILL": "0x7b"}, "eager": {"SDXL_B200_NO_GRAPH": "1"},
           "nopdl": {"SDXL_B200_NO_PDL": "1"}}


def _run_worker(name, out_dir):
    env = {k: v for k, v in os.environ.items() if k not in SWITCHES}
    env.update(CONFIGS[name])
    out = os.path.join(out_dir, f"{name}.pt")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [WORKER, out]
    p = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, f"worker [{name}] exited with {p.returncode}:\n{p.stderr[-6000:]}"
    return torch.load(out, weights_only=True)


def test_fills_graphs_and_pdl_change_nothing(tmp_path):
    base = _run_worker("base", str(tmp_path))
    assert all(bool(torch.isfinite(v).all()) for v in base.values())
    for name in ("nan", "big", "eager", "nopdl"):
        got = _run_worker(name, str(tmp_path))
        assert got.keys() == base.keys()
        for k in base:
            assert torch.equal(got[k], base[k]), f"[{name}] {k}: {first_difference(base[k], got[k])}"
