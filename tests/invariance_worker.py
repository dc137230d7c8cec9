"""One fixed list of engine workloads, every output saved to the file given on the command line (tests/test_workspace_invariance_gpu.py
runs it once per configuration and compares the files bit for bit).

Each call is made three times in a row: the first runs its plan eagerly, the second captures the CUDA graph and the third replays
it. Run 1 is saved; both must be finite and run 3 must equal run 1, so that a comparison with SDXL_B200_NO_GRAPH=1 compares the
graph against eager launches; the outputs are saved before the process exits with 1 if any of these fails. Every workload that
samples gets a model of its own, so the sampler's and the plan's buffers are fresh in run 1.

    python invariance_worker.py OUT.pt [--torch-nan]

--torch-nan: torch fills the memory of every tensor it allocates with NaN (torch.utils.deterministic.fill_uninitialized_memory),
so an output element the library does not write shows up as NaN. The library's own memory is filled by SDXL_B200_FILL."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, os.path.join(ROOT, "stable-diffusion-xl-burn_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import sdxl_b200  # noqa: E402
from sdxl_b200 import (SDXL_BASE, SDXL_VAE, TINY, TINY_CLIP, TINY_CONTROLNET, TINY_INPAINT, TINY_OPEN_CLIP, TINY_REFINER,  # noqa: E402
                       TINY_T2I_ADAPTER, TINY_VAE, ClipTextEncoder, Conditioning, ControlNet, Diffuser, Embedder, IPAdapter,
                       LatentDecoder, OpenClipTokenizer, T2IAdapter, synth_weights)
from sdxl_b200.clip_vision import TINY_VIT_80, ClipVisionEncoder, synth_vision_weights  # noqa: E402
from sdxl_b200.ip_adapter import ResamplerConfig, synth_ip_adapter  # noqa: E402
from sdxl_b200.schedulers import Schedule  # noqa: E402
import freeu_oracle as FO  # noqa: E402
from harness import arb, first_difference, h16f, tiny_conditioning  # noqa: E402
from lora_cases import layer_paths, make_adapter  # noqa: E402

T = 499
X = arb(2, 4, 16, 16)                       # a 128 x 128 pixel latent, the size of tiny_conditioning()
C_CTX = h16f(arb(2, 7, TINY.context_dim))
Y = h16f(arb(2, TINY.adm_in_channels))


def gen(seed):
    return torch.Generator().manual_seed(seed)


class Recorder:
    def __init__(self):
        self.out = {}
        self.problems = []

    def thrice(self, name, fn):
        """Runs fn three times (eager, capture, replay); keeps run 1 and checks that run 3 equals it. fn returns a tensor or a
        dict of them; every tensor is recorded as name/key."""
        runs = [fn() for _ in range(3)]
        torch.cuda.synchronize()
        one, three = (r if isinstance(r, dict) else {"": r} for r in (runs[0], runs[2]))
        for k, v in one.items():
            key = name if k == "" else f"{name}/{k}"
            v = v.detach().cpu().clone()
            w = three[k].detach().cpu()
            bad1, bad3 = (~torch.isfinite(t) if t.is_floating_point() else torch.zeros_like(t, dtype=torch.bool) for t in (v, w))
            if bad1.any() or bad3.any():
                first = tuple(int(i) for i in (bad1 | bad3).nonzero()[0])
                self.problems.append(f"{key}: non-finite values, {int(bad1.sum())} of {v.numel()} in run 1 (eager) and {int(bad3.sum())} in "
                                     f"run 3 (graph replay), the first at {first}")
            elif not torch.equal(v, w):
                self.problems.append(f"{key}: run 3 (graph replay) differs from run 1 (eager): {first_difference(v, w)}")
            self.out[key] = v


# ---- workloads -----------------------------------------------------------------------------------------------------------------
def unet_forwards(R, ctx, w):
    d = Diffuser(ctx, TINY, w)
    # the shapes of test_unet_gpu.test_unet_forward_vs_oracle: (2, 16, 16) is the CFG batch; (1, 12, 20) has ragged rows
    for B, h, wd, n_ctx, t in [(1, 8, 8, 3, 1), (2, 16, 16, 77, 999), (1, 32, 32, 77, 500), (3, 8, 16, 5, 249), (1, 12, 20, 7, 700)]:
        x, c, y = arb(B, 4, h, wd), h16f(arb(B, n_ctx, TINY.context_dim)), h16f(arb(B, TINY.adm_in_channels))
        d.set_conditioning(c, y)
        R.thrice(f"unet/{B}x{h}x{wd}", lambda: d.unet_forward(x, [t]))
        R.thrice(f"unet/{B}x{h}x{wd}/f16", lambda: d.unet_forward(x.half(), [t]))
    d.close()


SCHEDULES = {
    "euler": Schedule("euler", "karras", 4),
    "euler_ancestral": Schedule("euler_ancestral", "karras", 4),
    "dpmpp_2m": Schedule("dpmpp_2m", "karras", 4),
    "lcm": Schedule("lcm", "lcm", 4),
    "euler_no_cfg": Schedule("euler", "trailing", 4, no_cfg=True),
    "dpmpp_2m_no_cfg": Schedule("dpmpp_2m", "karras", 4, no_cfg=True),
}


def samplers(R, ctx, w):
    cond = Conditioning(**tiny_conditioning(refiner=True))
    noise = torch.randn(2, 4, 16, 16, generator=gen(0))
    d = Diffuser(ctx, TINY, w)
    R.thrice("sample/ddim_cfg", lambda: d.sample_latent(cond, 7.5, 4, noise=noise))
    d.close()
    d = Diffuser(ctx, TINY, w)
    R.thrice("sample/ddim_guidance1", lambda: d.sample_latent(cond, 1.0, 4, seed=3))
    d.close()
    for name, sch in SCHEDULES.items():
        d = Diffuser(ctx, TINY, w)   # fresh sampler buffers: run 1 reads whatever its arena holds where it reads unwritten memory
        R.thrice(f"sample/{name}", lambda: d.sample_latent(cond, 7.5, 4, seed=11, schedule=sch))
        d.close()


def inpainting_and_refiner(R, ctx, w):
    cond = Conditioning(**tiny_conditioning(1, 5, refiner=True))
    g = gen(3)
    noise0, step_noise, ref_lat = torch.randn(1, 4, 16, 16, generator=g), torch.randn(10, 1, 4, 16, 16, generator=g), \
        torch.randn(1, 4, 16, 16, generator=g)
    mask = torch.zeros(1, 4, 16, 16, dtype=torch.bool)
    mask[:, :, :5, :] = True
    d = Diffuser(ctx, TINY, w)
    R.thrice("inpainting/ddim", lambda: d.sample_latent_with_inpainting(cond, 7.5, 10, ref_lat, mask, init_noise=noise0,
                                                                       step_noise=step_noise))
    d.close()
    d = Diffuser(ctx, TINY, w)
    R.thrice("inpainting/euler_ancestral", lambda: d.sample_latent_with_inpainting(cond, 7.5, 4, ref_lat, mask, seed=5,
                                                                                  schedule=Schedule("euler_ancestral", "trailing", 4)))
    d.close()

    d = Diffuser(ctx, TINY_REFINER, synth_weights(TINY_REFINER, seed=1))
    rc = Conditioning(**tiny_conditioning(2, 6, (64, 128), refiner=True))
    g = gen(5)
    latent, noise = torch.randn(2, 4, 8, 16, generator=g), torch.randn(2, 4, 8, 16, generator=g)
    R.thrice("refiner/refine_latent", lambda: d.refine_latent(latent, rc, 7.5, 800, 50, noise=noise))
    d.close()

    wi = synth_weights(TINY_INPAINT, seed=0)
    g = gen(10)
    ic = torch.cat([(torch.rand(2, 1, 16, 16, generator=g) > 0.5).float(), torch.randn(2, 4, 16, 16, generator=g)], dim=1)
    d = Diffuser(ctx, TINY_INPAINT, wi)
    d.set_inpaint_condition(ic)
    d.set_conditioning(C_CTX, Y)
    R.thrice("inpaint_unet/forward", lambda: d.unet_forward(X, [T]))
    d.close()
    d = Diffuser(ctx, TINY_INPAINT, wi)
    d.set_inpaint_condition(ic[:1])
    R.thrice("inpaint_unet/sample", lambda: d.sample_latent(Conditioning(**tiny_conditioning()), 7.5, 4, seed=2))
    d.close()


def attachments(R, ctx, w):
    def forward_with(name, attach, detach, models=()):
        d = Diffuser(ctx, TINY, w)
        attach(d)
        d.set_conditioning(C_CTX, Y)
        R.thrice(f"{name}/forward", lambda: d.unet_forward(X, [T]))
        detach(d)
        d.close()
        d = Diffuser(ctx, TINY, w)
        attach(d)
        R.thrice(f"{name}/sample", lambda: d.sample_latent(Conditioning(**tiny_conditioning()), 7.5, 4, seed=9))
        d.close()
        for m in models:
            m.close()

    net = ControlNet(ctx, TINY_CONTROLNET, synth_weights(TINY_CONTROLNET, seed=1))
    hint = torch.rand(2, 3, 128, 128, generator=gen(2))
    R.thrice("controlnet/hint_embedding", lambda: net.embed_hint(hint))
    forward_with("controlnet", lambda d: d.set_controls([(net, hint, 1.0)]), lambda d: d.set_controls([]), [net])

    D = 32
    ip = IPAdapter(ctx, TINY, D, synth_ip_adapter(TINY, D, seed=3))
    emb = torch.randn(2, D, generator=gen(4))
    R.thrice("ip_adapter/project", lambda: ip.project(emb))
    forward_with("ip_adapter", lambda d: d.set_image_prompt(ip, emb, 0.8, negative=torch.zeros_like(emb)),
                 lambda d: d.set_image_prompt(None))

    Dp, Lp = 40, 19
    plus = IPAdapter(ctx, TINY, Dp, synth_ip_adapter(TINY, Dp, seed=5, resampler=ResamplerConfig(depth=2, heads=2, tokens=16)))
    h = torch.randn(1, 2, Lp, Dp, generator=gen(7))
    R.thrice("ip_adapter_plus/resample", lambda: plus.resample(h[:, 0]))
    forward_with("ip_adapter_plus", lambda d: d.set_image_prompt(plus, h, 0.9, negative=torch.randn(1, 2, Lp, Dp, generator=gen(8)) * 0.5),
                 lambda d: d.set_image_prompt(None), [plus])

    mask = torch.zeros(2, 128, 128)
    mask[0, :, :64], mask[1, :, 64:] = 1, 1
    two = torch.randn(1, 2, D, generator=gen(4))
    forward_with("ip_masked", lambda d: d.set_image_prompts([(ip, two, 0.8, None, mask), (ip, two.flip(1), 0.5, None, mask.flip(0))]),
                 lambda d: d.set_image_prompts([]), [ip])

    t2i = T2IAdapter(ctx, TINY_T2I_ADAPTER, synth_weights(TINY_T2I_ADAPTER, seed=1))
    th = torch.rand(1, 3, 128, 128, generator=gen(2))
    R.thrice("t2i_adapter/features", lambda: dict(enumerate(t2i.features(th))))
    forward_with("t2i_adapter", lambda d: d.set_t2i_adapters([(t2i, th, 1.0)]), lambda d: d.set_t2i_adapters([]), [t2i])

    d = Diffuser(ctx, TINY, w)
    d.set_pag("mid", 3.0)
    R.thrice("pag/sample", lambda: d.sample_latent(Conditioning(**tiny_conditioning()), 7.5, 4, seed=9,
                                                   schedule=Schedule("euler", "trailing", 4)))
    d.set_conditioning(h16f(arb(3, 7, TINY.context_dim)), h16f(arb(3, TINY.adm_in_channels)))
    R.thrice("pag/forward", lambda: d.unet_forward(arb(3, 4, 16, 16), [T], perturbed_rows=1))
    d.close()

    forward_with("freeu", lambda d: d.set_freeu(*FO.RECOMMENDED_SDXL), lambda d: d.set_freeu(None))

    d = Diffuser(ctx, TINY, w)
    d.set_conditioning(C_CTX, Y)
    R.thrice("lora/unmerged", lambda: d.unet_forward(X, [T]))
    d.set_adapters([(make_adapter(TINY, layer_paths(TINY), rank=4, seed=1), 0.5)])
    R.thrice("lora/merged", lambda: d.unet_forward(X, [T]))
    d.set_adapters([])
    R.thrice("lora/restored", lambda: d.unet_forward(X, [T]))
    d.close()
    if not torch.equal(R.out["lora/restored"], R.out["lora/unmerged"]):
        R.problems.append("lora/restored: the forward after set_adapters([]) differs from the unmerged one: "
                          + first_difference(R.out["lora/unmerged"], R.out["lora/restored"]))


def vae_and_encoders(R, ctx):
    vae = LatentDecoder(ctx, TINY_VAE, synth_weights(TINY_VAE, seed=0))
    lat = torch.randn(2, 4, 8, 16, generator=gen(1))
    R.thrice("vae/decode", lambda: vae.decode_latent(lat.cuda()))
    img = torch.rand(2, 3, 64, 128, generator=gen(2)) * 2 - 1
    R.thrice("vae/encode", lambda: vae.encode_image(img.cuda()))
    vae.close()

    mini = os.path.join(HERE, "golden", "mini_bpe")
    tok = OpenClipTokenizer(os.path.join(mini, "mini_merges.txt"), os.path.join(mini, "mini_vocab.txt"))
    e1 = ClipTextEncoder(ctx, TINY_CLIP, synth_weights(TINY_CLIP, seed=1))
    e2 = ClipTextEncoder(ctx, TINY_OPEN_CLIP, synth_weights(TINY_OPEN_CLIP, seed=2))
    emb = Embedder(ctx, e1, e2, tok, tok)

    def text():
        c = emb.text_to_conditioning("a photo of a cat", (64, 64), (0, 0), (64, 64))
        return {f: getattr(c, f) for f in c._fields() if getattr(c, f) is not None}
    R.thrice("text_to_conditioning", text)
    e1.close()
    e2.close()

    enc = ClipVisionEncoder(ctx, TINY_VIT_80, synth_vision_weights(TINY_VIT_80, seed=1))
    px = torch.randn(3, 3, TINY_VIT_80.image_size, TINY_VIT_80.image_size, generator=gen(6))
    R.thrice("clip_vision/embeds", lambda: enc.encode(px))
    R.thrice("clip_vision/hidden", lambda: enc.encode_hidden(px))
    R.thrice("clip_vision/hidden_1", lambda: enc.encode_hidden(px, 1))
    enc.close()


def fullsize(R, ctx):
    """SDXL base at 832 x 1216: levels 104 x 152, 52 x 76 and 26 x 38 leave ragged pixel tiles in every GEMM and attention."""
    w = sdxl_b200.synth_weights(SDXL_BASE, seed=0, device=str(ctx.device))
    d = Diffuser(ctx, SDXL_BASE, sdxl_b200.build_pack(w))
    del w
    g = gen(1)
    x = torch.randn(2, 4, 104, 152, generator=g)
    x[1] = x[0]
    d.set_conditioning(torch.randn(2, 77, 2048, generator=g).half(), torch.randn(2, 2816, generator=g).half())
    R.thrice("sdxl_base/832x1216", lambda: d.unet_forward(x, [999]))
    d.close()
    wv = synth_weights(SDXL_VAE, seed=7, device=str(ctx.device))
    vae = LatentDecoder(ctx, SDXL_VAE, sdxl_b200.build_pack(wv))
    del wv
    lat = torch.randn(1, 4, 104, 152, generator=gen(2))
    R.thrice("sdxl_vae/decode_104x152", lambda: vae.decode_latent(lat.cuda()))
    vae.close()


def main():
    out_path = sys.argv[1]
    if "--torch-nan" in sys.argv[2:]:
        torch.use_deterministic_algorithms(True, warn_only=True)
        torch.utils.deterministic.fill_uninitialized_memory = True
    ctx = sdxl_b200.Context(0)
    R = Recorder()
    w = synth_weights(TINY, seed=0)
    unet_forwards(R, ctx, w)
    samplers(R, ctx, w)
    inpainting_and_refiner(R, ctx, w)
    attachments(R, ctx, w)
    vae_and_encoders(R, ctx)
    fullsize(R, ctx)
    ctx.synchronize()
    torch.save({"outputs": R.out, "fill": int(ctx.lib.sdxl_debug_fill()), "problems": R.problems}, out_path)
    ctx.close()
    for p in R.problems:
        print(p, file=sys.stderr)
    sys.exit(1 if R.problems else 0)


if __name__ == "__main__":
    main()
