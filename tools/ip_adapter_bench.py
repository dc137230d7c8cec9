#!/usr/bin/env python
"""Sampler step time without an image prompt, with the base adapter's 1 image (4 tokens) and 4 images (16 tokens), and with an
IP-Adapter Plus prompt of 1 image (16 tokens) and 4 images (64 tokens), with image-prompt sets (DESIGN.md §13: base 1 image plus
Plus 1 image, unmasked and each masked to one half; one base prompt of 2 images masked to the two halves), the attention kernel's
share of a step, the set_image_prompt and set_image_prompts time (base: projection; Plus: Resampler) and the vision encoder's time per image (ViT-H/14 image_embeds and hidden states,
ViT-bigG/14 image_embeds); SDXL base + ViT-H-sized base and Plus IP-Adapters (synthetic weights) on one GPU.

    python tools/ip_adapter_bench.py [out.json] [--steps K] [--warmup W] [--reps R]

Step time: bench.py's method (sampler_begin, W warm-up steps, CUDA events around K sampler steps, CFG 7.5 at 1024^2, batch 1),
with no prompt and the four prompts alternated R times in one process; the order rotates from one alternation to the next, so a
clock that drifts during the run does not always fall on the same configuration. Attention share: profile_plan of one step (CUDA events per
launch, eager). set_image_prompt: host wall clock around a call that ends in a stream synchronise (embedding upload, token
projection or Resampler for the prompt and its negative, K/V hoist of the 70 cross-attentions), median of R, for a new attachment
(plan rebuilt at the next step) and for an in-place rewrite. The card's name, power limit and clocks are read in the same run.
"""
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "stable-diffusion-xl-burn_b200"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)

import torch  # noqa: E402
import sdxl_b200  # noqa: E402
from sdxl_b200 import build_pack  # noqa: E402
from sdxl_b200.clip_vision import SDXL_VIT_BIGG, SDXL_VIT_H, ClipVisionEncoder, synth_vision_weights  # noqa: E402
from sdxl_b200.ip_adapter import SDXL_PLUS, synth_ip_adapter  # noqa: E402
from controlnet_bench import gpu_info  # noqa: E402

HW = 1024
D = 1024   # ViT-H/14 image_embeds
D_PLUS = 1280   # ViT-H/14 hidden width
L_PLUS = 257    # ViT-H/14 tokens per image


def main():
    args = sys.argv[1:]
    opt = lambda name, d: type(d)(args[args.index(name) + 1]) if name in args else d  # noqa: E731
    steps, warmup, reps = opt("--steps", 31), opt("--warmup", 4), opt("--reps", 3)
    out_path = args[0] if args and not args[0].startswith("--") else None
    ctx = sdxl_b200.Context(0)
    dev = str(ctx.device)
    res = {"gpu": gpu_info()}
    d = sdxl_b200.Diffuser(ctx, sdxl_b200.SDXL_BASE, sdxl_b200.build_pack(sdxl_b200.synth_weights(sdxl_b200.SDXL_BASE, seed=0, device=dev)))
    ad = sdxl_b200.IPAdapter(ctx, sdxl_b200.SDXL_BASE, D, synth_ip_adapter(sdxl_b200.SDXL_BASE, D, seed=1))
    plus = sdxl_b200.IPAdapter(ctx, sdxl_b200.SDXL_BASE, D_PLUS, synth_ip_adapter(sdxl_b200.SDXL_BASE, D_PLUS, seed=1, resampler=SDXL_PLUS))
    torch.cuda.empty_cache()
    g = lambda s: torch.Generator().manual_seed(s)  # noqa: E731
    emb = {k: torch.randn(1, k, D, generator=g(10 + k)) for k in (1, 4)}
    hid = {k: torch.randn(1, k, L_PLUS, D_PLUS, generator=g(20 + k)) for k in (1, 4)}
    hid_neg = {k: torch.randn(1, k, L_PLUS, D_PLUS, generator=g(30 + k)) for k in (1, 4)}
    kinds = ["none", "base_1", "base_4", "plus_1", "plus_4", "base_plus", "base_plus_masked", "base_2_masked"]
    left = torch.zeros(1, HW, HW)
    left[:, :, :HW // 2] = 1
    emb2 = torch.randn(1, 2, D, generator=g(40))
    cond = sdxl_b200.Conditioning(
        context_full=torch.randn(1, 77, 2048, generator=g(1)).half(), unconditional_context_full=torch.randn(77, 2048, generator=g(2)).half(),
        channel_context=torch.randn(1, 2816, generator=g(3)).half(), unconditional_channel_context=torch.randn(2816, generator=g(4)).half(),
        resolution=(HW, HW))
    ts = sdxl_b200.ddim_timesteps(30)
    step_size = 1000 // 30

    def prompt(kind, scale=1.0):
        if kind == "none":
            d.set_image_prompt(None)
        elif kind.startswith("base_plus"):
            m = kind.endswith("masked")
            d.set_image_prompts([(ad, emb[1], scale, None, left if m else None),
                                 (plus, hid[1], scale, hid_neg[1], 1 - left if m else None)])
        elif kind == "base_2_masked":
            d.set_image_prompts([(ad, emb2, scale, None, torch.cat([left, 1 - left]))])
        elif kind.startswith("base"):
            d.set_image_prompt(ad, emb[int(kind[-1])], scale)
        else:
            d.set_image_prompt(plus, hid[int(kind[-1])], scale, negative=hid_neg[int(kind[-1])])

    def attach(kind):
        prompt(kind)
        d.sampler_begin(cond, 7.5)

    def run_steps():
        d.sampler_set_latent(ctx.randn(4 * (HW // 8) ** 2, seed=0).reshape(1, 4, HW // 8, HW // 8))
        for i in range(warmup):
            t = ts[i % len(ts)]
            d.sampler_step(t, t - step_size if t >= step_size else -1)
        ctx.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(ctx.stream)
        for i in range(steps):
            t = ts[i % len(ts)]
            d.sampler_step(t, t - step_size if t >= step_size else -1)
        e1.record(ctx.stream)
        ctx.synchronize()
        return e0.elapsed_time(e1) / steps

    step = {k: [] for k in kinds}
    for r in range(reps):
        for k in kinds[r % len(kinds):] + kinds[:r % len(kinds)]:
            attach(k)
            step[k].append(round(run_steps(), 3))
    res["step_ms"] = {k: {"median": statistics.median(v), "runs": v} for k, v in step.items()}
    b = res["step_ms"]["none"]["median"]
    res["step_ratio_vs_base"] = {k: round(v["median"] / b, 3) for k, v in res["step_ms"].items()}
    res["gpu_after_steps"] = gpu_info()
    print(json.dumps(res["step_ms"]), flush=True)

    res["attention"] = {}
    for k in kinds:
        attach(k)
        run_steps()
        prof = d.profile_plan()
        total = sum(v["ms"] for v in prof.values())
        a = prof.get("attention_wgmma", {"ms": 0.0, "launches": 0})
        res["attention"][k] = {"attention_ms": round(a["ms"], 3), "launches": a["launches"], "step_ms_eager": round(total, 3),
                                           "share": round(a["ms"] / total, 4), "plan_flops": d.plan_flops}

    def timed(fn, before=lambda: None):
        ts_ = []
        for _ in range(reps):
            before()
            ctx.synchronize()
            t0 = time.perf_counter()
            fn()
            ctx.synchronize()
            ts_.append((time.perf_counter() - t0) * 1e3)
        return round(statistics.median(ts_), 2)

    attach("none")
    res["set_image_prompt_ms"] = {
        "attach_one_image": timed(lambda: prompt("base_1"), before=lambda: prompt("none")),
        "rescale_in_place": timed(lambda: prompt("base_1", 0.6)),
        "plus_attach_one_image": timed(lambda: prompt("plus_1"), before=lambda: prompt("none")),
        "plus_in_place_one_image": timed(lambda: prompt("plus_1", 0.6)),
        "plus_attach_four_images": timed(lambda: prompt("plus_4"), before=lambda: prompt("none")),
    }
    res["set_image_prompts_ms"] = {
        "attach_base_plus_masked": timed(lambda: prompt("base_plus_masked"), before=lambda: prompt("none")),
        "rewrite_base_plus_masked": timed(lambda: prompt("base_plus_masked", 0.6)),
    }
    d.set_image_prompt(None)
    res["encode_ms_per_image"] = {}
    for name, vcfg in (("vit_h", SDXL_VIT_H), ("vit_bigg", SDXL_VIT_BIGG)):
        enc = ClipVisionEncoder(ctx, vcfg, build_pack(synth_vision_weights(vcfg, seed=2, device=dev)))
        px = torch.randn(4, 3, 224, 224, device=ctx.device)
        for _ in range(3):
            enc.encode(px)
        ctx.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(ctx.stream)
        for _ in range(10):
            enc.encode(px)
        e1.record(ctx.stream)
        ctx.synchronize()
        res["encode_ms_per_image"][name] = round(e0.elapsed_time(e1) / 40, 3)
        if vcfg is SDXL_VIT_H:   # IP-Adapter Plus features: hidden_states[-2] (31 of 32 blocks, no pooled output)
            for _ in range(3):
                enc.encode_hidden(px)
            ctx.synchronize()
            e0.record(ctx.stream)
            for _ in range(10):
                enc.encode_hidden(px)
            e1.record(ctx.stream)
            ctx.synchronize()
            res["encode_ms_per_image"]["vit_h_hidden"] = round(e0.elapsed_time(e1) / 40, 3)
        enc.close()
        torch.cuda.empty_cache()
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    ad.close()
    plus.close()
    d.close()
    ctx.close()


if __name__ == "__main__":
    main()
