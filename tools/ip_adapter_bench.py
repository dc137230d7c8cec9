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

import stepbench as sb
import torch
import sdxl_b200
from sdxl_b200 import build_pack
from sdxl_b200.clip_vision import SDXL_VIT_BIGG, SDXL_VIT_H, ClipVisionEncoder, synth_vision_weights
from sdxl_b200.ip_adapter import SDXL_PLUS, synth_ip_adapter

HW = sb.HW
D = 1024   # ViT-H/14 image_embeds
D_PLUS = 1280   # ViT-H/14 hidden width
L_PLUS = 257    # ViT-H/14 tokens per image


def main():
    out_path, steps, warmup, reps = sb.options(steps=31, warmup=4, reps=3)
    ctx = sdxl_b200.Context(0)
    dev = str(ctx.device)
    res = {"gpu": sb.gpu_info()}
    d = sb.load_unet(ctx)
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
    cond = sb.conditioning()

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

    def run(k):
        attach(k)
        return sb.run_steps(ctx, d, steps, warmup)

    res["step_ms"] = sb.step_rounds(kinds, reps, run)
    b = res["step_ms"]["none"]["median"]
    res["step_ratio_vs_base"] = {k: round(v["median"] / b, 3) for k, v in res["step_ms"].items()}
    res["gpu_after_steps"] = sb.gpu_info()
    print(json.dumps(res["step_ms"]), flush=True)

    res["attention"] = {}
    for k in kinds:
        attach(k)
        sb.run_steps(ctx, d, steps, warmup)
        prof = d.profile_plan()
        total = sum(v["ms"] for v in prof.values())
        a = prof.get("attention_wgmma", {"ms": 0.0, "launches": 0})
        res["attention"][k] = {"attention_ms": round(a["ms"], 3), "launches": a["launches"], "step_ms_eager": round(total, 3),
                                           "share": round(a["ms"] / total, 4), "plan_flops": d.plan_flops}

    attach("none")
    res["set_image_prompt_ms"] = {
        "attach_one_image": sb.timed(ctx, reps, lambda: prompt("base_1"), before=lambda: prompt("none")),
        "rescale_in_place": sb.timed(ctx, reps, lambda: prompt("base_1", 0.6)),
        "plus_attach_one_image": sb.timed(ctx, reps, lambda: prompt("plus_1"), before=lambda: prompt("none")),
        "plus_in_place_one_image": sb.timed(ctx, reps, lambda: prompt("plus_1", 0.6)),
        "plus_attach_four_images": sb.timed(ctx, reps, lambda: prompt("plus_4"), before=lambda: prompt("none")),
    }
    res["set_image_prompts_ms"] = {
        "attach_base_plus_masked": sb.timed(ctx, reps, lambda: prompt("base_plus_masked"), before=lambda: prompt("none")),
        "rewrite_base_plus_masked": sb.timed(ctx, reps, lambda: prompt("base_plus_masked", 0.6)),
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
    res["gpu_after"] = sb.gpu_info()
    sb.report(res, out_path)
    ad.close()
    plus.close()
    d.close()
    ctx.close()


if __name__ == "__main__":
    main()
