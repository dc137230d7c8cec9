#!/usr/bin/env python
"""Instruction-based editing (Diffuser.set_edit_image, DESIGN.md §21) against text-to-image on SDXL-base-shaped UNets, synthetic weights,
one GPU, 1024^2, batch 1, in one process.

    python tools/edit_bench.py [out.json] [--steps K] [--warmup W] [--reps R]

  step_ms     bench.py's step timing (sampler_begin, W warm-up steps, CUDA events around K sampler steps) for SDXL base with CFG 7.5
              (two row groups) and the edit UNet (8-channel first conv) with CFG 7.5 and image guidance 1.5 (three row groups),
              the two alternating over R rounds.
  kernel_us   each form of the step kernels on one 4 x 128 x 128 latent's rows (the plan's eps pitch 4): CUDA events around 200
              launches, median of R; the existing forms (cfg_ddim and guided_step on [cond | uncond]) beside the image-guidance
              forms (on [cond | img | uncond]), and the guidance-rescale statistics kernel in both forms.
The card's name, power limit and clocks are read in the same run.
"""
import statistics

import stepbench as sb
import torch
import sdxl_b200
from sdxl_b200 import _testing


def kernel_us(reps):
    HW, Cc, ld, n = (sb.HW // 8) ** 2, 4, 4, 200
    eps = torch.randn(3, HW, ld, device="cuda")
    x, xh, x_in, hist = (torch.randn(1, Cc, HW, device="cuda") for _ in range(4))
    scratch = _testing.guidance_stats_scratch(1)
    factor = torch.empty(1, device="cuda")
    coef = (0.9, 0.1, 0.0, 0.0, 0.7)
    forms = {
        "cfg_ddim": lambda: _testing.cfg_ddim(eps, ld, 1, Cc, HW, True, 7.5, 0.9, 0.4, 0.95, 0.3, x),
        "cfg_ddim_img": lambda: _testing.cfg_ddim_img(eps, ld, 1, Cc, HW, 5.0, 1.5, 0.9, 0.4, 0.95, 0.3, x),
        "guided_step": lambda: _testing.guided_step(eps, ld, 1, Cc, HW, True, False, 7.5, 0.0, 2.0, coef, xh, x_in),
        "guided_step_img": lambda: _testing.guided_step_img(eps, ld, 1, Cc, HW, 5.0, 1.5, 2.0, coef, xh, x_in),
        "guided_step_rows": lambda: _testing.guided_step_rows(eps, ld, 1, Cc, HW, True, False, 7.5, 0.0, 2.0, (0.9, 0.0, 0.1, 0.2, 0.0, 0.0, 0.7),
                                                              (0.0,) * 5, xh, x_in, hist),
        "guided_step_img_rows": lambda: _testing.guided_step_img(eps, ld, 1, Cc, HW, 5.0, 1.5, 2.0, (0.9, 0.0, 0.1, 0.2, 0.0, 0.0, 0.7), xh, x_in,
                                                                 hist, rows=(0.0,) * 5),
        "guidance_stats": lambda: _testing.guidance_stats(eps, ld, 1, Cc, HW, False, 7.5, 0.0, 0.7, scratch, factor),
        "guidance_stats_img": lambda: _testing.guidance_stats_img(eps, ld, 1, Cc, HW, 5.0, 1.5, 0.7, scratch, factor),
    }
    res = {k: [] for k in forms}
    for _ in range(reps):
        for name, f in forms.items():   # alternate the forms within each round
            for _ in range(10):
                f()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                f()
            e1.record()
            torch.cuda.synchronize()
            res[name].append(round(e0.elapsed_time(e1) * 1e3 / n, 3))
    return {k: {"median": statistics.median(v), "runs": v} for k, v in res.items()}


def main():
    out_path, steps, warmup, reps = sb.options(steps=21, warmup=3, reps=5)
    ctx = sdxl_b200.Context(0)
    res = {"gpu": sb.gpu_info()}
    base = sb.load_unet(ctx)
    edit = sb.load_unet(ctx, sdxl_b200.SDXL_EDIT)
    edit.set_edit_image(0.5 * torch.randn(1, 4, sb.HW // 8, sb.HW // 8, generator=torch.Generator().manual_seed(5)), 1.5)
    cond = sb.conditioning()
    runs = {"base_cfg": lambda: sb.run_steps(ctx, base, steps, warmup, begin=cond),
            "edit_cfg_img": lambda: sb.run_steps(ctx, edit, steps, warmup, begin=cond)}
    res["step_ms"] = sb.step_rounds(list(runs), reps, lambda name: runs[name]())
    med = {k: v["median"] for k, v in res["step_ms"].items()}
    res["edit_over_base"] = round(med["edit_cfg_img"] / med["base_cfg"], 4)
    res["kernel_us"] = kernel_us(reps)
    res["gpu_after"] = sb.gpu_info()
    sb.report(res, out_path)
    base.close()
    edit.close()
    ctx.close()


if __name__ == "__main__":
    main()
