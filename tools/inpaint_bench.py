#!/usr/bin/env python
"""Sampler step time of SDXL base and of the SDXL inpainting UNet (9 input channels, a condition attached), synthetic weights, one GPU,
in one process.

    python tools/inpaint_bench.py [out.json] [--steps K] [--warmup W] [--reps R]

Step time: bench.py's method (sampler_begin, W warm-up steps, CUDA events around K sampler steps, CFG 7.5 at 1024^2, batch 1), the two
UNets alternating over R rounds (base first in even rounds, inpaint first in odd ones). Also the per-kind profile of one step of each
(Diffuser.profile_plan: the first conv is kind conv_in, one-source for base and two-source for inpaint) and the card's name, power
limit and clocks read in the same run.
"""
import json

import stepbench as sb
import torch
import sdxl_b200


def main():
    out_path, steps, warmup, reps = sb.options(steps=31, warmup=4, reps=4)
    ctx = sdxl_b200.Context(0)
    res = {"gpu": sb.gpu_info()}
    models = {}
    for name, cfg in (("base", sdxl_b200.SDXL_BASE), ("inpaint", sdxl_b200.SDXL_INPAINT)):
        models[name] = sb.load_unet(ctx, cfg)
        torch.cuda.empty_cache()
    g = lambda s: torch.Generator().manual_seed(s)  # noqa: E731
    h = sb.HW // 8
    mask = torch.zeros(1, 1, h, h)
    mask[:, :, h // 4:3 * h // 4, h // 4:3 * h // 4] = 1.0
    models["inpaint"].set_inpaint_condition(torch.cat([mask, torch.randn(1, 4, h, h, generator=g(5)) * (1 - mask)], dim=1))
    cond = sb.conditioning()

    res["step_ms"] = sb.step_rounds(["base", "inpaint"], reps, lambda name: sb.run_steps(ctx, models[name], steps, warmup, begin=cond))
    res["step_ratio_inpaint_vs_base"] = round(res["step_ms"]["inpaint"]["median"] / res["step_ms"]["base"]["median"], 4)
    print(json.dumps(res["step_ms"]), flush=True)
    for name, d in models.items():
        sb.run_steps(ctx, d, steps, warmup, begin=cond)
        prof = d.profile_plan()
        res[f"profile_{name}"] = prof
        res[f"conv_in_us_{name}"] = round(prof["conv_in"]["ms"] * 1e3, 1)
    res["gpu_after"] = sb.gpu_info()
    sb.report(res, out_path)
    models["inpaint"].set_inpaint_condition(None)
    for d in models.values():
        d.close()
    ctx.close()


if __name__ == "__main__":
    main()
