#!/usr/bin/env python
"""Sampler step time of SDXL base without and with FreeU (the recommended SDXL values s1 = 0.9, s2 = 0.2, b1 = 1.3, b2 = 1.4),
synthetic weights, one GPU, in one process.

    python tools/freeu_bench.py [out.json] [--steps K] [--warmup W] [--reps R]

Step time: bench.py's method (sampler_begin, W warm-up steps, CUDA events around K sampler steps, CFG 7.5 at 1024^2, batch 1), one UNet
per variant so no plan is rebuilt between rounds, the two alternating over R rounds (each round starts with the other one). Also the
per-kind profile of one FreeU step (Diffuser.profile_plan; the FreeU launches are kind freeu), the bytes the freeu launches move per
step and the card's name, power limit and clocks read in the same run.
"""
import json

import stepbench as sb
import torch
import sdxl_b200

FREEU = (0.9, 0.2, 1.3, 1.4)
VARIANTS = (("none", None), ("freeu", FREEU))


def main():
    out_path, steps, warmup, reps = sb.options(steps=31, warmup=4, reps=3)
    ctx = sdxl_b200.Context(0)
    res = {"gpu": sb.gpu_info()}
    models = {}
    for name, values in VARIANTS:
        d = sb.load_unet(ctx)
        if values is not None:
            d.set_freeu(*values)
        models[name] = d
        torch.cuda.empty_cache()
    h = sb.HW // 8
    cond = sb.conditioning()

    res["step_ms"] = sb.step_rounds([n for n, _ in VARIANTS], reps, lambda name: sb.run_steps(ctx, models[name], steps, warmup, begin=cond))
    res["step_ratio_freeu_vs_none"] = round(res["step_ms"]["freeu"]["median"] / res["step_ms"]["none"]["median"], 4)
    print(json.dumps(res["step_ms"]), flush=True)
    sb.run_steps(ctx, models["freeu"], steps, warmup, begin=cond)
    prof = models["freeu"].profile_plan()
    total = sum(v["ms"] for v in prof.values())
    res["profile_freeu"] = prof
    # per CFG row (2 rows): the skip read twice and written once, the first half of x read and written, at output blocks 0..5
    cfg = sdxl_b200.SDXL_BASE
    mc, mults = cfg.model_channels, cfg.channel_mults
    n_lv = len(mults)
    skip_c = [mults[-1] * mc] * 2 + [mults[-2] * mc] + [mults[-2] * mc] * 2 + [mults[-3] * mc]   # input-block outputs, popped in reverse
    x_c = [mults[-1] * mc] * 3 + [mults[-1] * mc] + [mults[-2] * mc] * 2
    px = [(h >> (n_lv - 1)) ** 2] * 3 + [(h >> (n_lv - 2)) ** 2] * 3
    nbytes = 2 * sum(4 * p * (3 * c + xc) for p, c, xc in zip(px, skip_c, x_c))
    fu = prof["freeu"]
    res["freeu_kernel"] = {"us": round(fu["ms"] * 1e3, 1), "launches": fu["launches"], "share_of_step": round(fu["ms"] / total, 5),
                           "bytes_per_step": nbytes, "GB_per_s": round(nbytes / (fu["ms"] * 1e-3) / 1e9, 1)}
    res["gpu_after"] = sb.gpu_info()
    sb.report(res, out_path)
    for d in models.values():
        d.set_freeu(None)
        d.close()
    ctx.close()


if __name__ == "__main__":
    main()
