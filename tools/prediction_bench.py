#!/usr/bin/env python
"""The v prediction and guidance rescale (Diffuser.set_prediction, DESIGN.md §18) on SDXL base, synthetic weights, one GPU, 1024^2,
CFG 7.5, batch 1, in one process.

    python tools/prediction_bench.py [out.json] [--steps K] [--warmup W] [--reps R]

  step_ms   bench.py's step timing (sampler_begin, W warm-up steps, CUDA events around K sampler steps) for the epsilon model on the
            loaded table and the v model on the zero-terminal-SNR table, each without and with guidance rescale 0.7 (which adds the
            statistics kernel's launch to every step), the variants alternating over R rounds. The step's cost depends on the data
            through the card's power limit, so each rescale cost is taken against the same model on the same table.
  stats_us  the statistics kernel alone on the step's rows (cond | uncond of one 4 x 128 x 128 latent, the plan's eps pitch):
            CUDA events around 200 launches, median of R.
The card's name, power limit and clocks are read in the same run.
"""
import json
import statistics

import stepbench as sb
import torch
import sdxl_b200
from sdxl_b200 import _testing

# (prediction, phi, zero-terminal-SNR table): the epsilon variants on the loaded table, as bench.py runs, the v variants on the table v
# models are sampled with (an epsilon model on it reaches its t = 999 with sqrt(alpha) = 2^-12 and its latent leaves any useful range)
VARIANTS = {"epsilon": ("epsilon", 0.0, False), "epsilon_rescale_0.7": ("epsilon", 0.7, False), "v": ("v_prediction", 0.0, True),
            "v_rescale_0.7": ("v_prediction", 0.7, True)}


def stats_us(reps, ld):
    HW, C = (sb.HW // 8) ** 2, 4
    eps = torch.randn(2, HW, ld, device="cuda")
    scratch = _testing.guidance_stats_scratch(1)
    factor = torch.empty(1, device="cuda")
    n = 200
    out = []
    for _ in range(reps):
        for _ in range(10):
            _testing.guidance_stats(eps, ld, 1, C, HW, False, 7.5, 0.0, 0.7, scratch, factor)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            _testing.guidance_stats(eps, ld, 1, C, HW, False, 7.5, 0.0, 0.7, scratch, factor)
        e1.record()
        torch.cuda.synchronize()
        out.append(round(e0.elapsed_time(e1) * 1e3 / n, 3))
    return {"median": statistics.median(out), "runs": out, "eps_pitch": ld}


def main():
    out_path, steps, warmup, reps = sb.options(steps=31, warmup=4, reps=5)
    ctx = sdxl_b200.Context(0)
    d = sb.load_unet(ctx)
    cond = sb.conditioning()
    res = {"gpu": sb.gpu_info()}

    def step(name):
        kind, phi, zsnr = VARIANTS[name]
        d.set_prediction(kind, phi, zero_terminal_snr=zsnr)
        return sb.run_steps(ctx, d, steps, warmup, begin=cond)
    res["step_ms"] = sb.step_rounds(list(VARIANTS), reps, step)
    med = {k: v["median"] for k, v in res["step_ms"].items()}
    res["rescale_cost_ms"] = {"epsilon": round(med["epsilon_rescale_0.7"] - med["epsilon"], 4), "v": round(med["v_rescale_0.7"] - med["v"], 4)}
    d.set_prediction()
    res["stats_us"] = stats_us(reps, 4)   # the plan's eps rows have a pitch of out_channels = 4
    res["gpu_after"] = sb.gpu_info()
    sb.report(res, out_path)
    d.close()
    ctx.close()


if __name__ == "__main__":
    main()
