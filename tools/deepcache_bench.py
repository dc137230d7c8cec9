#!/usr/bin/env python
"""DeepCache (Diffuser.set_deepcache) on SDXL base, synthetic weights, one GPU, 1024^2, CFG 7.5, batch 1, in one process.

    python tools/deepcache_bench.py [out.json] [--steps K] [--warmup W] [--reps R] [--profile 0|1]

  step_ms   bench.py's step timing (sampler_begin, W warm-up steps, CUDA events around K sampler steps): the full step (interval 1)
            and the cached step of branches 0, 1, 2, 3 and 5 (an interval longer than the run: the first warm-up step is the only
            full one), the variants alternating over R rounds.
  ddim_ms   the 30-step DDIM loop (sample_latent; the reference's loop runs 31 iterations) at interval 1, 2, 3 and 5, branch 0,
            host clock around the call ending in a synchronise, alternating over R rounds.
  dpm_ms    the 20-step DPM++ 2M Karras loop at interval 1 and 3, branch 0, the same way.
  --profile 1: instead, a torch.profiler trace of 10 cached branch-0 steps (a run of its own): the device time and launch count per
            kernel name per step, and the Chrome trace written next to out.json (<out>_trace.json) when one is given.
The card's name, power limit and clocks are read in the same run.
"""
import json
import os

import stepbench as sb
import torch
import sdxl_b200

BRANCHES = (0, 1, 2, 3, 5)
LONG = 1 << 30   # an interval no run reaches: every step after sampler_begin's first is cached


def profile_cached(ctx, d, cond, out_path):
    d.set_deepcache(LONG, 0)
    sb.run_steps(ctx, d, 10, 3, begin=cond)   # builds, captures and warms both lists
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        sb.run_steps(ctx, d, 10, 1, begin=None)
    kernels = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            k = kernels.setdefault(e.name, [0.0, 0])
            k[0] += e.device_time_total / 1e3
            k[1] += 1
    res = {"gpu": sb.gpu_info(), "kernels_ms_per_step": {n: round(v[0] / 11, 4) for n, v in sorted(kernels.items(), key=lambda kv: -kv[1][0])},
           "launches_per_step": {n: v[1] / 11 for n, v in kernels.items()},
           "table": prof.key_averages().table(sort_by="cuda_time_total", row_limit=30)}
    if out_path:
        prof.export_chrome_trace(os.path.splitext(out_path)[0] + "_trace.json")
    return res


def main():
    out_path, steps, warmup, reps, do_profile = sb.options(steps=31, warmup=4, reps=3, profile=0)
    ctx = sdxl_b200.Context(0)
    d = sb.load_unet(ctx)
    cond = sb.conditioning()
    if do_profile:
        sb.report(profile_cached(ctx, d, cond, out_path), out_path)
        d.set_deepcache(None)
        d.close()
        ctx.close()
        return
    res = {"gpu": sb.gpu_info()}
    variants = {"full": (1, 0), **{f"cached_b{b}": (LONG, b) for b in BRANCHES}}

    def step(name):
        d.set_deepcache(*variants[name])
        return sb.run_steps(ctx, d, steps, warmup, begin=cond)
    res["step_ms"] = sb.step_rounds(list(variants), reps, step)
    full = res["step_ms"]["full"]["median"]
    res["cached_over_full"] = {b: round(res["step_ms"][f"cached_b{b}"]["median"] / full, 4) for b in BRANCHES}
    print(json.dumps(res["step_ms"]), flush=True)

    h = sb.HW // 8
    noise = ctx.randn(4 * h * h, seed=0).reshape(1, 4, h, h)

    def loop(n_steps, interval, schedule=None):
        def run():
            d.set_deepcache(interval, 0)
            d.sample_latent(cond, 7.5, n_steps, noise=noise, schedule=schedule)
        run()   # warm-up: builds and captures the plan for this call
        return sb.timed(ctx, 1, run)
    res["ddim_ms"] = sb.step_rounds([f"interval_{k}" for k in (1, 2, 3, 5)], reps, lambda n: loop(30, int(n.split("_")[1])))
    dpm = sdxl_b200.schedulers.Schedule("dpmpp_2m", "karras", 20)
    res["dpm_ms"] = sb.step_rounds([f"interval_{k}" for k in (1, 3)], reps, lambda n: loop(20, int(n.split("_")[1]), dpm))
    for key in ("ddim_ms", "dpm_ms"):
        one = res[key]["interval_1"]["median"]
        res[key.replace("_ms", "_speedup")] = {k: round(one / v["median"], 3) for k, v in res[key].items()}
    res["gpu_after"] = sb.gpu_info()
    sb.report(res, out_path)
    d.set_deepcache(None)
    d.close()
    ctx.close()


if __name__ == "__main__":
    main()
