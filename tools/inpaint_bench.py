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
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "stable-diffusion-xl-burn_b200")):
    sys.path.insert(0, p)

import torch  # noqa: E402
import sdxl_b200  # noqa: E402

HW = 1024


def gpu_info():
    try:
        q = "name,power.limit,clocks.max.sm,clocks.sm"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


def main():
    args = sys.argv[1:]
    opt = lambda name, d: type(d)(args[args.index(name) + 1]) if name in args else d  # noqa: E731
    steps, warmup, reps = opt("--steps", 31), opt("--warmup", 4), opt("--reps", 4)
    out_path = args[0] if args and not args[0].startswith("--") else None
    ctx = sdxl_b200.Context(0)
    dev = str(ctx.device)
    res = {"gpu": gpu_info()}
    models = {}
    for name, cfg in (("base", sdxl_b200.SDXL_BASE), ("inpaint", sdxl_b200.SDXL_INPAINT)):
        models[name] = sdxl_b200.Diffuser(ctx, cfg, sdxl_b200.build_pack(sdxl_b200.synth_weights(cfg, seed=0, device=dev)))
        torch.cuda.empty_cache()
    g = lambda s: torch.Generator().manual_seed(s)  # noqa: E731
    h = HW // 8
    mask = torch.zeros(1, 1, h, h)
    mask[:, :, h // 4:3 * h // 4, h // 4:3 * h // 4] = 1.0
    models["inpaint"].set_inpaint_condition(torch.cat([mask, torch.randn(1, 4, h, h, generator=g(5)) * (1 - mask)], dim=1))
    cond = sdxl_b200.Conditioning(
        context_full=torch.randn(1, 77, 2048, generator=g(1)).half(), unconditional_context_full=torch.randn(77, 2048, generator=g(2)).half(),
        channel_context=torch.randn(1, 2816, generator=g(3)).half(), unconditional_channel_context=torch.randn(2816, generator=g(4)).half(),
        resolution=(HW, HW))
    ts = sdxl_b200.ddim_timesteps(30)
    step_size = 1000 // 30

    def run_steps(d):
        d.sampler_begin(cond, 7.5)
        d.sampler_set_latent(ctx.randn(4 * h * h, seed=0).reshape(1, 4, h, h))
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

    step = {"base": [], "inpaint": []}
    for r in range(reps):
        for name in (("base", "inpaint") if r % 2 == 0 else ("inpaint", "base")):
            step[name].append(round(run_steps(models[name]), 3))
    res["step_ms"] = {k: {"median": statistics.median(v), "runs": v} for k, v in step.items()}
    res["step_ratio_inpaint_vs_base"] = round(res["step_ms"]["inpaint"]["median"] / res["step_ms"]["base"]["median"], 4)
    print(json.dumps(res["step_ms"]), flush=True)
    for name, d in models.items():
        run_steps(d)
        prof = d.profile_plan()
        res[f"profile_{name}"] = prof
        res[f"conv_in_us_{name}"] = round(prof["conv_in"]["ms"] * 1e3, 1)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    models["inpaint"].set_inpaint_condition(None)
    for d in models.values():
        d.close()
    ctx.close()


if __name__ == "__main__":
    main()
