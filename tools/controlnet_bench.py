#!/usr/bin/env python
"""Sampler step time with 0, 1 and 2 ControlNets attached, and the set_controls time, SDXL base + SDXL ControlNets (synthetic
weights) on one GPU.

    python tools/controlnet_bench.py [out.json] [--steps K] [--warmup W] [--reps R] [--dump per_op.csv]

Step time: bench.py's method (sampler_begin, W warm-up steps, CUDA events around K sampler steps, CFG 7.5 at 1024^2, batch 1),
with 0, 1 and 2 controls alternated R times in one process. set_controls: host wall clock around a call that ends in a stream
synchronise (hint upload, hint encoding at 1024^2, zero-conv scaling, conditioning hoist), median of R, for a new attachment
(plan rebuilt at the next step) and for a scale change (in place). Also the per-kind profile of one step with one control,
the per-op CSV (--dump) and the card's name, power limit and clocks read in the same run.
"""
import json
import os
import statistics
import subprocess
import sys
import time

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
    steps, warmup, reps, dump = opt("--steps", 31), opt("--warmup", 4), opt("--reps", 3), opt("--dump", "")
    out_path = args[0] if args and not args[0].startswith("--") else None
    ctx = sdxl_b200.Context(0)
    dev = str(ctx.device)
    res = {"gpu": gpu_info()}
    d = sdxl_b200.Diffuser(ctx, sdxl_b200.SDXL_BASE, sdxl_b200.build_pack(sdxl_b200.synth_weights(sdxl_b200.SDXL_BASE, seed=0, device=dev)))
    nets = [sdxl_b200.ControlNet(ctx, sdxl_b200.SDXL_CONTROLNET,
                                 sdxl_b200.build_pack(sdxl_b200.synth_weights(sdxl_b200.SDXL_CONTROLNET, seed=s, device=dev))) for s in (1, 2)]
    torch.cuda.empty_cache()
    g = lambda s: torch.Generator().manual_seed(s)  # noqa: E731
    hints = [torch.rand(1, 3, HW, HW, generator=g(10 + i)).to(ctx.device) for i in range(2)]
    cond = sdxl_b200.Conditioning(
        context_full=torch.randn(1, 77, 2048, generator=g(1)).half(), unconditional_context_full=torch.randn(77, 2048, generator=g(2)).half(),
        channel_context=torch.randn(1, 2816, generator=g(3)).half(), unconditional_channel_context=torch.randn(2816, generator=g(4)).half(),
        resolution=(HW, HW))
    ts = sdxl_b200.ddim_timesteps(30)
    step_size = 1000 // 30

    def attach(k):
        d.set_controls([(nets[i], hints[i], 1.0) for i in range(k)])
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

    step = {0: [], 1: [], 2: []}
    for _ in range(reps):
        for k in (0, 1, 2):
            attach(k)
            step[k].append(round(run_steps(), 3))
    res["step_ms"] = {f"{k}_controls": {"median": statistics.median(v), "runs": v} for k, v in step.items()}
    b = res["step_ms"]["0_controls"]["median"]
    res["step_ratio_vs_base"] = {k: round(v["median"] / b, 3) for k, v in res["step_ms"].items()}
    print(json.dumps(res["step_ms"]), flush=True)

    def timed(fn, before=lambda: None):
        ts_ = []
        for _ in range(reps):
            before()          # untimed set-up
            ctx.synchronize()
            t0 = time.perf_counter()
            fn()
            ctx.synchronize()
            ts_.append((time.perf_counter() - t0) * 1e3)
        return round(statistics.median(ts_), 2)

    res["set_controls_ms"] = {
        # attach to a UNet with no control (the detach before it is not timed)
        "attach_one": timed(lambda: d.set_controls([(nets[0], hints[0], 1.0)]), before=lambda: d.set_controls([])),
        "rescale_in_place": timed(lambda: d.set_controls([(nets[0], hints[0], 0.8)])),
    }
    attach(1)
    run_steps()
    res["profile_one_control"] = d.profile_plan()
    res["plan_flops"] = {}
    for k in (0, 1):
        attach(k)
        run_steps()
        res["plan_flops"][f"{k}_controls"] = d.plan_flops
    if dump:
        attach(1)
        run_steps()
        d.profile_dump(dump)
    d.set_controls([])
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    for n in nets:
        n.close()
    d.close()
    ctx.close()


if __name__ == "__main__":
    main()
