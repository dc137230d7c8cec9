#!/usr/bin/env python
"""Sampler step time with 0, 1 and 2 ControlNets attached, and the set_controls time, SDXL base + SDXL ControlNets (synthetic
weights) on one GPU.

    python tools/controlnet_bench.py [out.json] [--steps K] [--warmup W] [--reps R] [--dump per_op.csv]

Step time: bench.py's method (sampler_begin, W warm-up steps, CUDA events around K sampler steps, CFG 7.5 at 1024^2, batch 1),
with 0, 1 and 2 controls alternated in rotating order over R rounds in one process. set_controls: host wall clock around a call
that ends in a stream synchronise (hint upload, hint encoding at 1024^2, zero-conv scaling, conditioning hoist), median of R, for a
new attachment (plan rebuilt at the next step) and for a scale change (in place). Also the per-kind profile of one step with one
control, the per-op CSV (--dump) and the card's name, power limit and clocks read in the same run.
"""
import json

import stepbench as sb
import torch
import sdxl_b200


def main():
    out_path, steps, warmup, reps, dump = sb.options(steps=31, warmup=4, reps=3, dump="")
    ctx = sdxl_b200.Context(0)
    dev = str(ctx.device)
    res = {"gpu": sb.gpu_info()}
    d = sb.load_unet(ctx)
    nets = [sdxl_b200.ControlNet(ctx, sdxl_b200.SDXL_CONTROLNET,
                                 sdxl_b200.build_pack(sdxl_b200.synth_weights(sdxl_b200.SDXL_CONTROLNET, seed=s, device=dev))) for s in (1, 2)]
    torch.cuda.empty_cache()
    g = lambda s: torch.Generator().manual_seed(s)  # noqa: E731
    hints = [torch.rand(1, 3, sb.HW, sb.HW, generator=g(10 + i)).to(ctx.device) for i in range(2)]
    cond = sb.conditioning()

    def attach(k):
        d.set_controls([(nets[i], hints[i], 1.0) for i in range(k)])
        d.sampler_begin(cond, 7.5)

    def run(k):
        attach(k)
        return sb.run_steps(ctx, d, steps, warmup)

    res["step_ms"] = {f"{k}_controls": v for k, v in sb.step_rounds([0, 1, 2], reps, run).items()}
    b = res["step_ms"]["0_controls"]["median"]
    res["step_ratio_vs_base"] = {k: round(v["median"] / b, 3) for k, v in res["step_ms"].items()}
    print(json.dumps(res["step_ms"]), flush=True)

    res["set_controls_ms"] = {
        # attach to a UNet with no control (the detach before it is not timed)
        "attach_one": sb.timed(ctx, reps, lambda: d.set_controls([(nets[0], hints[0], 1.0)]), before=lambda: d.set_controls([])),
        "rescale_in_place": sb.timed(ctx, reps, lambda: d.set_controls([(nets[0], hints[0], 0.8)])),
    }
    attach(1)
    sb.run_steps(ctx, d, steps, warmup)
    res["profile_one_control"] = d.profile_plan()
    res["plan_flops"] = {}
    for k in (0, 1):
        attach(k)
        sb.run_steps(ctx, d, steps, warmup)
        res["plan_flops"][f"{k}_controls"] = d.plan_flops
    if dump:
        attach(1)
        sb.run_steps(ctx, d, steps, warmup)
        d.profile_dump(dump)
    d.set_controls([])
    res["gpu_after"] = sb.gpu_info()
    sb.report(res, out_path)
    for n in nets:
        n.close()
    d.close()
    ctx.close()


if __name__ == "__main__":
    main()
