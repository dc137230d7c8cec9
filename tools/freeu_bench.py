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
FREEU = (0.9, 0.2, 1.3, 1.4)
VARIANTS = (("none", None), ("freeu", FREEU))


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
    steps, warmup, reps = opt("--steps", 31), opt("--warmup", 4), opt("--reps", 3)
    out_path = args[0] if args and not args[0].startswith("--") else None
    ctx = sdxl_b200.Context(0)
    dev = str(ctx.device)
    res = {"gpu": gpu_info()}
    models = {}
    for name, values in VARIANTS:
        d = sdxl_b200.Diffuser(ctx, sdxl_b200.SDXL_BASE, sdxl_b200.build_pack(sdxl_b200.synth_weights(sdxl_b200.SDXL_BASE, seed=0, device=dev)))
        if values is not None:
            d.set_freeu(*values)
        models[name] = d
        torch.cuda.empty_cache()
    g = lambda s: torch.Generator().manual_seed(s)  # noqa: E731
    h = HW // 8
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

    names = [n for n, _ in VARIANTS]
    step = {n: [] for n in names}
    for r in range(reps):
        for name in names[r % 2:] + names[:r % 2]:
            step[name].append(round(run_steps(models[name]), 3))
    res["step_ms"] = {k: {"median": statistics.median(v), "runs": v} for k, v in step.items()}
    res["step_ratio_freeu_vs_none"] = round(res["step_ms"]["freeu"]["median"] / res["step_ms"]["none"]["median"], 4)
    print(json.dumps(res["step_ms"]), flush=True)
    run_steps(models["freeu"])
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
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    for d in models.values():
        d.set_freeu(None)
        d.close()
    ctx.close()


if __name__ == "__main__":
    main()
