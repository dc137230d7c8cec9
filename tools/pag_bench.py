#!/usr/bin/env python
"""Sampler step time of SDXL base without perturbed-attention guidance, with PAG on the 10 mid-block self-attentions ("mid", diffusers'
default) and with PAG on all 70 self-attentions, synthetic weights, one GPU, in one process.

    python tools/pag_bench.py [out.json] [--steps K] [--warmup W] [--reps R]

Step time: bench.py's method (sampler_begin, W warm-up steps, CUDA events around K sampler steps, CFG 7.5 at 1024^2, batch 1), one UNet
per variant so no plan is rebuilt between rounds, the three in rotating order over R rounds. Also the per-kind profile of one PAG step of
each PAG variant (Diffuser.profile_plan; the identity self-attention is kind pag_identity) and the card's name, power limit and clocks
read in the same run.
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
VARIANTS = (("none", None), ("mid", "mid"), ("all", [".*"]))


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
    for name, layers in VARIANTS:
        d = sdxl_b200.Diffuser(ctx, sdxl_b200.SDXL_BASE, sdxl_b200.build_pack(sdxl_b200.synth_weights(sdxl_b200.SDXL_BASE, seed=0, device=dev)))
        if layers is not None:
            d.set_pag(layers, 3.0)
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
        for name in names[r % 3:] + names[:r % 3]:
            step[name].append(round(run_steps(models[name]), 3))
    res["step_ms"] = {k: {"median": statistics.median(v), "runs": v} for k, v in step.items()}
    for name in ("mid", "all"):
        res[f"step_ratio_{name}_vs_none"] = round(res["step_ms"][name]["median"] / res["step_ms"]["none"]["median"], 4)
    print(json.dumps(res["step_ms"]), flush=True)
    for name in ("mid", "all"):
        run_steps(models[name])
        prof = models[name].profile_plan()
        total = sum(v["ms"] for v in prof.values())
        res[f"profile_{name}"] = prof
        res[f"pag_identity_{name}"] = {"us": round(prof["pag_identity"]["ms"] * 1e3, 1), "launches": prof["pag_identity"]["launches"],
                                       "share_of_step": round(prof["pag_identity"]["ms"] / total, 5)}
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    for d in models.values():
        d.set_pag(None)
        d.close()
    ctx.close()


if __name__ == "__main__":
    main()
