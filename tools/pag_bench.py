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

import stepbench as sb
import torch
import sdxl_b200

VARIANTS = (("none", None), ("mid", "mid"), ("all", [".*"]))


def main():
    out_path, steps, warmup, reps = sb.options(steps=31, warmup=4, reps=3)
    ctx = sdxl_b200.Context(0)
    res = {"gpu": sb.gpu_info()}
    models = {}
    for name, layers in VARIANTS:
        d = sb.load_unet(ctx)
        if layers is not None:
            d.set_pag(layers, 3.0)
        models[name] = d
        torch.cuda.empty_cache()
    cond = sb.conditioning()

    res["step_ms"] = sb.step_rounds([n for n, _ in VARIANTS], reps, lambda name: sb.run_steps(ctx, models[name], steps, warmup, begin=cond))
    for name in ("mid", "all"):
        res[f"step_ratio_{name}_vs_none"] = round(res["step_ms"][name]["median"] / res["step_ms"]["none"]["median"], 4)
    print(json.dumps(res["step_ms"]), flush=True)
    for name in ("mid", "all"):
        sb.run_steps(ctx, models[name], steps, warmup, begin=cond)
        prof = models[name].profile_plan()
        total = sum(v["ms"] for v in prof.values())
        res[f"profile_{name}"] = prof
        res[f"pag_identity_{name}"] = {"us": round(prof["pag_identity"]["ms"] * 1e3, 1), "launches": prof["pag_identity"]["launches"],
                                       "share_of_step": round(prof["pag_identity"]["ms"] / total, 5)}
    res["gpu_after"] = sb.gpu_info()
    sb.report(res, out_path)
    for d in models.values():
        d.set_pag(None)
        d.close()
    ctx.close()


if __name__ == "__main__":
    main()
