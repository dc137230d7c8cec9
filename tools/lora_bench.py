#!/usr/bin/env python
"""LoRA apply / restore time and the sampler step with an adapter merged, SDXL base (synthetic weights) on one GPU.

    python tools/lora_bench.py [out.json] [--steps K] [--warmup W] [--reps R] [--family lora|loha|lokr|dora]

Adapters of rank 8, 32 and 128 cover every attention, feed-forward and proj_in/out Linear of the UNet (722 layers, the
layer set of a kohya SDXL LoRA). For each rank, host wall clock around a call that ends in a stream synchronise, median of R:
  apply_from_clean_ms   sdxl_unet_set_adapters on an unmerged model: backup allocation + copy, then the merge
  reapply_ms            the same adapter at another scale while merged: restore from the backups, then the merge
  restore_ms            n = 0: restore every layer and free the backups
plus the re-apply timed with CUDA events alone and the merge's FLOP count (merge_tflops_lower_bound divides it by the whole
re-apply, restore copies included). The step time uses bench.py's method (sampler_begin, W warm-up steps, CUDA events around K sampler steps,
CFG 7.5 at 1024^2, batch 1), base and rank-32-merged alternating over R rounds in one process.

--family loha | lokr | dora measures that family at rank 32 on the same 722 Linears, with a rank-32 LoRA timed the same way in the
same process beside it, and the step with the family's adapter merged against base. loha: both Hadamard factor pairs of rank 32;
lokr: w1 given whole ([a, b], a and b the divisors of N and I nearest their square roots), w2 as a rank-32 product; dora: the LoHa
adapter plus a row-form dora_scale (DESIGN.md §19), and the same with a column-form dora_scale ([1, I]) timed after it
(the step uses the row form).
"""
import math
import statistics
import time

import stepbench as sb
import torch
import sdxl_b200
from sdxl_b200.lora import unet_lora_modules


def _divisor(n):
    return max(a for a in range(1, int(math.isqrt(n)) + 1) if n % a == 0)


def adapter(cfg, paths, rank, dev, seed, family="lora"):
    shapes = {n[: -len("/weight")]: s for n, s, _, _ in sdxl_b200.unet_tensor_specs(cfg) if n.endswith("/weight")}
    g = torch.Generator(device=dev).manual_seed(seed)
    out, flops = {}, 0.0

    def rnd(*shape):
        return (torch.randn(*shape, generator=g, device=dev) * 0.02).half()

    for p in paths:
        k, n = shapes[p]   # Linear [in, out]
        if family == "lora":
            out[f"{p}/lora_down"], out[f"{p}/lora_up"] = rnd(rank, k), rnd(n, rank)
            flops += 2.0 * n * k * rank
        elif family in ("loha", "dora", "dora_col"):
            out[f"{p}/hada_w1_a"], out[f"{p}/hada_w1_b"] = rnd(n, rank), rnd(rank, k)
            out[f"{p}/hada_w2_a"], out[f"{p}/hada_w2_b"] = rnd(n, rank), rnd(rank, k)
            flops += 4.0 * n * k * rank + n * k
            if family == "dora":
                out[f"{p}/dora_scale"] = torch.ones(n, device=dev)
            elif family == "dora_col":
                out[f"{p}/dora_scale"] = torch.ones(1, k, device=dev)
        elif family == "lokr":
            a, b = _divisor(n), _divisor(k)
            out[f"{p}/lokr_w1"] = rnd(a, b)
            out[f"{p}/lokr_w2_a"], out[f"{p}/lokr_w2_b"] = rnd(n // a, rank), rnd(rank, k // b)
            flops += 2.0 * (n // a) * (k // b) * rank + n * k
        else:
            raise SystemExit(f"--family {family}: expected lora, loha, lokr or dora")
    return sdxl_b200.build_pack(out), flops


def timed(ctx, fn, reps):
    ts = []
    for _ in range(reps):
        ctx.synchronize()
        t0 = time.perf_counter()
        fn()
        ctx.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts), ts


def main():
    out_path, steps, warmup, reps, family = sb.options(steps=31, warmup=4, reps=3, family="lora")
    ctx = sdxl_b200.Context(0)
    dev = ctx.device
    cfg = sdxl_b200.SDXL_BASE
    d = sb.load_unet(ctx, cfg)
    torch.cuda.empty_cache()
    paths = [r for _, r, _ in unet_lora_modules(cfg) if "/transformer" in r]
    shapes = {n[: -len("/weight")]: s for n, s, _, _ in sdxl_b200.unet_tensor_specs(cfg) if n.endswith("/weight")}
    touched_bytes = sum(shapes[p][0] * shapes[p][1] * 2 for p in paths)
    res = {"gpu": sb.gpu_info(), "layers": len(paths), "touched_weight_bytes": touched_bytes, "family": family, "ranks": {}}

    runs = [(r, "lora") for r in (8, 32, 128)] if family == "lora" else [(32, "lora"), (32, family)]
    if family == "dora":
        runs.append((32, "dora_col"))
    for rank, fam in runs:
        pack, flops = adapter(cfg, paths, rank, dev, seed=rank, family=fam)
        timed(ctx, lambda: (d.set_adapters([(pack, 1.0)]), d.set_adapters([])), 1)   # warm-up
        apply_clean, _ = timed(ctx, lambda: d.set_adapters([(pack, 1.0)]), 1)
        restore_times, apply_times = [], [apply_clean]
        for _ in range(reps - 1):
            r, _ = timed(ctx, lambda: d.set_adapters([]), 1)
            restore_times.append(r)
            a, _ = timed(ctx, lambda: d.set_adapters([(pack, 1.0)]), 1)
            apply_times.append(a)
        reapply, _ = timed(ctx, lambda: d.set_adapters([(pack, 0.5)]), reps)
        # the same re-apply with CUDA events on the ctx stream (restore copies + merge kernels, no host work)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ctx.synchronize()
        e0.record(ctx.stream)
        d.set_adapters([(pack, 0.75)])
        e1.record(ctx.stream)
        ctx.synchronize()
        reapply_dev = e0.elapsed_time(e1)
        restore, _ = timed(ctx, lambda: d.set_adapters([]), 1)
        restore_times.append(restore)
        rs = statistics.median(restore_times)
        res["ranks"][rank if family == "lora" else f"{fam}{rank}"] = {
            "apply_from_clean_ms": round(statistics.median(apply_times), 2), "reapply_ms": round(reapply, 2),
            "reapply_device_ms": round(reapply_dev, 2), "restore_ms": round(rs, 2),
            "merge_flops": flops, "merge_tflops_lower_bound": round(flops / reapply_dev * 1e-9, 2)}
        print(f"{fam} rank {rank}: {res['ranks'][rank if family == 'lora' else f'{fam}{rank}']}", flush=True)
        del pack

    # ---- step time, bench.py's method: base and rank-32-merged alternated
    d.sampler_begin(sb.conditioning(), 7.5)
    pack32, _ = adapter(cfg, paths, 32, dev, seed=32, family=family)
    merged = "rank32" if family == "lora" else f"{family}32"

    def run(name):
        d.set_adapters([] if name == "base" else [(pack32, 1.0)])
        return sb.run_steps(ctx, d, steps, warmup)

    res["step_ms"] = sb.step_rounds(["base", merged], reps, run)
    d.set_adapters([])
    res["gpu_after"] = sb.gpu_info()
    sb.report(res, out_path)
    d.close()
    ctx.close()


if __name__ == "__main__":
    main()
