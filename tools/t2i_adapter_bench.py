#!/usr/bin/env python
"""Sampler step time with 0, 1 and 2 T2I-Adapters attached, the set_t2i_adapters time and the adapter forward time, SDXL base +
SDXL-sized adapters (synthetic weights) on one GPU.

    python tools/t2i_adapter_bench.py [out.json] [--steps K] [--warmup W] [--reps R]

Step time: bench.py's method (sampler_begin, W warm-up steps, CUDA events around K sampler steps, CFG 7.5 at 1024^2, batch 1), with
0, 1 and 2 adapters attached, R rounds in rotating order (0 1 2, 1 2 0, 2 0 1, ...) in one process. set_t2i_adapters: host wall
clock around a call that ends in a stream synchronise (hint upload, adapter forward, scale-and-sum), median of R, for a new attachment
(plan rebuilt at the next step) and for an in-place rewrite. Adapter forward: CUDA events around T2IAdapter.features of one 1024^2
hint (the forward plus the NHWC -> NCHW copies of its outputs), median of R, and its FLOPs counted from the shapes. Also the per-kind
profile of one step with one adapter and the card's name, power limit and clocks read in the same run.
"""
import json
import statistics

import stepbench as sb
import torch
import sdxl_b200

HW = sb.HW


def adapter_flops(cfg, H, W):
    """2 * MACs of one adapter forward on an H x W hint (convolutions only)."""
    ch, f = cfg.channels, 0.0
    for k in range(4):
        px = (H // (16 if k < 2 else 32)) * (W // (16 if k < 2 else 32))
        if k == 0:
            f += 2.0 * px * ch[0] * cfg.in_channels * 256 * 9
        if k in (1, 2):
            f += 2.0 * px * ch[k] * ch[k - 1]
        f += cfg.n_res_blocks * 2.0 * px * ch[k] * ch[k] * 10   # block1 3x3 + block2 1x1
    return f


def main():
    out_path, steps, warmup, reps = sb.options(steps=31, warmup=4, reps=3)
    ctx = sdxl_b200.Context(0)
    dev = str(ctx.device)
    res = {"gpu": sb.gpu_info()}
    acfg = sdxl_b200.SDXL_T2I_ADAPTER
    d = sb.load_unet(ctx)
    ads = [sdxl_b200.T2IAdapter(ctx, acfg, sdxl_b200.build_pack(sdxl_b200.synth_weights(acfg, seed=s, device=dev))) for s in (1, 2)]
    torch.cuda.empty_cache()
    g = lambda s: torch.Generator().manual_seed(s)  # noqa: E731
    hints = [torch.rand(1, 3, HW, HW, generator=g(10 + i)).to(ctx.device) for i in range(2)]
    cond = sb.conditioning()

    def attach(k):
        d.set_t2i_adapters([(ads[i], hints[i], 1.0) for i in range(k)])
        d.sampler_begin(cond, 7.5)

    def run(k):
        attach(k)
        return sb.run_steps(ctx, d, steps, warmup)

    res["step_ms"] = {f"{k}_adapters": v for k, v in sb.step_rounds([0, 1, 2], reps, run).items()}
    b = res["step_ms"]["0_adapters"]["median"]
    res["step_ratio_vs_base"] = {k: round(v["median"] / b, 4) for k, v in res["step_ms"].items()}
    print(json.dumps(res["step_ms"]), flush=True)

    res["set_t2i_adapters_ms"] = {
        # attach to a UNet with no adapter (the detach before it is not timed)
        "attach_one": sb.timed(ctx, reps, lambda: d.set_t2i_adapters([(ads[0], hints[0], 1.0)]), before=lambda: d.set_t2i_adapters([])),
        "rewrite_in_place": sb.timed(ctx, reps, lambda: d.set_t2i_adapters([(ads[0], hints[0], 0.8)])),
        "attach_two": sb.timed(ctx, reps, lambda: d.set_t2i_adapters([(ads[i], hints[i], 1.0) for i in range(2)]),
                               before=lambda: d.set_t2i_adapters([])),
    }
    fw = []
    ads[0].features(hints[0])
    for _ in range(max(reps, 5)):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ctx.synchronize()
        e0.record(ctx.stream)
        ads[0].features(hints[0])
        e1.record(ctx.stream)
        ctx.synchronize()
        fw.append(e0.elapsed_time(e1))
    res["adapter_forward_ms_per_image"] = round(statistics.median(fw), 3)
    res["adapter_forward_gflop_per_image"] = round(adapter_flops(acfg, HW, HW) * 1e-9, 1)
    attach(1)
    sb.run_steps(ctx, d, steps, warmup)
    res["profile_one_adapter"] = d.profile_plan()
    # the four adds' HBM traffic per CFG step: read x and F, write x, over 2 rows
    res["add_bytes_per_step"] = sum(2 * 3 * 4 * (HW // d_) ** 2 * c for c, d_ in zip(acfg.channels, (16, 16, 32, 32)))
    d.set_t2i_adapters([])
    res["gpu_after"] = sb.gpu_info()
    sb.report(res, out_path)
    for a in ads:
        a.close()
    d.close()
    ctx.close()


if __name__ == "__main__":
    main()
