#!/usr/bin/env python
"""Step and image time of the scheduled samplers against the DDIM loop, SDXL base (synthetic weights) at 1024^2, batch 1, one GPU.

    python tools/sampler_bench.py [out.json] [--steps N] [--reps R]

CUDA events on the ctx stream around whole on-device calls (device-resident conditioning and output, seeded noise), every
configuration warmed once and then run R times in rotating order in one process:
  (a) ms per step at the same N (default 10, so that the DDIM loop also runs N steps): DDIM through sdxl_sample_latent against
      Euler, Euler-ancestral, DPM++ 2M (Karras) and LCM through sdxl_sample_latent_scheduled, all with CFG 7.5;
  (b) ms per image: 30-step DDIM CFG (31 iterations, as the reference's loop runs them), 20-step DPM++ 2M Karras CFG, 4-step Euler
      trailing without CFG;
  (c) the step kernel alone: CUDA events around 200 launches at the 1024^2 latent, CFG rows, in-kernel noise.
Also the card's name, power limit and clocks read in the same run. Fails without a GPU. Synthetic weights: times only, the latents
say nothing about image quality."""
import statistics

import stepbench as sb
import torch
import sdxl_b200
from sdxl_b200 import _testing
from sdxl_b200.schedulers import Schedule

HW = sb.HW


def main():
    out_path, n, reps = sb.options(steps=10, reps=3)
    reps = max(reps, 3)
    if not torch.cuda.is_available():
        raise SystemExit("sampler_bench: no CUDA device; there is nothing to measure without one")
    ctx = sdxl_b200.Context(0)
    dev = str(ctx.device)
    res = {"gpu": sb.gpu_info(), "resolution": HW, "steps": n, "reps": reps}
    d = sb.load_unet(ctx)
    cond = sb.conditioning()

    def timed(schedule, steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(ctx.stream)
        d.sample_latent(cond, 7.5, steps, seed=1, schedule=schedule)
        e1.record(ctx.stream)
        e1.synchronize()
        return e0.elapsed_time(e1)

    def rounds(configs):
        """configs: name -> (schedule | None, n_steps, iterations). Returns name -> list of ms per call."""
        names = list(configs)
        for k in names:
            timed(*configs[k][:2])   # warm-up: plan build, graph capture
        ms = {k: [] for k in names}
        for r in range(reps):
            for k in names[r % len(names):] + names[:r % len(names)]:
                ms[k].append(timed(*configs[k][:2]))
        return ms

    step_cfgs = {"ddim": (None, n, n), "euler": (Schedule("euler", "reference", n), n, n),
                 "euler_ancestral": (Schedule("euler_ancestral", "reference", n), n, n),
                 "dpmpp_2m_karras": (Schedule("dpmpp_2m", "karras", n), n, n), "lcm": (Schedule("lcm", "lcm", n), n, n)}
    if 1000 % n:
        raise SystemExit("sampler_bench: --steps must divide 1000 so that the DDIM loop runs the same number of steps")
    ms = rounds(step_cfgs)
    res["ms_per_step"] = {k: {"median": statistics.median(v) / n, "min": min(v) / n, "max": max(v) / n} for k, v in ms.items()}
    image_cfgs = {"ddim_30_cfg": (None, 30, 31), "dpmpp_2m_karras_20_cfg": (Schedule("dpmpp_2m", "karras", 20), 20, 20),
                  "euler_trailing_4_no_cfg": (Schedule("euler", "trailing", 4, no_cfg=True), 4, 4)}
    ms = rounds(image_cfgs)
    res["ms_per_image"] = {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "unet_steps": image_cfgs[k][2]} for k, v in ms.items()}

    # (c) the kernel alone
    lat = (1, 4, HW // 8, HW // 8)
    eps = torch.randn(2, (HW // 8) ** 2, 4, device=dev)
    xh, x_in, hist = (torch.zeros(lat, device=dev) for _ in range(3))
    for name, coef in (("euler", (0.9, 0.1, 0.0, 0.0, 0.5)), ("dpmpp_2m_history", (0.9, 0.15, -0.05, 0.0, 0.5)),
                       ("ancestral_in_kernel_noise", (0.9, 0.1, 0.0, 0.3, 0.5))):
        run = lambda: _testing.guided_step(eps, 4, 1, 4, (HW // 8) ** 2, True, False, 7.5, 0.0, 1.0, coef, xh, x_in, hist, coef[2] != 0.0, seed=1)  # noqa: E731
        for _ in range(20):
            run()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(200):
            run()
        e1.record()
        e1.synchronize()
        res.setdefault("step_kernel_us", {})[name] = e0.elapsed_time(e1) / 200 * 1e3
    d.close()
    ctx.close()
    sb.report(res, out_path)


if __name__ == "__main__":
    main()
