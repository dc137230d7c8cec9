#!/usr/bin/env python
"""Step and image time of the scheduled samplers against the DDIM loop, SDXL base (synthetic weights) at 1024^2, batch 1, one GPU.

    python tools/sampler_bench.py [out.json] [--steps N] [--reps R]

CUDA events on the ctx stream around whole on-device calls (device-resident conditioning and output, seeded noise), every
configuration warmed once and then run R times in rotating order in one process:
  (a) ms per step at the same N (default 10, so that the DDIM loop also runs N steps): DDIM through sdxl_sample_latent against
      Euler, Euler-ancestral, DPM++ 2M (Karras) and LCM through sdxl_sample_latent_scheduled, all with CFG 7.5;
  (b) ms per image: 30-step DDIM CFG (31 iterations, as the reference's loop runs them), 20-step DPM++ 2M Karras CFG, 4-step Euler
      trailing without CFG;
  (c) the step kernel alone: CUDA events around 200 launches at the 1024^2 latent, CFG rows, in-kernel noise, in its one-row
      form and in the two-row form of DESIGN.md §20 (UniPC's corrected launch, Heun's second stage);
  (d) ms per UNet evaluation at the same N, Karras: Euler against DPM++ 2M SDE, DPM++ 3M SDE, UniPC, Heun and DPM2 (Heun and DPM2
      evaluate 2N - 1 times), and ms per image of 20-step DPM++ 2M SDE Karras, 20-step UniPC Karras and 10-step Heun Karras.
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

    # (d) the samplers of DESIGN.md §20: time per evaluation against Euler's, and per image
    eval_cfgs = {name: (Schedule(name, "karras", n), n, Schedule(name, "karras", n).n_evaluations())
                 for name in ("euler", "dpmpp_2m_sde", "dpmpp_3m_sde", "unipc", "heun_discrete", "dpm_2")}
    ms = rounds(eval_cfgs)
    res["ms_per_evaluation_karras"] = {k: {"median": statistics.median(v) / eval_cfgs[k][2], "min": min(v) / eval_cfgs[k][2],
                                           "max": max(v) / eval_cfgs[k][2], "evaluations": eval_cfgs[k][2]} for k, v in ms.items()}
    image2_cfgs = {"dpmpp_2m_sde_karras_20_cfg": (Schedule("dpmpp_2m_sde", "karras", 20), 20, 20),
                   "unipc_karras_20_cfg": (Schedule("unipc", "karras", 20), 20, 20),
                   "heun_karras_10_cfg": (Schedule("heun_discrete", "karras", 10), 10, 19)}
    ms = rounds(image2_cfgs)
    res["ms_per_image"].update({k: {"median": statistics.median(v), "min": min(v), "max": max(v), "unet_steps": image2_cfgs[k][2]}
                                for k, v in ms.items()})

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
    xs, h2 = torch.zeros(lat, device=dev), torch.zeros(lat, device=dev)
    for name, coef, rows, flags in (("unipc_corrected_two_row", (0.0, 0.4, 0.6, 0.3, -0.2, 0.0, 0.5), (0.0, 0.9, 0.2, 0.5, -0.1), (True, True, True)),
                                    ("heun_stage2_two_row", (0.2, 1.1, -0.2, -0.1, 0.0, 0.0, 0.5), (0.0,) * 5, (False, False, False)),
                                    ("sde_3m_two_row_in_kernel_noise", (0.9, 0.0, 0.1, -0.05, 0.02, 0.3, 0.5), (0.0,) * 5, (True, False, True))):
        run = lambda: _testing.guided_step_rows(eps, 4, 1, 4, (HW // 8) ** 2, True, False, 7.5, 0.0, 1.0, coef, rows, xh, x_in, hist=hist,  # noqa: E731
                                                h2=h2, xs=xs, write_hist=flags[0], write_xs=flags[1], shift=flags[2], seed=1)
        for _ in range(20):
            run()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(200):
            run()
        e1.record()
        e1.synchronize()
        res["step_kernel_us"][name] = e0.elapsed_time(e1) / 200 * 1e3
    d.close()
    ctx.close()
    sb.report(res, out_path)


if __name__ == "__main__":
    main()
