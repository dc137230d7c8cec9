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
from sdxl_b200 import _testing  # noqa: E402
from sdxl_b200.schedulers import Schedule  # noqa: E402

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
    n, reps = opt("--steps", 10), max(opt("--reps", 3), 3)
    out_path = args[0] if args and not args[0].startswith("--") else None
    if not torch.cuda.is_available():
        raise SystemExit("sampler_bench: no CUDA device; there is nothing to measure without one")
    ctx = sdxl_b200.Context(0)
    dev = str(ctx.device)
    res = {"gpu": gpu_info(), "resolution": HW, "steps": n, "reps": reps}
    d = sdxl_b200.Diffuser(ctx, sdxl_b200.SDXL_BASE, sdxl_b200.build_pack(sdxl_b200.synth_weights(sdxl_b200.SDXL_BASE, seed=0, device=dev)))
    g = lambda s: torch.Generator().manual_seed(s)  # noqa: E731
    cond = sdxl_b200.Conditioning(
        context_full=torch.randn(1, 77, 2048, generator=g(1)).half(), unconditional_context_full=torch.randn(77, 2048, generator=g(2)).half(),
        channel_context=torch.randn(1, 2816, generator=g(3)).half(), unconditional_channel_context=torch.randn(2816, generator=g(4)).half(),
        resolution=(HW, HW))

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
    print(json.dumps(res, indent=1))
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
