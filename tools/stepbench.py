"""What the *_bench.py scripts share: the command line, the card's name, power limit and clocks, SDXL base (synthetic weights) on
the device, its CFG conditioning at HW x HW, bench.py's step timing, rounds in rotating order and the JSON they print and write.

Importing this module puts the repository and the package on sys.path, so a script next to it can then import sdxl_b200."""
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


def options(**defaults):
    """`[out.json] [--name value ...]`: returns out.json (or None), then the value of each --name in the order of defaults, typed like
    its default."""
    args = sys.argv[1:]
    out_path = args[0] if args and not args[0].startswith("--") else None
    return (out_path, *(type(d)(args[args.index(f"--{k}") + 1]) if f"--{k}" in args else d for k, d in defaults.items()))


def gpu_info():
    try:
        q = "name,power.limit,clocks.max.sm,clocks.sm"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


def load_unet(ctx, cfg=sdxl_b200.SDXL_BASE):
    """cfg's UNet with synthetic weights (seed 0, drawn on the device), loaded on ctx."""
    return sdxl_b200.Diffuser(ctx, cfg, sdxl_b200.build_pack(sdxl_b200.synth_weights(cfg, seed=0, device=str(ctx.device))))


def conditioning():
    """SDXL base CFG conditioning at HW x HW, batch 1: context, unconditional context, label vector and unconditional label vector
    drawn from seeds 1 to 4."""
    g = lambda s: torch.Generator().manual_seed(s)  # noqa: E731
    return sdxl_b200.Conditioning(
        context_full=torch.randn(1, 77, 2048, generator=g(1)).half(), unconditional_context_full=torch.randn(77, 2048, generator=g(2)).half(),
        channel_context=torch.randn(1, 2816, generator=g(3)).half(), unconditional_channel_context=torch.randn(2816, generator=g(4)).half(),
        resolution=(HW, HW))


def run_steps(ctx, d, steps, warmup, begin=None):
    """bench.py's step time, ms per step: a seeded latent, `warmup` steps, then CUDA events around `steps` steps of the 30-step DDIM
    schedule. begin: a Conditioning to sampler_begin with (CFG 7.5) first; None steps on the sampler d has already begun."""
    if begin is not None:
        d.sampler_begin(begin, 7.5)
    h = HW // 8
    ts = sdxl_b200.ddim_timesteps(30)
    step_size = 1000 // 30

    def step(i):
        t = ts[i % len(ts)]
        d.sampler_step(t, t - step_size if t >= step_size else -1)

    d.sampler_set_latent(ctx.randn(4 * h * h, seed=0).reshape(1, 4, h, h))
    for i in range(warmup):
        step(i)
    ctx.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(ctx.stream)
    for i in range(steps):
        step(i)
    e1.record(ctx.stream)
    ctx.synchronize()
    return e0.elapsed_time(e1) / steps


def step_rounds(names, reps, run):
    """run(name) -> ms per step for every name in each of `reps` rounds, each round starting one name later than the last, so that
    a clock drifting during the run does not always fall on the same name. Returns name -> {"median", "runs"}."""
    runs = {k: [] for k in names}
    for r in range(reps):
        for k in names[r % len(names):] + names[:r % len(names)]:
            runs[k].append(round(run(k), 3))
    return {k: {"median": statistics.median(v), "runs": v} for k, v in runs.items()}


def timed(ctx, reps, fn, before=lambda: None):
    """Median of `reps` host wall-clock times, in ms, of fn() ending in a stream synchronise; before() is untimed set-up."""
    ts = []
    for _ in range(reps):
        before()
        ctx.synchronize()
        t0 = time.perf_counter()
        fn()
        ctx.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return round(statistics.median(ts), 2)


def report(res, out_path):
    """Prints res as one JSON line and writes it to out_path when one was given."""
    print(json.dumps(res), flush=True)
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
