"""Implicit-GEMM time per shape group of the SDXL base step, three ways side by side (DESIGN.md §6):

  warm     the group's GEMM launched alone, the same launch repeated (its weights stay in L2)
  cold     the same launch, with a 128 MB device buffer written before each timed launch (the weights come from HBM)
  in plan  the group's launches in one eager pass of the step's plan (profile_dump: CUDA events per launch)

Groups are (M tiles, N, K blocks) with the plan's N tile and epilogue; convolutions are timed alone as plain GEMMs of the same M,
N and K. Prints the card's name, power limit and median SM clock.

usage: python tools/gemm_inplan.py [out.json] [--reps R]
"""
import argparse
import csv
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "stable-diffusion-xl-burn_b200"))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def smi(fields):
    r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={fields}", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, timeout=30)
    return [v.strip() for v in r.stdout.strip().split(",")]


class ClockSampler:
    """SM clock every 100 ms while a measurement runs (nvidia-smi's own loop, stopped and reaped by stop())."""

    def __init__(self):
        self.p = None

    def start(self):
        self.p = subprocess.Popen(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=clocks.sm",
                                   "--format=csv,noheader,nounits", "-lms", "100"], stdout=subprocess.PIPE, text=True)

    def stop(self):
        self.p.terminate()
        out, _ = self.p.communicate(timeout=30)
        vals = [int(v) for v in out.split() if v.strip().isdigit()]
        return statistics.median(vals) if vals else None


def plan_groups(path):
    groups = {}
    with open(path) as f:
        for r in csv.DictReader(f):
            if r["kind"] != "igemm":
                continue
            key = (int(r["M_tiles"]), int(r["N"]), int(r["Kblocks"]), int(r["BN"]), int(r["mode"]), int(r["out_f32"]), int(r["res"]))
            g = groups.setdefault(key, {"launches": 0, "us": 0.0})
            g["launches"] += 1
            g["us"] += float(r["us"])
    return groups


def time_alone(key, reps, flush):
    from sdxl_b200 import _testing as T
    mt, N, kb, BN, mode, out_f32, res = key
    M, K = mt * 128, kb * 64
    g = torch.Generator(device="cuda").manual_seed(0)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.1).half()
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.1).half()
    bias = torch.randn(N, device="cuda", generator=g)
    if mode == 1:   # GEGLU: f16 [M, N / 2]
        out, ldo = torch.empty(M, N // 2, device="cuda", dtype=torch.float16), N // 2
    else:
        out, ldo = torch.empty(M, N, device="cuda", dtype=torch.float32 if out_f32 else torch.float16), N
    r = torch.randn(M, N, device="cuda", generator=g) if res else None
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * reps)]

    def launch():
        T.igemm(a, (1, 1, M, K), w, N, K, (M, 1, 1), [(0, 0, 0, 0, kb)], out, ldo, bias=bias, res=r, ldr=N if res else 0,
                mode=mode, geglu_bn=BN if mode == 1 else 0)

    for _ in range(5):
        launch()
    for i in range(reps):
        if flush is not None:
            flush.add_(1.0)   # 128 MB written through L2: evicts the weights
        else:
            torch.cuda._sleep(100000)   # keeps the device busy while the host enqueues, as the flush does: no launch-latency gap
        ev[2 * i].record()
        launch()
        ev[2 * i + 1].record()
    torch.cuda.synchronize()
    return statistics.median(ev[2 * i].elapsed_time(ev[2 * i + 1]) * 1e3 for i in range(reps))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", nargs="?", default=None)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "gemm_inplan.py measures on a GPU"
    import sdxl_b200
    name, plim, smax = smi("name,power.limit,clocks.max.sm")
    ctx = sdxl_b200.Context(0)
    cfg = sdxl_b200.SDXL_BASE
    pack = sdxl_b200.build_pack(sdxl_b200.synth_weights(cfg, seed=0, device="cuda"))
    d = sdxl_b200.Diffuser(ctx, cfg, pack)
    ctx.synchronize()
    del pack
    torch.cuda.empty_cache()
    sys.path.insert(0, ROOT)
    from bench import make_conditioning
    d.sampler_begin(make_conditioning(0, torch.device("cuda")), 7.5)
    d.sampler_set_latent(ctx.randn(4 * 128 * 128, seed=0, subsequence=0).reshape(1, 4, 128, 128))
    for _ in range(3):
        d.sampler_step(999, 966)
    ctx.synchronize()
    clk = ClockSampler()
    clk.start()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "ops.csv")
        d.profile_plan()                 # warm pass
        d.profile_dump(path)
        groups = plan_groups(path)
    flush = torch.zeros(32 << 20, device="cuda")   # 128 MB
    rows = []
    for key, g in sorted(groups.items(), key=lambda kv: -kv[1]["us"]):
        warm = time_alone(key, args.reps, None)
        cold = time_alone(key, args.reps, flush)
        rows.append({"M_tiles": key[0], "N": key[1], "Kblocks": key[2], "BN": key[3], "geglu": key[4] == 1, "f32_out": bool(key[5]),
                     "residual": bool(key[6]), "launches": g["launches"],
                     "alone_warm_us": warm, "alone_cold_us": cold, "in_plan_us": g["us"] / g["launches"]})
    sm_clock = clk.stop()
    d.close()
    ctx.close()
    head = {"gpu": name, "power_limit_w": float(plim), "max_sm_clock_mhz": int(smax), "median_sm_clock_mhz": sm_clock}
    print(f"{name}, power limit {plim} W, max SM clock {smax} MHz, median SM clock {sm_clock} MHz")
    print(f"{'M-tiles, N, K-blocks':>22} {'BN':>4} {'epilogue':>12} {'launches':>8} {'warm us':>8} {'cold us':>8} {'plan us':>8} "
          f"{'plan/warm':>9} {'plan/cold':>9} {'plan total us':>13}")
    tot = 0.0
    for r in rows:
        epi = "geglu" if r["geglu"] else ("f32" if r["f32_out"] else "f16") + ("+res" if r["residual"] else "")
        tot += r["in_plan_us"] * r["launches"]
        print(f"{r['M_tiles']:>6}, {r['N']:>5}, {r['Kblocks']:>6}  {r['BN']:>4} {epi:>12} {r['launches']:>8} {r['alone_warm_us']:>8.1f} "
              f"{r['alone_cold_us']:>8.1f} {r['in_plan_us']:>8.1f} {r['in_plan_us'] / r['alone_warm_us']:>9.2f} "
              f"{r['in_plan_us'] / r['alone_cold_us']:>9.2f} {r['in_plan_us'] * r['launches']:>13.0f}")
    print(f"all GEMMs in the plan: {tot:.0f} us")
    if args.out:
        with open(args.out, "w") as f:
            json.dump({**head, "groups": rows, "in_plan_total_us": tot}, f, indent=1)


if __name__ == "__main__":
    main()
