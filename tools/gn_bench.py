#!/usr/bin/env python
"""GroupNorm (gn_launch: stats + apply) time per launch on the plans' GroupNorm shapes, CUDA events.

  python tools/gn_bench.py [out.json] [--reps R] [--rounds N] [--lib NAME=PATH ...]

Each --lib is a libsdxl_b200_testing.so (default: the in-tree one, named "tree"). With several, every round times every shape
with each library in turn (rotating which goes first), so two builds are compared in one process under the same conditions;
the reported figure is the median over rounds of the mean time per launch. Shapes: the SDXL-base step's resnet / transformer
GroupNorms at 1024^2 (B = 2: the CFG batch) and the VAE decoder's at a 1024^2 image (B = 1), with the number of times one
step (or one decode) runs each, so the per-step and per-decode GroupNorm totals follow. Prints the card's name, power limit
and SM clock beside the numbers.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_LIB = os.path.join(ROOT, "stable-diffusion-xl-burn_b200", "sdxl_b200", "libsdxl_b200_testing.so")

# (label, B, HW, C1, C2, silu, launches per UNet forward / per decode): block_program's resnet GroupNorms (two each, the first
# on the skip concatenation in the decoder), one per transformer, the output head; the VAE decoder's mid block (two resnets and
# the attention), four up blocks of three resnets and norm_out
UNET = [("unet 320 @128^2", 2, 16384, 320, 0, 1, 8), ("unet 320+320 @128^2", 2, 16384, 320, 320, 1, 2),
        ("unet 640+320 @128^2", 2, 16384, 640, 320, 1, 1), ("unet 320 @64^2", 2, 4096, 320, 0, 1, 1),
        ("unet 640 @64^2", 2, 4096, 640, 0, 1, 11), ("unet 640+320 @64^2", 2, 4096, 640, 320, 1, 1),
        ("unet 640+640 @64^2", 2, 4096, 640, 640, 1, 1), ("unet 1280+640 @64^2", 2, 4096, 1280, 640, 1, 1),
        ("unet 640 @32^2", 2, 1024, 640, 0, 1, 1), ("unet 1280 @32^2", 2, 1024, 1280, 0, 1, 16),
        ("unet 1280+640 @32^2", 2, 1024, 1280, 640, 1, 1), ("unet 1280+1280 @32^2", 2, 1024, 1280, 1280, 1, 2)]
VAE = [("vae 512 @128^2", 1, 16384, 512, 0, 1, 11), ("vae 512 @256^2", 1, 65536, 512, 0, 1, 6),
       ("vae 512 @512^2", 1, 262144, 512, 0, 1, 1), ("vae 256 @512^2", 1, 262144, 256, 0, 1, 5),
       ("vae 256 @1024^2", 1, 1048576, 256, 0, 1, 1), ("vae 128 @1024^2", 1, 1048576, 128, 0, 1, 6)]


def load(path):
    lib = C.CDLL(path)
    P, I = C.c_void_p, C.c_int
    lib.sdxl_test_gn.restype = I
    lib.sdxl_test_gn.argtypes = [P, P, I, P, I, I, I, I, P, P, C.c_float, I, P, P, P, P]
    lib.sdxl_test_gn_scratch_floats.restype = C.c_size_t
    lib.sdxl_test_gn_scratch_floats.argtypes = [I, I]
    lib.sdxl_test_gn_scratch_init.restype = I
    lib.sdxl_test_gn_scratch_init.argtypes = [P, P, I, I]
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out", nargs="?", default=None)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "gn_bench needs a GPU"
    libs = {}
    for spec in args.lib or [f"tree={DEFAULT_LIB}"]:
        name, path = spec.split("=", 1)
        libs[name] = load(path)
    names = list(libs)
    dev = torch.device("cuda")
    stream = torch.cuda.current_stream().cuda_stream
    scratch = {n: torch.empty(libs[n].sdxl_test_gn_scratch_floats(2, 32), dtype=torch.float32, device=dev) for n in names}
    for n in names:
        assert libs[n].sdxl_test_gn_scratch_init(stream, scratch[n].data_ptr(), 2, 32) == 0
    shapes = UNET + VAE
    g = torch.Generator(device=dev).manual_seed(0)
    times = {n: {s[0]: [] for s in shapes} for n in names}
    for label, B, HW, C1, C2, silu, _ in shapes:
        x1 = torch.randn(B, HW, C1, generator=g, device=dev)
        x2 = torch.randn(B, HW, C2, generator=g, device=dev) if C2 else None
        Cc = C1 + C2
        gam, bet = torch.ones(Cc, device=dev), torch.zeros(Cc, device=dev)
        y = torch.empty(B, HW, Cc, dtype=torch.float16, device=dev)

        def launch(n):
            rc = libs[n].sdxl_test_gn(stream, x1.data_ptr(), C1, x2.data_ptr() if x2 is not None else None, C2, B, HW, 32,
                                      gam.data_ptr(), bet.data_ptr(), 1e-5, silu, y.data_ptr(), None, None, scratch[n].data_ptr())
            assert rc == 0, f"{n} {label}: gn returned {rc}"

        for n in names:          # warm-up
            for _ in range(5):
                launch(n)
        torch.cuda.synchronize()
        for r in range(args.rounds):
            order = names[r % len(names):] + names[:r % len(names)]
            for n in order:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.reps):
                    launch(n)
                e1.record()
                e1.synchronize()
                times[n][label].append(e0.elapsed_time(e1) * 1e3 / args.reps)
        del x1, x2, y
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "reps": args.reps, "rounds": args.rounds, "us_per_launch": {}, "totals_us": {}}
    print(f"# {smi}")
    print(f"{'shape':24s} " + " ".join(f"{n + ' us (min..max)':>26s}" for n in names))
    for label, B, HW, C1, C2, silu, cnt in shapes:
        row = []
        for n in names:
            t = times[n][label]
            res["us_per_launch"].setdefault(n, {})[label] = {"median": statistics.median(t), "min": min(t), "max": max(t)}
            row.append(f"{statistics.median(t):9.2f} ({min(t):7.2f}..{max(t):7.2f})")
        print(f"{label:24s} " + " ".join(f"{c:>26s}" for c in row))
    for n in names:
        per = res["us_per_launch"][n]
        res["totals_us"][n] = {"unet_step_x_count": sum(per[s[0]]["median"] * s[6] for s in UNET),
                               "vae_decode_x_count": sum(per[s[0]]["median"] * s[6] for s in VAE)}
        print(f"{n}: GroupNorm per UNet forward (B = 2) {res['totals_us'][n]['unet_step_x_count']:.1f} us, "
              f"per VAE decode {res['totals_us'][n]['vae_decode_x_count']:.1f} us")
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    sys.exit(main())
