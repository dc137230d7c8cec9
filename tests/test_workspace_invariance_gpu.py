"""No engine path reads device memory it has not written, and CUDA graphs and PDL change no result.

tests/invariance_worker.py runs one fixed list of workloads (tiny UNet forwards at every test shape, DDIM and every scheduled
sampler with and without CFG, inpainting, the refiner, the inpainting UNet, each attachment alone, a LoRA merge and restore, the
VAE, both text encoders, the vision encoder, and at full size an SDXL-base CFG forward at 832 x 1216 and an SDXL VAE decode) and
saves every output. The library reads its switches once per process, so each configuration is one subprocess:

  base   nothing set: the reference run; every output must be finite.
  nan    SDXL_B200_FILL=0xff (NaN in f16 and f32) and torch's NaN fill of the tensors the Python wrappers allocate: a read of
         unwritten memory that reaches an output, including 0 * stale, turns it into NaN.
  big    SDXL_B200_FILL=0x7b (f16 61280, f32 1.3e36): reads that a NaN would hide, such as fmaxf(NaN, x) = x in a max reduction.
  eager  SDXL_B200_NO_GRAPH=1: a value captured into a CUDA graph that should have been read from device memory.
  nopdl  SDXL_B200_NO_PDL=1: results that depend on the overlap of programmatic dependent launches in this run.

Each configuration must reproduce every base output bit for bit. Inside each process the third run of every call (a graph replay)
must equal the first (eager)."""
import os
import subprocess
import sys

import pytest
import torch

from harness import first_difference

pytestmark = pytest.mark.gpu
WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "invariance_worker.py")
SWITCHES = ("SDXL_B200_FILL", "SDXL_B200_NO_GRAPH", "SDXL_B200_NO_PDL")
CONFIGS = {
    "base": ({}, []),
    "nan": ({"SDXL_B200_FILL": "0xff"}, ["--torch-nan"]),
    "big": ({"SDXL_B200_FILL": "0x7b"}, []),
    "eager": ({"SDXL_B200_NO_GRAPH": "1"}, []),
    "nopdl": ({"SDXL_B200_NO_PDL": "1"}, []),
}


def run_worker(name, out_dir):
    env_set, args = CONFIGS[name]
    env = {k: v for k, v in os.environ.items() if k not in SWITCHES}
    env.update(env_set)
    out = os.path.join(out_dir, f"{name}.pt")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [WORKER, out] + args
    p = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, f"worker [{name}] exited with {p.returncode}:\n{p.stderr[-6000:]}"
    res = torch.load(out, weights_only=True)
    want_fill = int(env_set["SDXL_B200_FILL"], 0) if "SDXL_B200_FILL" in env_set else -1
    assert res["fill"] == want_fill, f"[{name}] sdxl_debug_fill() = {res['fill']}, expected {want_fill}"
    return res["outputs"]


@pytest.fixture(scope="module")
def base(tmp_path_factory):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    outs = run_worker("base", str(tmp_path_factory.mktemp("invariance")))
    bad = [k for k, v in outs.items() if v.is_floating_point() and not bool(torch.isfinite(v).all())]
    assert not bad, f"base run: non-finite outputs {bad}"
    return outs


@pytest.mark.parametrize("config", ["nan", "big", "eager", "nopdl"])
def test_outputs_bit_identical_to_base(base, config, tmp_path):
    outs = run_worker(config, str(tmp_path))
    assert sorted(outs) == sorted(base), f"[{config}] the workload list differs from the base run's"
    diffs = [f"{k}: {first_difference(base[k], outs[k])}" for k in base if not torch.equal(base[k], outs[k])]
    print(f"[{config}] {len(base)} outputs, {len(diffs)} differ from base")
    assert not diffs, f"[{config}] {len(diffs)} of {len(base)} outputs differ from base; first: " + "\n".join(diffs[:12])
