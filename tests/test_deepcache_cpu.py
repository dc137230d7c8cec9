"""DeepCache, host side: the oracle's cached forward right after a full forward on the same inputs is the full forward for every
branch, interval 1 is the plain oracle chains, and the C ABI."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import sdxl_b200
from sdxl_b200 import TINY, TINY_CONTROLNET, TINY_REFINER, _lib, synth_weights
from oracle import unet_oracle as O
import deepcache_oracle as DO
import freeu_oracle as FO
import scheduler_oracle as SO
from harness import h16f, tiny_conditioning

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_W = {}


def _weights(cfg, seed):
    if (cfg, seed) not in _W:
        _W[(cfg, seed)] = O.to_f32(synth_weights(cfg, seed=seed))
    return _W[(cfg, seed)]


def _inputs(cfg, seed=1):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(2, 4, 16, 16, generator=g), torch.tensor([499]), h16f(torch.randn(2, 7, cfg.context_dim, generator=g)),
            h16f(torch.randn(2, cfg.adm_in_channels, generator=g)))


@pytest.mark.parametrize("cfg, seed", [(TINY, 0), (TINY_REFINER, 1)], ids=["tiny", "tiny_refiner"])
@pytest.mark.parametrize("freeu", [None, FO.RECOMMENDED_SDXL], ids=["plain", "freeu"])
def test_cached_after_full_is_full(cfg, seed, freeu):
    """The full forward is unet_oracle's, and the cached forward on the feature it kept, at the same inputs, equals it for every
    branch; with FreeU the feature is the tensor before FreeU scales it."""
    w = _weights(cfg, seed)
    x, t, c, y = _inputs(cfg)
    att = O.Attach(freeu=freeu)
    plain = O.unet_forward(cfg, w, x, t, c, y, att)
    assert DO.n_branches(cfg) == 9
    for b in range(DO.n_branches(cfg)):
        full, feature = DO.unet_forward(cfg, w, x, t, c, y, att, b)
        cached, kept = DO.unet_forward(cfg, w, x, t, c, y, att, b, feature)
        assert torch.equal(full, plain) and kept is None
        assert torch.equal(cached, full), f"branch {b}"


def test_cached_with_controlnet_takes_the_shallow_residuals():
    w, wc = _weights(TINY, 0), _weights(TINY_CONTROLNET, 7)
    x, t, c, y = _inputs(TINY)
    hint = torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(4))
    att = O.Attach(controls=[(TINY_CONTROLNET, wc, hint, 0.8)])
    for b in (0, 4, 8):
        full, feature = DO.unet_forward(TINY, w, x, t, c, y, att, b)
        cached, _ = DO.unet_forward(TINY, w, x, t, c, y, att, b, feature)
        assert torch.equal(cached, full)
        assert not torch.equal(DO.unet_forward(TINY, w, x * 0.5, t, c, y, att, b, feature)[0], full)


def test_interval_1_is_the_plain_ddim_chains():
    w = _weights(TINY, 0)
    alphas = sdxl_b200.alphas_cumprod(TINY.n_steps)
    oc = O.OracleConditioning(**tiny_conditioning(refiner=True))
    noise = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(0))
    want = O.sample_latent(TINY, w, alphas, noise, oc, 7.5, 3)
    for b in (0, 5):
        assert torch.equal(DO.sample_latent(TINY, w, alphas, noise, oc, 7.5, 3, 1, b), want)
    assert not torch.equal(DO.sample_latent(TINY, w, alphas, noise, oc, 7.5, 3, 2, 0), want)
    wr = _weights(TINY_REFINER, 1)
    g = torch.Generator().manual_seed(5)
    latent, rn = torch.randn(2, 4, 16, 16, generator=g), torch.randn(2, 4, 16, 16, generator=g)
    want = O.refine_latent(TINY_REFINER, wr, alphas, latent, oc, 7.5, 990, 200, rn)
    assert torch.equal(DO.refine_latent(TINY_REFINER, wr, alphas, latent, oc, 7.5, 990, 200, rn, 1, 3), want)


def test_interval_1_is_the_plain_scheduled_chain():
    w = _weights(TINY, 0)
    alphas = sdxl_b200.alphas_cumprod(TINY.n_steps)
    a64 = np.array([O.get_alpha(alphas, i) for i in range(TINY.n_steps)])
    oc = O.OracleConditioning(**tiny_conditioning(refiner=True))
    t, sig = SO.schedule("karras", 3, a64)
    x = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(0)) * (sig[0] ** 2 + 1) ** 0.5

    def plain(x_in, tt):
        return O.forward_diffuser(TINY, w, x_in.float(), torch.tensor([float(tt)], dtype=torch.float32), oc, 7.5)
    want = SO.sample(plain, "dpmpp_2m", t, sig, x, None, 0, None, 1.0, 1.0, None, torch.where)
    got = SO.sample(DO.eps_fn(TINY, w, oc, 7.5, 1, 2), "dpmpp_2m", t, sig, x, None, 0, None, 1.0, 1.0, None, torch.where)
    assert torch.equal(got, want)


def test_deepcache_abi_from_c(tmp_path):
    """A C99 program using the DeepCache part of include/sdxl_b200.h compiles with -pedantic -Werror, links and sees the layout."""
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib_dir = os.path.join(ROOT, "stable-diffusion-xl-burn_b200", "sdxl_b200")
    exe = str(tmp_path / "deepcache_abi_check")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "c_abi", "deepcache_abi_check.c"), "-L", lib_dir, "-lsdxl_b200", "-Wl,-rpath," + lib_dir,
                        "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout.startswith("deepcache_abi_check ok"), (r.returncode, r.stdout, r.stderr)
    assert int(r.stdout.split()[-1]) == C.sizeof(_lib.Deepcache)
