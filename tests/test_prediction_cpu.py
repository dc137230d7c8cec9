"""v prediction, zero-terminal SNR and guidance rescale (DESIGN.md §18), host side: the float32 noise table against its float64
restatement, the oracle's v chains against its epsilon chains on an epsilon model wrapped as a v model, guidance rescale 0 as the plain
chain, the scheduler-config parsing of Diffuser.from_diffusers_dir, and the C ABI."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from sdxl_b200 import _lib
from sdxl_b200.schedulers import alphas_cumprod, prediction_of_config
import prediction_oracle as PR
import scheduler_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_zero_snr_table():
    got = alphas_cumprod(1000, zero_terminal_snr=True)
    want = PR.zero_snr_alphas(1000)
    assert got.dtype == np.float64 and got.shape == (1000,)
    assert got[-1] == 2.0 ** -24 and want[-1] == 2.0 ** -24
    # float32, as diffusers computes it: sqrt(alpha_bar) - sqrt(alpha_bar_T) rounds to within a few float32 ulps of 1, so the table
    # is within 1e-6 of the float64 restatement in sqrt(alpha_bar), and within 1e-6 relative only while alpha_bar is not small
    assert float(np.max(np.abs(np.sqrt(got) - np.sqrt(want)))) <= 1e-6
    assert float(np.max(np.abs(got / want - 1.0)[want > 0.25])) <= 1e-6
    assert np.all(np.diff(got) < 0) and np.all((got > 0) & (got < 1))
    s = PR.zero_snr_sqrt_alphas(1000)
    assert s[-1] == 0.0 and s[0] == math.sqrt(1.0 - 0.00085)
    plain = alphas_cumprod(1000)   # without the rescale: the epsilon table, in float32
    assert float(np.max(np.abs(plain / SO.sdxl_alphas(1000) - 1.0))) <= 1e-6


def _eps_model(x, t):
    """An analytic epsilon model, smooth in x and t."""
    return torch.tanh(x) * 0.5 + 0.1 * math.sin(0.01 * float(t)) * x


def test_v_wrapped_eps_model_is_the_eps_ddim_chain():
    alphas = PR.zero_snr_alphas(1000)
    x = torch.randn(2, 4, 8, 8, generator=torch.Generator().manual_seed(0), dtype=torch.float64)

    def v_model(x, t):   # v = sqrt(a) eps - sqrt(1 - a) x0 of the epsilon model at the same input
        a = float(alphas[t])
        e = _eps_model(x, t)
        x0 = (x - math.sqrt(1 - a) * e) / math.sqrt(a)
        return math.sqrt(a) * e - math.sqrt(1 - a) * x0
    for n in (4, 10):
        want = PR.ddim(_eps_model, alphas, x, n, v=False)
        got = PR.ddim(v_model, alphas, x, n, v=True)
        assert float((got - want).norm() / want.norm()) <= 1e-10


@pytest.mark.parametrize("sampler, spacing", [("euler", "trailing"), ("euler_ancestral", "trailing"), ("dpmpp_2m", "karras"),
                                               ("lcm", "lcm")])
def test_v_wrapped_eps_model_is_the_eps_scheduled_chain(sampler, spacing):
    alphas = PR.zero_snr_alphas(1000)
    t, sig = SO.schedule(spacing, 5, alphas)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 4, 8, 8, generator=g, dtype=torch.float64) * (sig[0] ** 2 + 1) ** 0.5
    noise = [torch.randn(2, 4, 8, 8, generator=g, dtype=torch.float64) for _ in range(5)]

    def v_model(x_in, tk):   # x_in is the VP latent at alpha_bar = 1 / (sigma^2 + 1)
        a = 1.0 / (SO.sigma_of_t(SO.log_sigmas(alphas), tk) ** 2 + 1.0)
        e = _eps_model(x_in, tk)
        x0 = (x_in - math.sqrt(1 - a) * e) / math.sqrt(a)
        return math.sqrt(a) * e - math.sqrt(1 - a) * x0
    it = iter(noise)
    want = SO.sample(_eps_model, sampler, t, sig, x, lambda: next(it), where=torch.where)
    it = iter(noise)
    got = PR.sample(v_model, sampler, t, sig, x, lambda: next(it), v=True)
    assert float((got - want).norm() / want.norm()) <= 1e-10
    it = iter(noise)
    assert torch.equal(PR.sample(_eps_model, sampler, t, sig, x, lambda: next(it), v=False), want)


def test_rescale_zero_is_the_plain_guidance():
    g = torch.randn(2, 4, 8, 8, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    c = g * 0.3 + 1.0
    assert torch.equal(PR.rescale_noise_cfg(g, c, 0.0), g)
    r = PR.rescale_noise_cfg(g, c, 1.0)
    for b in range(2):   # phi = 1: the guided output takes the conditional output's std
        assert abs(float(r[b].std() / c[b].std()) - 1.0) <= 1e-12
    assert torch.equal(PR.rescale_noise_cfg(torch.ones(1, 3, 2, 2, dtype=torch.float64), c[:1, :3, :2, :2], 0.7),
                       torch.ones(1, 3, 2, 2, dtype=torch.float64))   # std(g) = 0: the ratio is 1


SD = dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", num_train_timesteps=1000)


def test_scheduler_config_parsing():
    assert prediction_of_config(dict(SD, prediction_type="epsilon")) is None
    assert prediction_of_config({}) is None
    assert prediction_of_config(dict(SD, beta_schedule="linear")) is None   # epsilon on the loaded table: the file's betas are unused
    p = prediction_of_config(dict(SD, prediction_type="v_prediction", rescale_betas_zero_snr=True, timestep_spacing="trailing"))
    assert p["prediction"] == "v_prediction" and p["zero_terminal_snr"]
    assert np.array_equal(p["alphas"], alphas_cumprod(1000, 0.00085, 0.012, True))
    p = prediction_of_config(dict(SD, prediction_type="v_prediction"))
    assert not p["zero_terminal_snr"] and np.array_equal(p["alphas"], alphas_cumprod(1000))
    p = prediction_of_config(dict(SD, rescale_betas_zero_snr=True, beta_end=0.02))
    assert p["prediction"] == "epsilon" and np.array_equal(p["alphas"], alphas_cumprod(1000, 0.00085, 0.02, True))
    with pytest.raises(_lib.SdxlError, match="prediction_type"):
        prediction_of_config(dict(SD, prediction_type="sample"))
    with pytest.raises(_lib.SdxlError, match="beta_schedule"):
        prediction_of_config(dict(SD, prediction_type="v_prediction", beta_schedule="linear"))
    with pytest.raises(_lib.SdxlError, match="beta_schedule"):
        prediction_of_config(dict(rescale_betas_zero_snr=True))   # diffusers' default schedule is linear


def test_prediction_abi_from_c(tmp_path):
    """A C99 program using the prediction part of include/sdxl_b200.h compiles with -pedantic -Werror, links and sees the layout."""
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib_dir = os.path.join(ROOT, "stable-diffusion-xl-burn_b200", "sdxl_b200")
    exe = str(tmp_path / "prediction_abi_check")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "c_abi", "prediction_abi_check.c"), "-L", lib_dir, "-lsdxl_b200", "-Wl,-rpath," + lib_dir,
                        "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout.startswith("prediction_abi_check ok"), (r.returncode, r.stdout, r.stderr)
    assert int(r.stdout.split()[-1]) == C.sizeof(_lib.Prediction)
