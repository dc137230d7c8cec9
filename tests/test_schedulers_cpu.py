"""Samplers and noise schedules, host side: sdxl_schedule_build and the coefficient function against the float64 oracle of
tests/scheduler_oracle.py, the oracle itself against closed-form ODE solutions and the DDIM update of oracle/unet_oracle.py,
the refusals and the C ABI."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

from sdxl_b200 import SdxlError, _lib, schedulers
from sdxl_b200.schedulers import SAMPLERS, SPACINGS, Schedule
import scheduler_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1000


def legal(spacing, n):
    return not (spacing == "leading" and (n - 1) * (N // n) + 1 > N - 1) and not (spacing == "lcm" and n > 50)


@pytest.mark.parametrize("f16", [False, True])
@pytest.mark.parametrize("spacing", sorted(SPACINGS))
def test_schedule_build_equals_the_oracle(spacing, f16):
    a = SO.sdxl_alphas(N, f16)
    ls = SO.log_sigmas(a)
    assert bool((np.diff(ls) > 0).all())
    for n in (1, 2, 4, 20, 30, 1000):
        if not legal(spacing, n):
            with pytest.raises(SdxlError, match="n_steps"):
                schedulers.build(a, Schedule("euler", spacing, n))
            continue
        t, sig = schedulers.build(a, Schedule("euler", spacing, n))
        wt, ws = SO.schedule(spacing, n, a)
        assert t.shape == (n,) and sig.shape == (n + 1,) and sig[n] == 0.0
        np.testing.assert_allclose(sig, ws, rtol=1e-12, atol=0)
        np.testing.assert_allclose(t, wt, rtol=1e-12, atol=1e-9)   # t = 0 of a Karras schedule is a difference of equal logs
        assert bool((np.diff(sig) < 0).all())
        for tk, sk in zip(t, sig):   # t <-> sigma round trip
            assert abs(SO.t_of_sigma(ls, sk) - tk) <= 1e-9 * max(1.0, tk)
            assert abs(SO.sigma_of_t(ls, tk) - sk) <= 1e-12 * sk


def test_karras_rho_and_known_points():
    a = SO.sdxl_alphas(N)
    t, sig = schedulers.build(a, Schedule("euler", "karras", 10, karras_rho=5.0))
    np.testing.assert_allclose(sig, SO.schedule("karras", 10, a, rho=5.0)[1], rtol=1e-12)
    smax = math.sqrt((1 - a[-1]) / a[-1])
    assert abs(sig[0] - smax) <= 1e-12 * smax and abs(t[0] - 999.0) < 1e-9 and abs(t[-1]) < 1e-9
    # values from the formulas of the spacings, worked by hand for n = 4
    assert list(schedulers.build(a, Schedule("euler", "reference", 4))[0]) == [999, 749, 499, 249]
    assert list(schedulers.build(a, Schedule("euler", "leading", 4))[0]) == [751, 501, 251, 1]
    assert list(schedulers.build(a, Schedule("euler", "trailing", 4))[0]) == [999, 749, 499, 249]
    np.testing.assert_allclose(schedulers.build(a, Schedule("euler", "linspace", 4))[0], [999, 666, 333, 0], rtol=1e-14)
    np.testing.assert_allclose(schedulers.build(a, Schedule("euler", "linspace", 3))[0], [999, 499.5, 0], rtol=1e-14)
    assert list(schedulers.build(a, Schedule("euler", "lcm", 4))[0]) == [999, 759, 499, 259]
    assert list(schedulers.build(a, Schedule("euler", "trailing", 16))[0][:4]) == [999, 937, 874, 811]   # 937.5 and 812.5 round to even


# ---- the oracle, pinned by things that are not samplers --------------------------------------------------------------------
def gaussian_eps(s_data):
    """Data ~ N(0, s^2 I): the ideal noise prediction of the VP-scaled input at sigma is sigma * xh / (sigma^2 + s^2)."""
    def make(sig_of_t):
        def f(x_in, t):
            sigma = sig_of_t[t]
            xh = x_in * (sigma ** 2 + 1) ** 0.5
            return sigma * xh / (sigma ** 2 + s_data ** 2)
        return f
    return make


def ode_error(sampler, n, s_data=0.7):
    a = SO.sdxl_alphas(N)
    t, sig = SO.schedule("karras", n, a)
    x0 = np.array([1.0, -2.0, 0.5]) * (sig[0] ** 2 + 1) ** 0.5
    f = gaussian_eps(s_data)({tk: sk for tk, sk in zip(t, sig)})
    got = SO.sample(f, sampler, t, sig, x0, k1=n - 1)   # to sigma_{n-1} = sigma_min: the exact solution is known at every sigma
    want = x0 * ((sig[n - 1] ** 2 + s_data ** 2) / (sig[0] ** 2 + s_data ** 2)) ** 0.5
    return float(np.abs(got - want).max() / np.abs(want).max())


def test_orders_of_convergence():
    ns = [10, 20, 40, 80, 160]
    slope = {}
    for sampler in ("euler", "dpmpp_2m"):
        err = [ode_error(sampler, n) for n in ns]
        slope[sampler] = np.polyfit(np.log(ns), np.log(err), 1)[0]
        print(sampler, "errors", ["%.2e" % e for e in err], "slope %.2f" % slope[sampler])
    assert -1.25 < slope["euler"] < -0.8
    assert -2.4 < slope["dpmpp_2m"] < -1.7


def test_euler_ancestral_and_lcm_recurrences():
    a = SO.sdxl_alphas(N)
    t, sig = SO.schedule("trailing", 6, a)
    x0 = np.array([0.3, -1.1]) * (sig[0] ** 2 + 1) ** 0.5
    f = gaussian_eps(0.5)({tk: sk for tk, sk in zip(t, sig)})
    eul = SO.sample(f, "euler", t, sig, x0)
    never = lambda: (_ for _ in ()).throw(AssertionError("no noise with eta = 0"))   # noqa: E731
    assert np.array_equal(SO.sample(f, "euler_ancestral", t, sig, x0, draw=never, eta=0.0), eul)
    # with noise: each step lands on the Euler step to sigma_down plus s_noise * sigma_up * z (Karras et al., Algorithm 2's split)
    zs = [np.array([0.1 * (i + 1), -0.2]) for i in range(5)]
    it = iter(zs)
    x = x0
    for k in range(6):
        s, sn = sig[k], sig[k + 1]
        D = x - s * f(x / (s * s + 1) ** 0.5, t[k])
        up = min(sn, (sn * sn * (s * s - sn * sn) / (s * s)) ** 0.5)
        down = (sn * sn - up * up) ** 0.5
        x = D + (x - D) * (down / s) + (next(it) * up if sn > 0 else 0.0)
    it = iter(zs)
    np.testing.assert_allclose(SO.sample(f, "euler_ancestral", t, sig, x0, draw=lambda: next(it)), x, rtol=1e-13)
    # LCM: the consistency function's output re-noised to the next sigma; c_skip is ~0 away from t = 0
    it = iter(zs)
    x = x0
    for k in range(6):
        s, sn = sig[k], sig[k + 1]
        D = x - s * f(x / (s * s + 1) ** 0.5, t[k])
        ts = 10 * t[k]
        den = ts / (ts * ts + 0.25) ** 0.5 * D + 0.25 / (ts * ts + 0.25) * x / (s * s + 1) ** 0.5
        x = den + (sn * next(it) if sn > 0 else 0.0)
    it = iter(zs)
    np.testing.assert_allclose(SO.sample(f, "lcm", t, sig, x0, draw=lambda: next(it)), x, rtol=1e-13)


@pytest.mark.parametrize("spacing, n", [("reference", 10), ("leading", 7), ("trailing", 16), ("lcm", 4)])
def test_euler_is_the_ddim_update(spacing, n):
    """On integer timesteps Euler in the xh scaling is oracle/unet_oracle.py's DDIM update (diffuse_latent) in the VP scaling."""
    import torch
    from oracle import unet_oracle as O
    a = SO.sdxl_alphas(N, f16=True)
    t, sig = SO.schedule(spacing, n, a)
    rng = np.random.default_rng(0)
    x = rng.standard_normal(8)
    xh = x * (sig[0] ** 2 + 1) ** 0.5
    alphas = torch.tensor(a)
    for k in range(n):
        e = np.sin(3 * x + k)   # any prediction
        ca = O.get_alpha(alphas, int(t[k]))
        pa = O.get_alpha(alphas, int(t[k + 1])) if k + 1 < n else 1.0
        predx0 = (x - e * math.sqrt(1 - ca)) / math.sqrt(ca)
        x = predx0 * math.sqrt(pa) + e * math.sqrt(1 - pa)
        xh = SO.step("euler", k, t, sig, xh, xh - sig[k] * e)
        np.testing.assert_allclose(xh / (sig[k + 1] ** 2 + 1) ** 0.5, x, rtol=1e-12, atol=1e-13)


# ---- the engine's coefficient function --------------------------------------------------------------------------------------
def test_step_coefficients_equal_the_oracle():
    from sdxl_b200 import _testing
    lib = _testing.load()
    a = SO.sdxl_alphas(N, f16=True)
    worst = 0.0
    for sampler in sorted(SAMPLERS):
        for spacing, n in (("karras", 5), ("trailing", 4), ("leading", 10), ("lcm", 4), ("linspace", 1)):
            for eta, s_noise in ((0.0, 0.0), (0.6, 1.1)):
                sch = Schedule(sampler, spacing, n, eta=eta, s_noise=s_noise)
                t, sig = schedulers.build(a, sch)
                s = sch.to_struct()
                for k in range(n):
                    for has_prev in (0, 1):
                        out = (C.c_float * 5)()
                        lib.sdxl_test_step_coef(C.byref(s), k, t.ctypes.data, sig.ctypes.data, has_prev, out)
                        want = SO.coefficients(sampler, k, t, sig, bool(has_prev) and k > 0, eta or 1.0, s_noise or 1.0)
                        assert all(math.isfinite(v) for v in out)
                        for g, w in zip(out, want):
                            assert g == np.float32(w) or abs(g - w) <= 2e-7 * max(abs(w), 1e-3), (sampler, spacing, k, has_prev, list(out), want)
                            worst = max(worst, abs(g - w) / max(abs(w), 1e-3))
                if sampler != "lcm":   # the step to sigma = 0 returns the denoised latent exactly
                    lib.sdxl_test_step_coef(C.byref(s), n - 1, t.ctypes.data, sig.ctypes.data, 1, out)
                    assert list(out) == [0.0, 1.0, 0.0, 0.0, 1.0]
    print(f"step coefficients: worst relative difference {worst:.2e}")


# ---- refusals, Python surface, C ABI ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw, field", [
    (dict(n_steps=0), "n_steps"), (dict(n_steps=1001), "n_steps"), (dict(first_step=4), "first_step"), (dict(first_step=-1), "first_step"),
    (dict(last_step=5), "last_step"), (dict(first_step=2, last_step=2), "first_step"), (dict(renoise=True), "renoise"),
    (dict(karras_rho=-1.0), "karras_rho"), (dict(eta=float("nan")), "eta"), (dict(s_noise=-2.0), "s_noise"),
    (dict(spacing="lcm", n_steps=51), "n_steps"), (dict(spacing="leading", n_steps=1000), "n_steps"),
])
def test_invalid_schedules_name_the_field(kw, field):
    a = SO.sdxl_alphas(N)
    args = dict(sampler="euler", spacing="karras", n_steps=4)
    args.update(kw)
    with pytest.raises(SdxlError, match=field):
        schedulers.build(a, Schedule(**args))


def test_invalid_enums_and_tables():
    lib = _lib.load()
    a = SO.sdxl_alphas(N)
    t, sig = np.zeros(4), np.zeros(5)
    for field, v in (("sampler", 4), ("sampler", -1), ("spacing", 6), ("no_cfg", 2), ("renoise", 3)):
        s = Schedule("euler", "karras", 4).to_struct()
        setattr(s, field, v)
        assert lib.sdxl_schedule_build(a.ctypes.data, N, C.byref(s), t.ctypes.data, sig.ctypes.data) != 0
        assert field in lib.sdxl_schedule_last_error().decode()
    s = Schedule("euler", "karras", 4).to_struct()
    bad = a.copy()
    bad[10] = bad[9]
    assert lib.sdxl_schedule_build(bad.ctypes.data, N, C.byref(s), t.ctypes.data, sig.ctypes.data) != 0
    assert "alphas_cumprod[10]" in lib.sdxl_schedule_last_error().decode()
    assert lib.sdxl_schedule_build(None, N, C.byref(s), t.ctypes.data, sig.ctypes.data) != 0
    with pytest.raises(SdxlError, match="sampler"):
        Schedule("heun", "karras", 4).to_struct()


def test_from_strength_and_noise_count():
    """diffusers' img2img: init_timestep = min(int(n * strength), n) steps run."""
    assert Schedule.from_strength(30, 1.0).first_step == 0 and not Schedule.from_strength(30, 1.0).renoise
    s = Schedule.from_strength(30, 0.3, sampler="euler_ancestral", spacing="karras")
    assert (s.first_step, s.renoise, s.sampler, s.spacing) == (21, True, "euler_ancestral", "karras")
    assert s.n_noise(initial=False) == 1 + 8 and s.n_noise(initial=False, inpainting=True) == 1 + 9 + 8
    assert Schedule("euler", "karras", 10).n_noise(initial=True) == 1
    assert Schedule("lcm", "lcm", 4, last_step=2).n_noise(initial=True) == 3
    with pytest.raises(SdxlError, match="strength"):
        Schedule.from_strength(30, 0.01)


def test_scheduler_abi_from_c(tmp_path):
    """A C99 program using the schedule part of include/sdxl_b200.h compiles with -pedantic -Werror, links, builds a schedule
    without a GPU and sees the layout."""
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib_dir = os.path.join(ROOT, "stable-diffusion-xl-burn_b200", "sdxl_b200")
    exe = str(tmp_path / "scheduler_abi_check")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "c_abi", "scheduler_abi_check.c"), "-L", lib_dir, "-lsdxl_b200", "-Wl,-rpath," + lib_dir,
                        "-lm", "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout.startswith("scheduler_abi_check ok"), (r.returncode, r.stdout, r.stderr)
    assert int(r.stdout.split()[-1]) == C.sizeof(_lib.Schedule)
