"""DPM++ 2M SDE, DPM++ 3M SDE, UniPC, Heun and DPM2 (DESIGN.md §20), host side: the library's stage coefficients against the float64
recurrences of tests/scheduler2_oracle.py read off by linearity, the recurrences' orders of convergence on Gaussian data and the
SDE samplers' end variance, the noise count, the refusals, the C ABI, and the SASS of the step kernel's existing forms."""
import ctypes as C
import hashlib
import json
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from sdxl_b200 import SdxlError, _lib, _testing, schedulers
from sdxl_b200.schedulers import ALL_SAMPLERS, MORE_SAMPLERS, SAMPLERS, Schedule
import scheduler2_oracle as SO
import scheduler_oracle as SO1

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 1000
NEW = SO.SAMPLERS2
VARS = ("xh", "xs", "D", "H1", "H2", "z")


def close(g, w):
    return g == np.float32(w) or abs(g - w) <= 2e-7 * max(abs(w), 1e-3)


def oracle_step(sampler, k, t, sig, n_hist, ls, eta, s_noise, v):
    """One step of the oracle from the named inputs v (VARS; for Heun and DPM2 also X2 and D2, what the second evaluation sees and
    returns): (x', xs' of UniPC, the second evaluation's (x, sigma, t)). The call started n_hist steps before k."""
    Ds = [v["H2"], v["H1"]][2 - n_hist:]
    hist = {}
    if n_hist:
        hist = {"D": Ds, "h": [math.log(sig[j] / sig[j + 1]) for j in range(k - n_hist, k)],
                "lam": [-math.log(sig[j]) for j in range(k - n_hist, k)], "x_last": v["xs"] / (sig[k - 1] ** 2 + 1) ** 0.5,
                "order": min(2, n_hist, len(t) - k + 1)}
    seen = []

    def evaluate(x, s, tk):
        seen.append((x, s, tk))
        return v["X2"], v["D2"]
    x, hist = SO.step2(sampler, k, t, sig, v["xh"], v["D"], evaluate, hist, lambda: v["z"], eta, s_noise, ls)
    return x, hist.get("x_corrected"), seen


def unit(name, extra=()):
    v = {n: 0.0 for n in VARS + ("X2", "D2") + tuple(extra)}
    v[name] = 1.0
    return v


@pytest.mark.parametrize("sampler", NEW)
def test_stage_coefficients_equal_the_oracle(sampler):
    a = SO1.sdxl_alphas(N, f16=True)
    ls = SO1.log_sigmas(a)
    worst, checked = 0.0, 0
    for spacing, n in (("karras", 5), ("trailing", 4), ("leading", 10), ("lcm", 4), ("linspace", 1), ("karras", 12)):
        for eta, s_noise in ((0.0, 0.0), (0.6, 1.1)):
            sch = Schedule(sampler, spacing, n, eta=eta, s_noise=s_noise)
            t, sig = schedulers.build(a, sch)
            s = sch.to_struct()
            for k in range(n):
                for n_hist in range(0, min(k, 2) + 1):
                    st = _testing.step_stages(a, s, k, t, sig, n_hist)
                    O = lambda v: oracle_step(sampler, k, t, sig, n_hist, ls, eta or 1.0, s_noise or 1.0, v)   # noqa: E731
                    assert O({n: 0.0 for n in VARS + ("X2", "D2")})[0] == 0.0
                    two = sampler in ("heun_discrete", "dpm_2") and sig[k + 1] > 0
                    assert len(st) == (2 if two else 1), (sampler, k, st)
                    q = st[0]
                    assert (q["t"], q["sigma"]) == (t[k], sig[k])
                    if two:   # stage 1 lands where the second evaluation runs and saves xh (and D for Heun)
                        x2 = {n: O(unit(n))[2][0][0] for n in ("xh", "D")}
                        _, s2, t2 = O(unit("xh"))[2][0]
                        want = dict(cx=x2["xh"], cd=x2["D"], cs=0.0, ch=0.0, ch2=0.0, cn=0.0, sx=1.0, ss=0.0, sd=0.0, sh=0.0, sh2=0.0)
                        assert q["sigma_next"] == s2 and q["write_xs"] == 1 and q["hist"] == (1 if sampler == "heun_discrete" else 0)
                        q2 = st[1]
                        assert q2["sigma"] == s2 and abs(q2["t"] - t2) <= 1e-9 * max(t2, 1.0) and q2["sigma_next"] == sig[k + 1]
                        # stage 2 over (xs = x_k, H1 = D of stage 1, xh = what the second evaluation saw, D = its D)
                        want2 = dict(cs=O(unit("xh"))[0], ch=O(unit("D"))[0], cx=O(unit("X2"))[0], cd=O(unit("D2"))[0], ch2=0.0, cn=0.0)
                        assert q2["write_xs"] == 0 and q2["hist"] == 0
                        pairs = [(q, want), (q2, want2)]
                    else:
                        want = {c: O(unit(nm))[0] for c, nm in zip(("cx", "cs", "cd", "ch", "ch2", "cn"), VARS)}
                        if sampler == "unipc" and sig[k + 1] > 0:
                            want.update({c: O(unit(nm))[1] for c, nm in zip(("sx", "ss", "sd", "sh", "sh2"), VARS[:5])})
                            assert q["write_xs"] == 1
                        assert q["sigma_next"] == sig[k + 1]
                        pairs = [(q, want)]
                        if sig[k + 1] == 0:   # the step to sigma = 0 returns D exactly
                            assert [q[c] for c in ("cx", "cs", "cd", "ch", "ch2", "cn", "c_in")] == [0, 0, 1, 0, 0, 0, 1]
                        elif sampler in ("dpmpp_3m_sde", "unipc"):   # H2 <- H1, H1 <- D
                            assert q["hist"] == 1 + 2 * (n_hist >= 1)
                        elif sampler == "dpmpp_2m_sde":
                            assert q["hist"] == 1
                    for got, w in pairs:
                        assert got["c_in"] == np.float32(1 / (got["sigma_next"] ** 2 + 1) ** 0.5)
                        for c, wv in w.items():
                            assert math.isfinite(got[c]) and close(got[c], wv), (sampler, spacing, n, k, n_hist, c, got[c], wv)
                            worst = max(worst, abs(got[c] - wv) / max(abs(wv), 1e-3))
                            checked += 1
    print(f"{sampler}: {checked} stage coefficients, worst relative difference {worst:.2e}")


def test_single_stage_samplers_are_unchanged():
    """The four earlier samplers come out of the same function as one stage, as sdxl_test_step_coef has always read them."""
    a = SO1.sdxl_alphas(N, f16=True)
    for sampler in ("euler", "euler_ancestral", "dpmpp_2m", "lcm"):
        sch = Schedule(sampler, "karras", 6)
        t, sig = schedulers.build(a, sch)
        for k in range(6):
            for n_hist in (0, 1, 2):
                st = _testing.step_stages(a, sch.to_struct(), k, t, sig, n_hist)
                out = (C.c_float * 5)()
                _testing.load().sdxl_test_step_coef(C.byref(sch.to_struct()), k, t.ctypes.data, sig.ctypes.data, int(n_hist > 0), out)
                assert len(st) == 1 and [st[0][c] for c in ("cx", "cd", "ch", "cn", "c_in")] == list(out)
                assert st[0]["cs"] == st[0]["ch2"] == 0 and st[0]["write_xs"] == 0
                assert st[0]["hist"] == (1 if sampler == "dpmpp_2m" else 0)


# ---- the recurrences on Gaussian data ------------------------------------------------------------------------------------------
def gaussian_eps(s_data, ls):
    """Data ~ N(0, s^2 I): the ideal noise prediction of the VP-scaled input at sigma(t) is sigma * xh / (sigma^2 + s^2)."""
    def f(x_in, t):
        sigma = SO1.sigma_of_t(ls, t)
        xh = x_in * (sigma ** 2 + 1) ** 0.5
        return sigma * xh / (sigma ** 2 + s_data ** 2)
    return f


def ode_error(sampler, n, s_data=0.7, eta=1.0):
    a = SO1.sdxl_alphas(N)
    ls = SO1.log_sigmas(a)
    t, sig = SO1.schedule("karras", n, a)
    x0 = np.array([1.0, -2.0, 0.5]) * (sig[0] ** 2 + 1) ** 0.5
    never = lambda: (_ for _ in ()).throw(AssertionError("no noise at eta = 0"))   # noqa: E731
    got = SO.sample2(gaussian_eps(s_data, ls), sampler, t, sig, x0, draw=never, k1=n - 1, eta=eta, ls=ls)
    want = x0 * ((sig[n - 1] ** 2 + s_data ** 2) / (sig[0] ** 2 + s_data ** 2)) ** 0.5
    return float(np.abs(got - want).max() / np.abs(want).max())


def test_orders_of_convergence():
    ns = [10, 20, 40, 80, 160]
    slope, err = {}, {}
    for name, sampler, eta in (("heun", "heun_discrete", 1.0), ("dpm_2", "dpm_2", 1.0), ("dpmpp_3m (eta 0)", "dpmpp_3m_sde", 0.0),
                               ("dpmpp_2m_sde (eta 0)", "dpmpp_2m_sde", 0.0), ("unipc", "unipc", 1.0)):
        err[name] = [ode_error(sampler, n, eta=eta) for n in ns]
        slope[name] = np.polyfit(np.log(ns), np.log(err[name]), 1)[0]
        print(name, "errors", ["%.2e" % e for e in err[name]], "slope %.2f" % slope[name])
    assert -2.4 < slope["heun"] < -1.7 and -2.4 < slope["dpm_2"] < -1.7
    # k-diffusion's third-order term is phi_3 d2 with d2 = (d1_0 - d1_1) / (r0 + r1) ~ h^2 D'' / 2, half the Taylor term h^3 phi_3 D''
    # of the exponential integrator: the formula as written converges at second order, with a smaller constant than DPM++ 2M's
    # (DESIGN.md §20). Doubling that term in the oracle gives a slope of -2.8.
    assert -2.6 < slope["dpmpp_3m (eta 0)"] < -1.9
    assert -2.4 < slope["dpmpp_2m_sde (eta 0)"] < -1.7   # DPM++ 2M itself at eta = 0
    assert all(a < b for a, b in zip(err["dpmpp_3m (eta 0)"][1:], err["dpmpp_2m_sde (eta 0)"][1:]))
    assert slope["unipc"] < -1.8


@pytest.mark.parametrize("sampler", ["dpmpp_2m_sde", "dpmpp_3m_sde"])
def test_sde_samplers_end_at_the_data_variance(sampler):
    """N(0, s_d^2) data with its exact denoiser D = xh s_d^2 / (sigma^2 + s_d^2): started from the exact marginal at sigma_0, the
    SDE ends with the data's variance. Over 60 Karras steps the ratio is within 1 % of 1 (the statistical error is
    sqrt(2 / 4e5) = 0.22 %); the discretisation bias is +7 % / +3 % (2M / 3M) at 20 steps, +0.2 % / -0.1 % at 60."""
    a = SO1.sdxl_alphas(N)
    ls = SO1.log_sigmas(a)
    n, s_d, m = 60, 0.6, 400_000
    t, sig = SO1.schedule("karras", n, a)
    rng = np.random.default_rng(1)
    x = rng.standard_normal(m) * (sig[0] ** 2 + s_d ** 2) ** 0.5
    out = SO.sample2(gaussian_eps(s_d, ls), sampler, t, sig, x, draw=lambda: rng.standard_normal(m), ls=ls)
    ratio = float(out.var() / s_d ** 2)
    print(f"{sampler}: end variance / s_d^2 = {ratio:.4f} over {n} Karras steps")
    assert abs(ratio - 1.0) < 0.01


# ---- noise count, refusals, Python surface, C ABI, SASS ---------------------------------------------------------------------------
@pytest.mark.parametrize("sampler", NEW)
def test_n_noise_is_the_oracles_draw_count(sampler):
    a = SO1.sdxl_alphas(N)
    ls = SO1.log_sigmas(a)
    for kw in (dict(), dict(last_step=3), dict(first_step=2, renoise=True), dict(first_step=1, last_step=4, renoise=True)):
        for inpainting in (False, True):
            sch = Schedule(sampler, "karras", 6, **kw)
            t, sig = SO1.schedule("karras", 6, a)
            draws, evals = [0], []

            def draw():
                draws[0] += 1
                return np.zeros(2)
            x = np.ones(2) * (draw() + 1.0) if not sch.first_step else np.ones(2) + (draw() if sch.renoise else 0.0)
            blend = (np.zeros(2), np.array([True, False])) if inpainting else None
            SO.sample2(lambda x_in, tk: 0.3 * x_in, sampler, t, sig, x, draw, sch.first_step, sch.last_step or 6, blend=blend, ls=ls,
                       on_eval=evals.append)
            assert sch.n_noise(initial=not sch.first_step, inpainting=inpainting) == draws[0], (kw, inpainting)
            assert sch.n_evaluations() == len(evals)


def test_invalid_samplers_name_the_field():
    lib = _lib.load()
    a = SO1.sdxl_alphas(N)
    t, sig = np.zeros(4), np.zeros(5)
    for v in (4, 10, -1, 100):
        s = Schedule("euler", "karras", 4).to_struct()
        s.sampler = v
        assert lib.sdxl_schedule_build(a.ctypes.data, N, C.byref(s), t.ctypes.data, sig.ctypes.data) != 0
        assert "sampler" in lib.sdxl_schedule_last_error().decode()
    for name in NEW:
        assert name in MORE_SAMPLERS and name not in SAMPLERS
        schedulers.build(a, Schedule(name, "karras", 4))
    assert [MORE_SAMPLERS[s] for s in NEW] == [5, 6, 7, 8, 9] and ALL_SAMPLERS == {**SAMPLERS, **MORE_SAMPLERS}
    for name in ("dpmpp_sde", "heun"):
        with pytest.raises(SdxlError, match="sampler"):
            Schedule(name, "karras", 4).to_struct()


def test_sampler2_abi_from_c(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib_dir = os.path.join(ROOT, "stable-diffusion-xl-burn_b200", "sdxl_b200")
    exe = str(tmp_path / "sampler2_abi_check")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "c_abi", "sampler2_abi_check.c"), "-L", lib_dir, "-lsdxl_b200", "-Wl,-rpath," + lib_dir,
                        "-lm", "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout.startswith("sampler2_abi_check ok 9"), (r.returncode, r.stdout, r.stderr)


def test_existing_step_kernel_sass_is_unchanged(tmp_path):
    """The four one-row instantiations of guided_step_kernel compile to the instructions they compiled to before the two-row form
    existed (tests/golden/guided_step_sass.json: sha256 of each kernel's SASS without its address comments, from the same nvcc)."""
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "guided_step_sass.json")))
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not (os.path.exists(nvcc) and os.path.exists(cuobjdump)):
        pytest.skip("no CUDA toolkit")
    if subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout.strip().splitlines()[-1] != golden["nvcc"]:
        pytest.skip("a different nvcc than the digests were taken with")
    obj = str(tmp_path / "elementwise.o")
    src = os.path.join(ROOT, "stable-diffusion-xl-burn_b200", "csrc", "elementwise.cu")
    flags = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-Xcompiler",
             "-fvisibility=hidden"]
    r = subprocess.run([nvcc, *flags, "-c", src, "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True).stdout
    got, name, body = {}, None, []
    for line in sass.splitlines() + ["Function : end"]:
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            f = re.search(r"guided_step_kernelILb(\d)ELb(\d)ELb0EE", name or "")
            if f:
                text = "\n".join(re.sub(r"/\*[0-9a-f]{4}\*/", "", ln).strip() for ln in body if ln.strip())
                got[f"v={f.group(1)} rescale={f.group(2)}"] = hashlib.sha256(text.encode()).hexdigest()
            name, body = m.group(1), []
        elif name:
            body.append(line)
    assert got == golden["sha256"]
