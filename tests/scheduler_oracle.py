"""Float64 statement of the noise schedules and samplers of DESIGN.md §16, written from their sources (Karras et al. 2022,
"Elucidating the Design Space of Diffusion-Based Generative Models"; Lu et al. 2022, "DPM-Solver++", in k-diffusion's
sample_dpmpp_2m form; Luo et al. 2023, "Latent Consistency Models", in diffusers' LCMScheduler form), each sampler in its own
recurrence rather than as coefficients. Imports nothing from the engine. Works on numpy arrays and torch tensors alike."""
import math

import numpy as np


def sdxl_alphas(n=1000, f16=False):
    """SDXL's scaled-linear betas 0.00085 .. 0.012; f16: rounded to half precision as the model record stores them."""
    betas = np.linspace(0.00085 ** 0.5, 0.012 ** 0.5, n, dtype=np.float64) ** 2
    a = np.cumprod(1.0 - betas)
    return a.astype(np.float16).astype(np.float64) if f16 else a


def log_sigmas(alphas):
    a = np.asarray(alphas, dtype=np.float64)
    return 0.5 * np.log((1.0 - a) / a)


def sigma_of_t(ls, t):
    lo = min(int(math.floor(t)), len(ls) - 2)
    w = t - lo
    return math.exp((1.0 - w) * ls[lo] + w * ls[lo + 1])


def t_of_sigma(ls, sigma):
    """k-diffusion's sigma_to_t."""
    x = math.log(sigma)
    lo = int(np.clip(np.searchsorted(ls, x, side="right") - 1, 0, len(ls) - 2))
    w = min(max((x - ls[lo]) / (ls[lo + 1] - ls[lo]), 0.0), 1.0)
    return lo + w


def schedule(spacing, n, alphas, rho=7.0):
    """(t [n], sigma [n + 1]) with sigma[n] = 0."""
    ls = log_sigmas(alphas)
    N = len(ls)
    if spacing == "karras":
        smax, smin = math.exp(ls[-1]), math.exp(ls[0])
        ramp = np.linspace(0.0, 1.0, n) if n > 1 else np.zeros(1)
        sig = (smax ** (1 / rho) + ramp * (smin ** (1 / rho) - smax ** (1 / rho))) ** rho
        return np.array([t_of_sigma(ls, s) for s in sig]), np.append(sig, 0.0)
    if spacing == "reference":
        t = np.array([N - 1 - k * (N // n) for k in range(n)], dtype=np.float64)
    elif spacing == "leading":
        t = np.array([(n - 1 - k) * (N // n) + 1 for k in range(n)], dtype=np.float64)
    elif spacing == "trailing":
        t = np.round(np.arange(N, 0, -N / n))[:n] - 1
    elif spacing == "linspace":
        t = np.linspace(N - 1, 0, n) if n > 1 else np.array([N - 1.0])
    elif spacing == "lcm":
        origin = (np.arange(1, 51) * (N // 50) - 1)[::-1]
        t = origin[np.floor(np.linspace(0, 50, n, endpoint=False)).astype(int)].astype(np.float64)
    else:
        raise ValueError(spacing)
    return t, np.append([sigma_of_t(ls, v) for v in t], 0.0)


def step(sampler, k, t, sig, x, D, D_prev=None, draw=None, eta=1.0, s_noise=1.0):
    """x at sig[k] and the denoised prediction D -> x at sig[k + 1]. draw() returns the next noise tensor, called only when used."""
    s, sn = sig[k], sig[k + 1]
    if sampler == "euler":
        d = (x - D) / s
        return x + d * (sn - s)
    if sampler == "euler_ancestral":
        up = min(sn, eta * (sn ** 2 * (s ** 2 - sn ** 2) / s ** 2) ** 0.5)
        down = (sn ** 2 - up ** 2) ** 0.5
        d = (x - D) / s
        x = x + d * (down - s)
        return x + draw() * (s_noise * up) if up > 0 else x
    if sampler == "dpmpp_2m":
        if sn == 0:
            return D
        lam, lam_next = -math.log(s), -math.log(sn)
        h = lam_next - lam
        if D_prev is None:
            return (sn / s) * x - math.expm1(-h) * D
        r = (lam - (-math.log(sig[k - 1]))) / h
        Dd = (1 + 1 / (2 * r)) * D - (1 / (2 * r)) * D_prev
        return (sn / s) * x - math.expm1(-h) * Dd
    if sampler == "lcm":
        a, an = 1 / (s ** 2 + 1), 1 / (sn ** 2 + 1)
        x_vp = x * a ** 0.5
        ts = 10.0 * t[k]
        c_skip, c_out = 0.25 / (ts ** 2 + 0.25), ts / (ts ** 2 + 0.25) ** 0.5
        den = c_out * D + c_skip * x_vp
        if sn == 0:
            return den
        return (an ** 0.5 * den + (1 - an) ** 0.5 * draw()) / an ** 0.5
    raise ValueError(sampler)


def sample(eps_fn, sampler, t, sig, x, draw=None, k0=0, k1=None, eta=1.0, s_noise=1.0, blend=None, where=np.where):
    """Steps [k0, k1) from the state x at sig[k0]; eps_fn(x_in, t_k) is the guided noise prediction of the VP-scaled input.
    blend = (reference, mask): before each forward x = mask ? x : reference + sig[k] * draw()."""
    D_prev = None
    for k in range(k0, len(t) if k1 is None else k1):
        if blend is not None:
            x = where(blend[1], x, blend[0] + sig[k] * draw())
        D = x - sig[k] * eps_fn(x / (sig[k] ** 2 + 1) ** 0.5, t[k])
        x = step(sampler, k, t, sig, x, D, D_prev if sampler == "dpmpp_2m" else None, draw, eta, s_noise)
        D_prev = D
    return x


def coefficients(sampler, k, t, sig, has_prev, eta=1.0, s_noise=1.0):
    """(cx, cd, ch, cn, c_in) of step k, read off the recurrence by linearity."""
    def f(x, D, Dp, z):
        return step(sampler, k, t, sig, x, D, Dp if has_prev else None, lambda: z, eta, s_noise)
    base = f(0.0, 0.0, 0.0, 0.0)
    assert base == 0.0
    return f(1.0, 0.0, 0.0, 0.0), f(0.0, 1.0, 0.0, 0.0), f(0.0, 0.0, 1.0, 0.0), f(0.0, 0.0, 0.0, 1.0), 1 / (sig[k + 1] ** 2 + 1) ** 0.5
