"""Float64 statement of the samplers of DESIGN.md §20, beside tests/scheduler_oracle.py's of §16 (whose schedules and sigma table it
uses), each written from its source in its own recurrence rather than as coefficients. Imports nothing from the engine. Works on
numpy arrays and torch tensors alike."""
import math

import numpy as np

from scheduler_oracle import log_sigmas, sdxl_alphas, t_of_sigma  # noqa: F401  (sdxl_alphas, log_sigmas: the callers' tables)

# DPM++ 2M SDE and 3M SDE (k-diffusion sample_dpmpp_2m_sde, midpoint, and sample_dpmpp_3m_sde, after Lu et al.
# 2022), UniPC (Zhao et al. 2023, "UniPC: A Unified Predictor-Corrector Framework", in diffusers' UniPCMultistepScheduler form:
# solver_order 2, x0 prediction, bh2, corrector on, lower_order_final), Heun and DPM2 (Karras et al. 2022, Algorithm 1 without
# churn, and k-diffusion's sample_dpm_2). Each is written as its source writes it: k-diffusion's in the xh scaling, UniPC in the
# variance-preserving one with its linear solves. Keyed by the library's names (sdxl_b200.schedulers.MORE_SAMPLERS).
SAMPLERS2 = ("dpmpp_2m_sde", "dpmpp_3m_sde", "unipc", "heun_discrete", "dpm_2")


def _vp(sigma):
    """(alpha_t, sigma_t) of diffusers' _sigma_to_alpha_sigma_t."""
    a = 1.0 / (sigma ** 2 + 1) ** 0.5
    return a, sigma * a


def _unipc_rb(rks, hh, order):
    """UniPC's R and b (bh2: B(h) = expm1(hh)) for hh = -h."""
    h_phi_1 = math.expm1(hh)
    h_phi_k = h_phi_1 / hh - 1
    factorial_i = 1
    B_h = math.expm1(hh)
    R, b = [], []
    for i in range(1, order + 1):
        R.append(np.power(rks, i - 1))
        b.append(h_phi_k * factorial_i / B_h)
        factorial_i *= i + 1
        h_phi_k = h_phi_k / hh - 1 / factorial_i
    return np.stack(R), np.array(b), h_phi_1, B_h


def unipc_predictor(x, ms, lams, s0, st, order):
    """multistep_uni_p_bh_update: x (VP) at sigma s0, ms[-1] = D at s0, ms[-2] the one before, lams their lambdas -> x (VP) at st."""
    alpha_t, sigma_t = _vp(st)
    _, sigma_s0 = _vp(s0)
    lam_t, lam_s0 = -math.log(st), lams[-1]
    h = lam_t - lam_s0
    m0 = ms[-1]
    rks, D1s = [], []
    for i in range(1, order):
        rk = (lams[-(i + 1)] - lam_s0) / h
        rks.append(rk)
        D1s.append((ms[-(i + 1)] - m0) / rk)
    rks.append(1.0)
    R, b, h_phi_1, B_h = _unipc_rb(np.array(rks), -h, order)
    x_t_ = sigma_t / sigma_s0 * x - alpha_t * h_phi_1 * m0
    if D1s:
        rhos_p = [0.5] if order == 2 else np.linalg.solve(R[:-1, :-1], b[:-1])
        pred_res = sum(r * d for r, d in zip(rhos_p, D1s))
        return x_t_ - alpha_t * B_h * pred_res
    return x_t_


def unipc_corrector(x_last, ms, lams, s0, st, model_t, order):
    """multistep_uni_c_bh_update: the state (VP) at st corrected from x_last at s0, ms[-1] = D at s0 (history before this step's
    D), and model_t = D at st."""
    alpha_t, sigma_t = _vp(st)
    _, sigma_s0 = _vp(s0)
    lam_t, lam_s0 = -math.log(st), lams[-1]
    h = lam_t - lam_s0
    m0 = ms[-1]
    rks, D1s = [], []
    for i in range(1, order):
        rk = (lams[-(i + 1)] - lam_s0) / h
        rks.append(rk)
        D1s.append((ms[-(i + 1)] - m0) / rk)
    rks.append(1.0)
    R, b, h_phi_1, B_h = _unipc_rb(np.array(rks), -h, order)
    rhos_c = np.array([0.5]) if order == 1 else np.linalg.solve(R, b)
    x_t_ = sigma_t / sigma_s0 * x_last - alpha_t * h_phi_1 * m0
    corr_res = sum(r * d for r, d in zip(rhos_c[:-1], D1s)) if D1s else 0.0
    return x_t_ - alpha_t * B_h * (corr_res + rhos_c[-1] * (model_t - m0))


def step2(sampler, k, t, sig, x, D, evaluate=None, hist=None, draw=None, eta=1.0, s_noise=1.0, ls=None):
    """Step k of a §20 sampler from x at sig[k] and its denoised prediction D -> (x at sig[k + 1], state).
    evaluate(x, sigma, t) -> (x as evaluated, D) is the second evaluation of Heun and DPM2 (the latent blend may replace x).
    hist: this call's history, a dict {"D": [...], "h": [...], "x_last": VP state, "order": int} (a fresh dict on a call's first
    step), updated in place. draw() returns the next noise tensor. ls: the log-sigma table (DPM2's fractional midpoint timestep)."""
    hist = {} if hist is None else hist
    s, sn = sig[k], sig[k + 1]
    Ds, hs = hist.setdefault("D", []), hist.setdefault("h", [])
    if sampler == "heun_discrete":
        if sn == 0:
            return D, hist
        d = (x - D) / s
        x2, D2 = evaluate(x + d * (sn - s), sn, t[k + 1])
        d2 = (x2 - D2) / sn
        return x + (d + d2) / 2 * (sn - s), hist
    if sampler == "dpm_2":
        if sn == 0:
            return D, hist
        d = (x - D) / s
        sigma_mid = math.exp(0.5 * (math.log(s) + math.log(sn)))
        x2, D2 = evaluate(x + d * (sigma_mid - s), sigma_mid, t_of_sigma(ls, sigma_mid) if ls is not None else float("nan"))
        d2 = (x2 - D2) / sigma_mid
        return x + d2 * (sn - s), hist
    if sampler == "dpmpp_2m_sde":
        if sn == 0:
            x = D
        else:
            h = math.log(s) - math.log(sn)
            eta_h = eta * h
            x = sn / s * math.exp(-eta_h) * x + (-math.expm1(-h - eta_h)) * D
            if Ds:
                r = hs[-1] / h
                x = x + 0.5 * (-math.expm1(-h - eta_h)) * (1 / r) * (D - Ds[-1])
            if eta:
                x = x + draw() * sn * (-math.expm1(-2 * eta_h)) ** 0.5 * s_noise
            hs.append(h)
        Ds.append(D)
        return x, hist
    if sampler == "dpmpp_3m_sde":
        if sn == 0:
            x = D
        else:
            h = math.log(s) - math.log(sn)
            h_eta = h * (eta + 1)
            x = math.exp(-h_eta) * x + (-math.expm1(-h_eta)) * D
            if len(Ds) >= 2:
                r0, r1 = hs[-1] / h, hs[-2] / h
                d1_0 = (D - Ds[-1]) / r0
                d1_1 = (Ds[-1] - Ds[-2]) / r1
                d1 = d1_0 + (d1_0 - d1_1) * r0 / (r0 + r1)
                d2 = (d1_0 - d1_1) / (r0 + r1)
                phi_2 = math.expm1(-h_eta) / h_eta + 1
                phi_3 = phi_2 / h_eta - 0.5
                x = x + phi_2 * d1 - phi_3 * d2
            elif len(Ds) == 1:
                r = hs[-1] / h
                d = (D - Ds[-1]) / r
                phi_2 = math.expm1(-h_eta) / h_eta + 1
                x = x + phi_2 * d
            if eta:
                x = x + draw() * sn * (-math.expm1(-2 * h * eta)) ** 0.5 * s_noise
            hs.append(h)
        Ds.append(D)
        return x, hist
    if sampler == "unipc":
        lams = hist.setdefault("lam", [])
        xv = x * _vp(s)[0]
        if Ds:   # UniC on this step's state, of the previous step's predictor order
            xv = unipc_corrector(hist["x_last"], Ds, lams, sig[k - 1], s, D, hist["order"])
        hist["x_corrected"] = xv / _vp(s)[0]
        Ds.append(D)
        lams.append(-math.log(s))
        order = min(2, len(Ds), len(t) - k)
        hist["x_last"], hist["order"] = xv, order
        if sn == 0:
            return D, hist
        return unipc_predictor(xv, Ds, lams, s, sn, order) / _vp(sn)[0], hist
    raise ValueError(sampler)


def sample2(eps_fn, sampler, t, sig, x, draw=None, k0=0, k1=None, eta=1.0, s_noise=1.0, blend=None, where=np.where, ls=None,
            on_eval=None):
    """scheduler_oracle.sample for the samplers of §20: steps [k0, k1) from x at sig[k0], with a blend before every evaluation at its sigma and
    the noise drawn in the documented order (each evaluation's blend, then the sampler's). on_eval(t) is called per evaluation."""
    def evaluate(x, s, tk):
        if blend is not None:
            x = where(blend[1], x, blend[0] + s * draw())
        if on_eval is not None:
            on_eval(tk)
        return x, x - s * eps_fn(x / (s ** 2 + 1) ** 0.5, tk)
    hist = {}
    for k in range(k0, len(t) if k1 is None else k1):
        x, D = evaluate(x, sig[k], t[k])
        x, hist = step2(sampler, k, t, sig, x, D, evaluate, hist, draw, eta, s_noise, ls)
    return x
