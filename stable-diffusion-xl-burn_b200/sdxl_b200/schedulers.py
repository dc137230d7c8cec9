"""Samplers and noise schedules (include/sdxl_b200.h: sdxl_schedule; DESIGN.md §16, §20): the ctypes mirror with string names and
`build`, the host-only timestep / sigma table of a schedule. Needs no GPU."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Sequence, Tuple

import numpy as np

from . import _lib

SAMPLERS = {"euler": 0, "euler_ancestral": 1, "dpmpp_2m": 2, "lcm": 3}   # one evaluation and at most one history slot (§16)
# DESIGN.md §20: the SDE multistep samplers, UniPC, and the two-evaluation Heun (diffusers' HeunDiscreteScheduler, k-diffusion's
# sample_heun) and DPM2
MORE_SAMPLERS = {"dpmpp_2m_sde": 5, "dpmpp_3m_sde": 6, "unipc": 7, "heun_discrete": 8, "dpm_2": 9}
ALL_SAMPLERS = {**SAMPLERS, **MORE_SAMPLERS}
TWO_EVALUATIONS = ("heun_discrete", "dpm_2")   # UNet evaluations per step: two, except on the step to sigma = 0
SPACINGS = {"reference": 0, "leading": 1, "trailing": 2, "linspace": 3, "karras": 4, "lcm": 5}


@dataclass
class Schedule:
    """sampler: one of ALL_SAMPLERS; spacing: one of SPACINGS; the other fields as sdxl_schedule documents them."""
    sampler: str = "euler"
    spacing: str = "leading"
    n_steps: int = 30
    first_step: int = 0
    last_step: int = 0
    renoise: bool = False
    no_cfg: bool = False
    karras_rho: float = 0.0
    eta: float = 0.0
    s_noise: float = 0.0

    @classmethod
    def from_strength(cls, n_steps: int, strength: float, **kw) -> "Schedule":
        """img2img as diffusers computes it: the last min(int(n_steps * strength), n_steps) steps run, from the re-noised image."""
        if not 0.0 < strength <= 1.0:
            raise _lib.SdxlError(f"Schedule.from_strength: strength = {strength} outside (0, 1]")
        first = n_steps - min(int(n_steps * strength), n_steps)
        if first >= n_steps:
            raise _lib.SdxlError(f"Schedule.from_strength: strength = {strength} leaves no step of {n_steps}")
        return cls(n_steps=n_steps, first_step=first, renoise=first > 0, **kw)

    def to_struct(self) -> "_lib.Schedule":
        for what, table, v in (("sampler", ALL_SAMPLERS, self.sampler), ("spacing", SPACINGS, self.spacing)):
            if v not in table:
                raise _lib.SdxlError(f"Schedule: {what} = {v!r} is not one of {sorted(table)}")
        return _lib.Schedule(ALL_SAMPLERS[self.sampler], SPACINGS[self.spacing], int(self.n_steps), int(self.first_step), int(self.last_step),
                             int(self.renoise), int(self.no_cfg), float(self.karras_rho), float(self.eta), float(self.s_noise))

    def n_noise(self, initial: bool, inpainting: bool = False) -> int:
        """Noise tensors a call with this schedule consumes, in the order sdxl_sample_latent_scheduled documents (initial: the
        call draws its initial noise, i.e. first_step == 0 and no init tensor is passed)."""
        last = self.last_step or self.n_steps
        steps = last - self.first_step
        to_zero = 1 if last == self.n_steps else 0   # the call runs the step to sigma = 0
        n = int(initial) + int(self.renoise) + (self.n_evaluations() if inpainting else 0)   # a blend before every evaluation
        if self.sampler in ("euler_ancestral", "lcm", "dpmpp_2m_sde", "dpmpp_3m_sde"):   # none on the step to sigma = 0
            n += steps - to_zero
        return n

    def n_evaluations(self) -> int:
        """UNet evaluations of a call with this schedule (DeepCache counts these)."""
        last = self.last_step or self.n_steps
        steps = last - self.first_step
        return steps + (steps - (1 if last == self.n_steps else 0) if self.sampler in TWO_EVALUATIONS else 0)


def alphas_cumprod(n: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012, zero_terminal_snr: bool = False) -> np.ndarray:
    """alphas_cumprod f64 [n] of diffusers' scaled-linear betas, computed as diffusers computes it, in float32. zero_terminal_snr:
    the betas rescaled to zero terminal SNR first (Lin et al. 2023, Algorithm 1: diffusers' rescale_zero_terminal_snr) and the last
    entry set to 2^-24, as diffusers' Euler and DPM-Solver schedulers do (rescale_betas_zero_snr=True). For
    Diffuser.set_prediction (DESIGN.md §18)."""
    import torch
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, n, dtype=torch.float32) ** 2
    if zero_terminal_snr:
        sqrt_bar = torch.cumprod(1.0 - betas, dim=0).sqrt()
        first, last = sqrt_bar[0].clone(), sqrt_bar[-1].clone()
        sqrt_bar = (sqrt_bar - last) * (first / (first - last))   # sqrt(alpha_bar) from sqrt(alpha_bar_0) down to 0
        bar = sqrt_bar ** 2
        betas = 1.0 - torch.cat([bar[0:1], bar[1:] / bar[:-1]])
    a = torch.cumprod(1.0 - betas, dim=0)
    if zero_terminal_snr:
        a[-1] = 2.0 ** -24
    return a.double().numpy()


def prediction_of_config(config: dict):
    """Diffuser.set_prediction's keyword arguments for a diffusers scheduler_config.json (read as a dict), or None when the model is
    an epsilon model on the loaded noise table. Attaches only for prediction_type "v_prediction" or rescale_betas_zero_snr true, with
    the file's betas (diffusers' defaults where a key is missing). Refuses prediction_type "sample" and any other unknown type, and a
    beta_schedule other than "scaled_linear" when it attaches, naming the key."""
    kind = config.get("prediction_type", "epsilon")
    if kind not in _lib.PREDICTIONS:
        raise _lib.SdxlError(f"scheduler config: prediction_type = {kind!r} is not supported (one of {sorted(_lib.PREDICTIONS)})")
    zero_snr = bool(config.get("rescale_betas_zero_snr", False))
    if kind == "epsilon" and not zero_snr:
        return None
    if config.get("beta_schedule", "linear") != "scaled_linear":
        raise _lib.SdxlError(f"scheduler config: beta_schedule = {config.get('beta_schedule', 'linear')!r} is not supported (only "
                             f"'scaled_linear')")
    alphas = alphas_cumprod(int(config.get("num_train_timesteps", 1000)), float(config.get("beta_start", 0.0001)),
                            float(config.get("beta_end", 0.02)), zero_snr)
    return dict(prediction=kind, zero_terminal_snr=zero_snr, alphas=alphas)


def build(alphas: Sequence[float], schedule: Schedule) -> Tuple[np.ndarray, np.ndarray]:
    """(timesteps f64 [n_steps], sigmas f64 [n_steps + 1]) of `schedule` over an alphas_cumprod table (sdxl_schedule_build)."""
    lib = _lib.load()
    a = np.ascontiguousarray(np.asarray(alphas, dtype=np.float64))
    s = schedule.to_struct()
    n = max(int(schedule.n_steps), 0)
    t, sig = np.empty(n, dtype=np.float64), np.empty(n + 1, dtype=np.float64)
    rc = lib.sdxl_schedule_build(a.ctypes.data, a.size, C.byref(s), t.ctypes.data, sig.ctypes.data)
    if rc != 0:
        raise _lib.SdxlError(f"sdxl_schedule_build failed with {rc}: {lib.sdxl_schedule_last_error().decode()}")
    return t, sig


def t2i_t_min(alphas: Sequence[float], schedule: Schedule, factor: float) -> int:
    """t_min of diffusers' adapter_conditioning_factor on `schedule`: the T2I-Adapter features are added on the first
    int(n_iter * factor) of the steps the call runs, i.e. where lround(t_k) >= t_min (the comparison the device makes); 0 when that is
    every step, a t_min above every timestep when it is none."""
    t, _ = build(alphas, schedule)
    ts = t[schedule.first_step:schedule.last_step or schedule.n_steps]
    k = int(len(ts) * factor)
    if k >= len(ts):
        return 0
    return len(alphas) if k <= 0 else int(np.rint(ts[k - 1]))
