"""Samplers and noise schedules (include/sdxl_b200.h: sdxl_schedule; DESIGN.md §16): the ctypes mirror with string names and
`build`, the host-only timestep / sigma table of a schedule. Needs no GPU."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Sequence, Tuple

import numpy as np

from . import _lib

SAMPLERS = {"euler": 0, "euler_ancestral": 1, "dpmpp_2m": 2, "lcm": 3}
SPACINGS = {"reference": 0, "leading": 1, "trailing": 2, "linspace": 3, "karras": 4, "lcm": 5}


@dataclass
class Schedule:
    """sampler: one of SAMPLERS; spacing: one of SPACINGS; the other fields as sdxl_schedule documents them."""
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
        for what, table, v in (("sampler", SAMPLERS, self.sampler), ("spacing", SPACINGS, self.spacing)):
            if v not in table:
                raise _lib.SdxlError(f"Schedule: {what} = {v!r} is not one of {sorted(table)}")
        return _lib.Schedule(SAMPLERS[self.sampler], SPACINGS[self.spacing], int(self.n_steps), int(self.first_step), int(self.last_step),
                             int(self.renoise), int(self.no_cfg), float(self.karras_rho), float(self.eta), float(self.s_noise))

    def n_noise(self, initial: bool, inpainting: bool = False) -> int:
        """Noise tensors a call with this schedule consumes, in the order sdxl_sample_latent_scheduled documents (initial: the
        call draws its initial noise, i.e. first_step == 0 and no init tensor is passed)."""
        last = self.last_step or self.n_steps
        steps = last - self.first_step
        n = int(initial) + int(self.renoise) + (steps if inpainting else 0)
        if self.sampler in ("euler_ancestral", "lcm"):   # none on the step to sigma = 0
            n += steps - (1 if last == self.n_steps else 0)
        return n


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
