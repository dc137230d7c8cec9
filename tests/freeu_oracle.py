"""FreeU (DESIGN.md §15) beside the f32 CPU oracle, which applies diffusers' apply_freeu before the skip concatenations of
up_blocks[0] and up_blocks[1] (this engine's output_blocks/0..5) with diffusers' fourier_filter restated literally with torch.fft
(oracle/unet_oracle.py). Here: the closed form the kernel computes (fourier_filter_closed), in float64, as the kernel tests'
reference, and the recommended SDXL values."""
from __future__ import annotations

import math

import torch

RECOMMENDED_SDXL = (0.9, 0.2, 1.3, 1.4)   # the FreeU authors' values for SDXL (s1, s2, b1, b2)


def fourier_filter_closed(r: torch.Tensor, scale: float) -> torch.Tensor:
    """fourier_filter(r, 1, scale) in closed form: r + (scale - 1) / N * sum_{k in K} Re(X_k e^{i theta_k}), K = {0, -1 mod H} x
    {0, -1 mod W} as a set, X_k = sum r e^{-i theta_k}, theta_k(h, w) = 2 pi (k_h h / H + k_w w / W). In r's dtype (float64 for
    the kernels' reference)."""
    B, C, H, W = r.shape
    N = H * W
    hh = torch.arange(H, dtype=torch.float64)[:, None]
    ww = torch.arange(W, dtype=torch.float64)[None, :]
    out = r.double().clone()
    for kh in sorted({0, (H - 1) % H}):
        for kw in sorted({0, (W - 1) % W}):
            theta = 2 * math.pi * (kh * hh / H + kw * ww / W)
            X = (r.double() * torch.exp(-1j * theta)).sum(dim=(-2, -1))
            out += (scale - 1) / N * (X[..., None, None] * torch.exp(1j * theta)).real
    return out.to(r.dtype)
