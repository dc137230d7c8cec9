"""FreeU, host side: the closed form of diffusers' fourier_filter against its torch.fft statement, the oracle's identities with
the plain forward, the host twiddle table and the C ABI."""
import ctypes as C
import math
import os
import shutil
import subprocess

import pytest
import torch

from sdxl_b200 import TINY, _lib, synth_weights
from oracle import unet_oracle as O
import freeu_oracle as FO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXTENTS = [1, 2, 5, 7, 8, 32, 64]


@pytest.mark.parametrize("H", EXTENTS)
@pytest.mark.parametrize("W", EXTENTS)
def test_closed_form_is_the_fft_filter(H, W):
    """K = {0, -1} x {0, -1} as a set: H = 1 has one row frequency, H = 2 has -1 = 1."""
    g = torch.Generator().manual_seed(H * 100 + W)
    r = torch.randn(2, 3, H, W, generator=g, dtype=torch.float64)
    for s in (0.2, 0.9, 1.0, 1.7):
        want = O.fourier_filter(r, 1, s)
        got = FO.fourier_filter_closed(r, s)
        assert float((got - want).abs().max()) <= 1e-12 * max(1.0, float(want.abs().max()))


def test_filter_acts_on_the_lowest_bins_only():
    """The mask m is s on {0, -1} x {0, -1}. Taking the real part makes bin k and bin -k both scale by (m(k) + m(-k)) / 2: s on
    (0, 0), (s + 1) / 2 on (0, -1), (-1, 0), (-1, -1) and their mirrors, 1 elsewhere."""
    g = torch.Generator().manual_seed(3)
    r = torch.randn(1, 2, 8, 6, generator=g, dtype=torch.float64)
    s = 0.25
    ratio = torch.fft.fft2(O.fourier_filter(r, 1, s)) / torch.fft.fft2(r)
    m = torch.ones(8, 6, dtype=torch.float64)
    for kh in (0, 7):
        for kw in (0, 5):
            m[kh, kw] = s
    want = (m + torch.roll(torch.flip(m, (0, 1)), (1, 1), (0, 1))) / 2   # (m(k) + m(-k)) / 2
    assert want[0, 0] == s and want[0, 1] == (s + 1) / 2 and want[7, 5] == (s + 1) / 2 and want[3, 3] == 1
    assert torch.allclose(ratio, want.to(torch.complex128).expand_as(ratio), atol=1e-12)


def _inputs():
    w = O.to_f32(synth_weights(TINY, seed=0))
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 4, 16, 16, generator=g)
    ctx, y = torch.randn(2, 7, TINY.context_dim, generator=g), torch.randn(2, TINY.adm_in_channels, generator=g)
    return w, x, torch.tensor([499]), ctx, y


def test_oracle_identities():
    """All four values 1 is the plain forward up to FFT round-off; any value 0 is the plain forward exactly; the recommended values
    move it."""
    w, x, t, ctx, y = _inputs()
    plain = O.unet_forward(TINY, w, x, t, ctx, y)
    assert torch.equal(O.unet_forward(TINY, w, x, t, ctx, y, O.Attach(freeu=(0.9, 0.0, 1.3, 1.4))), plain)
    ones = O.unet_forward(TINY, w, x, t, ctx, y, O.Attach(freeu=(1.0, 1.0, 1.0, 1.0)))
    assert float((ones - plain).norm() / plain.norm()) < 1e-6
    moved = O.unet_forward(TINY, w, x, t, ctx, y, O.Attach(freeu=FO.RECOMMENDED_SDXL))
    assert float((moved - plain).norm() / plain.norm()) > 1e-3


def test_host_twiddles():
    """The table the plan uploads: cos and sin of 2 pi h / H and 2 pi w / W, rounded once from double precision."""
    from sdxl_b200 import _testing
    try:
        _testing.load()
    except Exception as e:   # the testing library is built by build(); nothing to check without it
        pytest.skip(f"testing library not loadable: {e}")
    for H, W in ((1, 2), (5, 7), (32, 64)):
        got = _testing.freeu_twiddles(H, W)
        a = [2 * math.pi * h / H for h in range(H)]
        b = [2 * math.pi * v / W for v in range(W)]
        want = torch.tensor([math.cos(v) for v in a] + [math.sin(v) for v in a] + [math.cos(v) for v in b] + [math.sin(v) for v in b],
                            dtype=torch.float64).float()
        assert torch.equal(got, want)


def test_freeu_abi_from_c(tmp_path):
    """A C99 program using the FreeU part of include/sdxl_b200.h compiles with -pedantic -Werror, links and sees the layout."""
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib_dir = os.path.join(ROOT, "stable-diffusion-xl-burn_b200", "sdxl_b200")
    exe = str(tmp_path / "freeu_abi_check")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "c_abi", "freeu_abi_check.c"), "-L", lib_dir, "-lsdxl_b200", "-Wl,-rpath," + lib_dir,
                        "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout.startswith("freeu_abi_check ok"), (r.returncode, r.stdout, r.stderr)
    assert int(r.stdout.split()[-1]) == C.sizeof(_lib.Freeu)
