"""CPU tests of image-prompt sets (DESIGN.md §13): the oracle's mask downsample (F.interpolate's grid on matching aspects, the
pad / truncate branches otherwise), the oracle's per-source attention against a direct softmax, the Python refusals made before any
library call, and a C program against the header."""
import ctypes as C
import os
import shutil
import subprocess
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from sdxl_b200 import TINY, SdxlError
from sdxl_b200 import _lib
from sdxl_b200.ip_adapter import set_image_prompts
from oracle import unet_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("H,W", [(1024, 1024), (832, 1216), (1216, 832), (128, 128)])
def test_downsample_matching_aspect_is_the_level_grid(H, W):
    """A mask of the latent's aspect lands on the level's own (h_l, w_l) grid: F.interpolate to that size, no pad or cut."""
    g = torch.Generator().manual_seed(H + W)
    m = (torch.rand(2, H, W, generator=g) > 0.5).float()
    for l in range(3):
        hl, wl = (H // 8) >> l, (W // 8) >> l
        assert O.mask_grid(H, W, hl * wl) == (hl, wl)
        want = F.interpolate(m[:, None], size=(hl, wl), mode="bicubic", align_corners=False)[:, 0].reshape(2, -1)
        assert torch.equal(O.downsample_mask(m, hl * wl), want)


def test_downsample_pads_and_truncates():
    """1216 x 832 (W / H = 0.684) against levels of another aspect: T = 4096 (64 x 64) gives mh = int(77.4) + 1 = 78, mw = 52 and
    4056 values padded with 40 zeros. mw = T // mh never overshoots T, so the cut happens only where mh alone exceeds T: a 64 x 8
    mask against T = 2 gives a 5 x 1 grid, cut to its first 2 values."""
    m = torch.rand(1, 1216, 832, generator=torch.Generator().manual_seed(1))
    assert O.mask_grid(1216, 832, 4096) == (78, 52)
    assert O.mask_grid(64, 8, 2) == (5, 1)
    for mask, T in ((m, 4096), (m, 1000), (m, 7), (torch.rand(1, 64, 8, generator=torch.Generator().manual_seed(2)), 2)):
        mh, mw = O.mask_grid(mask.shape[1], mask.shape[2], T)
        full = F.interpolate(mask[:, None], size=(mh, mw), mode="bicubic", align_corners=False)[:, 0].reshape(1, -1)
        got = O.downsample_mask(mask, T)
        assert got.shape == (1, T)
        n = min(T, mh * mw)
        assert torch.equal(got[:, :n], full[:, :n]) and bool((got[:, n:] == 0).all())
        assert (mh * mw < T) == (T != 2)   # padded, except the cut case


def test_multi_attention_against_softmax():
    g = torch.Generator().manual_seed(0)
    B, T, n_head = 2, 10, 2
    q = torch.randn(B, T, 128, generator=g)
    k, v = torch.randn(B, 5, 128, generator=g), torch.randn(B, 5, 128, generator=g)
    srcs = [(torch.randn(B, 4, 128, generator=g), torch.randn(B, 4, 128, generator=g), 0.7, None),
            (torch.randn(B, 3, 128, generator=g), torch.randn(B, 3, 128, generator=g), 1.3, torch.linspace(-0.1, 1.1, T))]

    def att(q, k, v):
        out = []
        for h in range(n_head):
            sl = slice(64 * h, 64 * h + 64)
            out.append(torch.softmax(q[..., sl] @ k[..., sl].transpose(1, 2) / 8, -1) @ v[..., sl])
        return torch.cat(out, -1)
    want = att(q, k, v) + 0.7 * att(q, *srcs[0][:2]) + 1.3 * srcs[1][3][None, :, None] * att(q, *srcs[1][:2])
    assert torch.allclose(O.multi_attention(q, k, v, srcs, n_head), want, atol=1e-5)


class _NoLibrary:
    """Stands in for the library: any call fails the test."""
    def __getattr__(self, name):
        raise AssertionError(f"library call {name} made")


def _fake():
    from sdxl_b200.ip_adapter import IPAdapter
    ad = IPAdapter.__new__(IPAdapter)
    ad.ctx = SimpleNamespace(lib=_NoLibrary(), device=torch.device("cpu"))
    ad.cfg, ad.image_embed_dim, ad.h, ad.attached = TINY, 16, C.c_void_p(1), 0
    return ad, SimpleNamespace(ctx=ad.ctx, h=C.c_void_p(2), cfg=TINY)


@pytest.mark.parametrize("case", ["five_prompts", "nine_sources", "mask_rank", "mask_images", "mask_size", "mask_nan", "tuple"])
def test_refused_before_any_library_call(case):
    ad, diffuser = _fake()
    e1, e3 = torch.zeros(1, 1, 16), torch.zeros(1, 3, 16)
    prompts = {
        "five_prompts": [(ad, e1, 1.0, None, None)] * 5,
        "nine_sources": [(ad, e3, 1.0, None, torch.ones(3, 64, 64))] * 3,
        "mask_rank": [(ad, e1, 1.0, None, torch.ones(64, 64))],
        "mask_images": [(ad, e3, 1.0, None, torch.ones(2, 64, 64))],
        "mask_size": [(ad, e1, 1.0, None, torch.ones(1, 64, 60))],
        "mask_nan": [(ad, e1, 1.0, None, torch.full((1, 64, 64), float("nan")))],
        "tuple": [(ad, e1, 1.0)],
    }[case]
    with pytest.raises(SdxlError):
        set_image_prompts(diffuser, prompts)
    assert ad.attached == 0


def test_mask_binarised_at_half():
    from sdxl_b200.ip_adapter import _mask
    m = torch.tensor([0.0, 0.49, 0.5, 1.0]).reshape(1, 1, 4).repeat(1, 8, 2)
    assert torch.equal(_mask(m, 1)[0, 0, :4], torch.tensor([0.0, 0.0, 1.0, 1.0]))
    assert torch.equal(_mask(torch.full((1, 8, 8), 200, dtype=torch.uint8), 1), torch.ones(1, 8, 8))
    assert torch.equal(_mask(torch.zeros(1, 8, 8, dtype=torch.bool), 1), torch.zeros(1, 8, 8))


def test_ip_multi_abi_check_compiles_and_runs(tmp_path):
    gcc = shutil.which("gcc") or shutil.which("cc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib_dir = os.path.join(ROOT, "stable-diffusion-xl-burn_b200", "sdxl_b200")
    exe = str(tmp_path / "ip_multi_abi_check")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "c_abi", "ip_multi_abi_check.c"), "-L", lib_dir, "-lsdxl_b200", "-Wl,-rpath," + lib_dir,
                        "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout.startswith("ip_multi_abi_check ok"), (r.returncode, r.stdout, r.stderr)
    assert int(r.stdout.split()[-1]) == C.sizeof(_lib.IpMask)
