"""ctypes binding of libsdxl_b200_testing.so (csrc/testing.cu): the internal kernel launchers, for kernel-level tests.

Tensors go in as CUDA torch tensors (the caller allocates every output); each call runs on the current torch stream and
raises `SdxlError` on a non-zero launcher status. Not part of the product API.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Sequence

import torch

from ._lib import SdxlError, SdxlLibraryMissing

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libsdxl_b200_testing.so")

P, I, F = C.c_void_p, C.c_int, C.c_float
PROTOTYPES = {
    "sdxl_test_igemm": (I, [P, P, I, I, I, I, I, P, I, I, I, I, I, P, I, I, I, I, I, I, I, P, I, P, I, I, P, I, P, I, I, I, I]),
    "sdxl_test_attention": (I, [P, P, I, I, P, I, I, I, I, I, I, I, P, I, P, I, I, I, I, P]),
    "sdxl_test_attention_multi": (I, [P, P, I, I, P, I, I, I, I, I, I, I, P, I, I, P, P, P, P]),
    "sdxl_test_ip_mask_resize": (I, [P, P, I, I, I, I, I, P]),
    "sdxl_test_attention_small": (I, [P, P, I, I, P, P, I, I, I, I, I, I, I, P, I, P, I, I]),
    "sdxl_test_perceiver_ln": (I, [P, P, P, I, I, I, I, P, P, P, P, F, P, P]),
    "sdxl_test_gn_scratch_floats": (C.c_size_t, [I, I]),
    "sdxl_test_gn_scratch_init": (I, [P, P, I, I]),
    "sdxl_test_gn": (I, [P, P, I, P, I, I, I, I, P, P, F, I, P, P, P, P]),
    "sdxl_test_gemv": (I, [P, P, I, I, I, P, I, P, P, I, I, I, I, P, I]),
    "sdxl_test_conv_in": (I, [P, P, I, I, I, I, I, I, P, P, I, P, P, I]),
    "sdxl_test_conv_in_cat": (I, [P, P, I, I, I, I, P, I, I, I, I, P, P, I, P]),
    "sdxl_test_pag_identity": (I, [P, P, I, C.c_long, P]),
    "sdxl_test_cfg_pag_ddim": (I, [P, P, I, I, I, I, I, F, F, F, F, F, F, P]),
    "sdxl_test_freeu_twiddles": (None, [I, I, P]),
    "sdxl_test_freeu": (I, [P, P, I, P, I, I, I, I, P, P, P]),
    "sdxl_test_repack_upconv": (I, [P, P, I, I, P, I]),
    "sdxl_test_repack_conv": (I, [P, P, I, I, I, I, P, I, I, I]),
    "sdxl_test_transpose_linear": (I, [P, P, I, I, P, I, I, I]),
    "sdxl_test_bias_to_f32": (I, [P, P, I, P, I, I]),
    "sdxl_test_lora_merge": (I, [P, I, I, I, I, P, P, P, P, P, P, I, C.c_size_t, I, I, I, I, P]),
    "sdxl_test_lora_upconv_merge": (I, [P, P, P, I, I, P, I]),
}
_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SdxlLibraryMissing(f"{LIB_PATH} not found: build it with `python stable-diffusion-xl-burn_b200/build.py`")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in PROTOTYPES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def _p(t: Optional[torch.Tensor]):
    if t is None:
        return None
    assert t.is_cuda and t.is_contiguous(), "kernel operands are contiguous CUDA tensors"
    return t.data_ptr()


def _call(name: str, *args) -> None:
    lib = load()
    rc = getattr(lib, name)(torch.cuda.current_stream().cuda_stream, *args)
    if rc != 0:
        raise SdxlError(f"{name} failed ({rc})")


def igemm(a0: torch.Tensor, a0_shape: Sequence[int], w: torch.Tensor, N: int, Ktot: int, out_whb: Sequence[int],
          segs: Sequence[Sequence[int]], out: torch.Tensor, ldo: int, *, a1: Optional[torch.Tensor] = None,
          a1_shape: Sequence[int] = (0, 0, 0, 0), bias: Optional[torch.Tensor] = None, bias_bstride: int = 0,
          res: Optional[torch.Tensor] = None, ldr: int = 0, mode: int = 0, geglu_bn: int = 0,
          opix: Optional[Sequence[int]] = None) -> None:
    """a0 / a1: NHWC f16 (Bn, H, W, C), channel pitch C. segs: (map, dw, dh, db, nkb). opix: (row, w, off) or dense."""
    seg = (C.c_int * (5 * len(segs)))(*[int(v) for s in segs for v in s])
    o = opix or (0, 0, 0)
    _call("sdxl_test_igemm", _p(a0), *a0_shape, a0_shape[3], _p(a1), *a1_shape, a1_shape[3], _p(w), N, Ktot, *out_whb, mode,
          geglu_bn, seg, len(segs), _p(out), int(out.dtype == torch.float32), ldo, _p(bias), bias_bstride, _p(res), ldr, *o)


def attention(q: torch.Tensor, q_pitch: int, q_col0: int, kv: torch.Tensor, kv_pitch: int, k_col0: int, v_col0: int,
              B: int, T: int, S: int, n_head: int, out: torch.Tensor, ldo: int, kip: Optional[torch.Tensor] = None,
              kip_pitch: int = 0, k_ip_col0: int = 0, v_ip_col0: int = 0, S_ip: int = 0,
              ip_scale: Optional[torch.Tensor] = None) -> None:
    _call("sdxl_test_attention", _p(q), q_pitch, q_col0, _p(kv), kv_pitch, k_col0, v_col0, B, T, S, n_head, _p(out), ldo,
          _p(kip), kip_pitch, k_ip_col0, v_ip_col0, S_ip, _p(ip_scale))


def attention_multi(q: torch.Tensor, q_pitch: int, q_col0: int, kv: torch.Tensor, kv_pitch: int, k_col0: int, v_col0: int,
                    B: int, T: int, S: int, n_head: int, out: torch.Tensor, ldo: int, sources: Sequence[tuple]) -> None:
    """sources: (kv [B * S_k, pitch] f16, pitch, k_col0, v_col0, S_k, scale f32 [1], mask f32 [T] or None) per image source."""
    n = len(sources)
    kvs = (C.c_void_p * n)(*[_p(s[0]) for s in sources])
    info = (C.c_int * (4 * n))(*[int(v) for s in sources for v in (s[1], s[2], s[3], s[4])])
    scales = (C.c_void_p * n)(*[_p(s[5]) for s in sources])
    masks = (C.c_void_p * n)(*[_p(s[6]) for s in sources])
    _call("sdxl_test_attention_multi", _p(q), q_pitch, q_col0, _p(kv), kv_pitch, k_col0, v_col0, B, T, S, n_head, _p(out), ldo, n,
          kvs, info, scales, masks)


def ip_mask_resize(mask: torch.Tensor, mh: int, mw: int, T: int) -> torch.Tensor:
    """f32 [T] of a mask plane f32 [H, W]: bicubic resize to (mh, mw), flattened, zero-padded or cut to T."""
    out = torch.empty(T, device=mask.device, dtype=torch.float32)
    _call("sdxl_test_ip_mask_resize", _p(mask), mask.shape[0], mask.shape[1], mh, mw, T, _p(out))
    return out


def attention_small(q, q_pitch, q_col0, k, v, kv_pitch, k_col0, v_col0, B, T, S, n_head, mask, causal, out, ldo,
                    head_dim) -> None:
    _call("sdxl_test_attention_small", _p(q), q_pitch, q_col0, _p(k), _p(v), kv_pitch, k_col0, v_col0, B, T, S, n_head,
          _p(mask), int(causal), _p(out), ldo, head_dim)


def perceiver_ln(x, lat, n, L, Q, C, g1, b1, g2, b2, eps, kv, q) -> None:
    """x f32 [n*L, C], lat f32 [n*Q, C] -> kv f16 [n, L+Q, C] and q f16 [n*Q, C]."""
    _call("sdxl_test_perceiver_ln", _p(x), _p(lat), n, L, Q, C, _p(g1), _p(b1), _p(g2), _p(b2), eps, _p(kv), _p(q))


def gn_scratch(B: int, n_group: int) -> torch.Tensor:
    """A GroupNorm scratch for up to B samples and n_group groups, its arrival counters zeroed once."""
    s = torch.empty(load().sdxl_test_gn_scratch_floats(B, n_group), dtype=torch.float32, device="cuda")
    _call("sdxl_test_gn_scratch_init", _p(s), B, n_group)
    return s


def group_norm(x1, x2, B, HW, n_group, gamma, beta, eps, silu, y, raw, y_lo, scratch) -> None:
    C1 = x1.shape[-1]
    C2 = 0 if x2 is None else x2.shape[-1]
    _call("sdxl_test_gn", _p(x1), C1, _p(x2), C2, B, HW, n_group, _p(gamma), _p(beta), eps, int(silu), _p(y), _p(raw),
          _p(y_lo), _p(scratch))


def gemv(inp, in_bstride, Bv, K, W, ldw, bias, add, add_bstride, N, in_silu, out_silu, out, out_bstride) -> None:
    _call("sdxl_test_gemv", _p(inp), in_bstride, Bv, K, _p(W), ldw, _p(bias), _p(add), add_bstride, N, int(in_silu),
          int(out_silu), _p(out), out_bstride)


def conv_in(x, Bx, B, Cin, H, W, w, bias, Cout, y, add=None, n_add=1) -> None:
    _call("sdxl_test_conv_in", _p(x), int(x.dtype == torch.float32), Bx, B, Cin, H, W, _p(w), _p(bias), Cout, _p(y), _p(add),
          n_add)


def conv_in_cat(x, Bx, B, C1, x2, n2, C2, H, W, w, bias, Cout, y) -> None:
    """The inpainting UNet's first conv: channels [0, C1) from x (f16 or f32), [C1, C1 + C2) from x2 f32 [n2, C2, H, W]."""
    _call("sdxl_test_conv_in_cat", _p(x), int(x.dtype == torch.float32), Bx, B, C1, _p(x2), n2, C2, H, W, _p(w), _p(bias), Cout, _p(y))


def pag_identity(qkv: torch.Tensor, C: int, rows: int, out: torch.Tensor) -> None:
    """out[r, :C] = qkv[r, 2C:3C] for r < rows; qkv f16 [rows, 3C], out f16 [rows, C]."""
    _call("sdxl_test_pag_identity", _p(qkv), C, rows, _p(out))


def cfg_pag_ddim(eps, ld, Bimg, C, HW, use_cfg, guidance, p_t, sqrt_a, sqrt_1ma, sqrt_ap, sqrt_1map, x) -> None:
    """x f32 NCHW [Bimg, C, HW] updated in place from eps NHWC f32 [groups * Bimg, HW, ld]."""
    _call("sdxl_test_cfg_pag_ddim", _p(eps), ld, Bimg, C, HW, int(use_cfg), guidance, p_t, sqrt_a, sqrt_1ma, sqrt_ap, sqrt_1map, _p(x))


def freeu_twiddles(H: int, W: int) -> torch.Tensor:
    """The host twiddle table of an H x W skip (f32 [2 * (H + W)]: cos and sin of 2 pi h / H, then of 2 pi w / W)."""
    out = torch.empty(2 * (H + W), dtype=torch.float32)
    load().sdxl_test_freeu_twiddles(H, W, out.data_ptr())
    return out


def freeu(r, C, x, Cx, B, H, W, tw, s, b) -> None:
    """In place: r f32 NHWC [B, H, W, C] := fourier_filter(r, 1, s[0]), x f32 NHWC [B, H, W, Cx][..., :Cx // 2] *= b[0]; tw, s, b on
    the device."""
    _call("sdxl_test_freeu", _p(r), C, _p(x), Cx, B, H, W, _p(tw), _p(s), _p(b))


def repack_upconv(src, O, I, dst, Ipad) -> None:
    _call("sdxl_test_repack_upconv", _p(src), O, I, _p(dst), Ipad)


def repack_conv(src, O, I, KH, KW, dst, Ktot, col0, Ipad) -> None:
    _call("sdxl_test_repack_conv", _p(src), O, I, KH, KW, _p(dst), Ktot, col0, Ipad)


def transpose_linear(src, K, N, dst, Kpad, dst_row0=0, geglu_bn=0) -> None:
    _call("sdxl_test_transpose_linear", _p(src), K, N, _p(dst), Kpad, dst_row0, geglu_bn)


def bias_to_f32(src, N, dst, geglu_bn=0, accumulate=False) -> None:
    _call("sdxl_test_bias_to_f32", _p(src), N, _p(dst), geglu_bn, int(accumulate))


def lora_merge(N, Kd, taps, terms, src, dst, ld, row0=0, col0=0, Ipad=0, geglu_bn=0, delta_out=None) -> None:
    """terms: [(up [N, r] f16, down [r, Kd] f16, coef)]; src / dst f16 or f32 (f32 storage)."""
    n = len(terms)
    ups = (C.c_void_p * n)(*[_p(u) for u, _, _ in terms])
    downs = (C.c_void_p * n)(*[_p(d) for _, d, _ in terms])
    rs = (C.c_int * n)(*[u.shape[1] for u, _, _ in terms])
    coefs = (C.c_float * n)(*[float(c) for _, _, c in terms])
    _call("sdxl_test_lora_merge", N, Kd, taps, n, ups, downs, rs, coefs, _p(src), _p(dst), int(dst.dtype == torch.float32), ld,
          row0, col0, Ipad, geglu_bn, _p(delta_out))


def lora_upconv_merge(src, delta, O, I, dst, Ipad) -> None:
    _call("sdxl_test_lora_upconv_merge", _p(src), _p(delta), O, I, _p(dst), Ipad)
