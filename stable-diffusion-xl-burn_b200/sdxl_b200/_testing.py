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

P, I, F, L, Z = C.c_void_p, C.c_int, C.c_float, C.c_long, C.c_size_t
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
    "sdxl_test_freeu_twiddles": (None, [I, I, P]),
    "sdxl_test_freeu": (I, [P, P, I, P, I, I, I, I, P, P, P]),
    "sdxl_test_repack_upconv": (I, [P, P, I, I, P, I]),
    "sdxl_test_repack_conv": (I, [P, P, I, I, I, I, P, I, I, I]),
    "sdxl_test_transpose_linear": (I, [P, P, I, I, P, I, I, I]),
    "sdxl_test_bias_to_f32": (I, [P, P, I, P, I, I]),
    "sdxl_test_lora_merge": (I, [P, I, I, I, I, P, P, P, P, P, P, I, C.c_size_t, I, I, I, I, P]),
    "sdxl_test_lora_upconv_merge": (I, [P, P, P, I, I, P, I]),
    "sdxl_test_lora_merge_kinds": (I, [P, I, I, I, I, P, P, P, P, P, I, C.c_size_t, I, I, I, I, P]),
    "sdxl_test_dora_norm": (I, [P, I, I, I, P, I, C.c_size_t, I, I, I, I, P, I, P]),
    "sdxl_test_dora_accum": (I, [P, I, I, I, P, I, C.c_size_t, I, I, I, I, P, P, P, I, F, P]),
    "sdxl_test_softmax_rows": (I, [P, P, Z, I, I, F, P, Z]),
    "sdxl_test_transpose_f16": (I, [P, P, Z, I, I, P, Z]),
    "sdxl_test_post_quant": (I, [P, P, I, I, I, P, P, F, P]),
    "sdxl_test_quant_out": (I, [P, P, I, I, I, L, P, P, F, P]),
    "sdxl_test_image_u8": (I, [P, P, L, I, P]),
    "sdxl_test_image_from_u8": (I, [P, P, I, L, P]),
    "sdxl_test_embed_tokens": (I, [P, P, I, I, I, I, P, P, P, P]),
    "sdxl_test_patchify": (I, [P, P, I, I, I, I, P]),
    "sdxl_test_vision_embed_ln": (I, [P, P, P, P, I, I, I, P, P, F, P]),
    "sdxl_test_mlp_act": (I, [P, P, Z, I, P]),
    "sdxl_test_ln_gather_f32": (I, [P, P, P, I, I, I, P, P, F, P]),
    "sdxl_test_pixel_unshuffle": (I, [P, P, I, I, I, I, P]),
    "sdxl_test_relu_f16": (I, [P, P, Z, P]),
    "sdxl_test_avg_pool2_f16": (I, [P, P, I, I, I, I, P]),
    "sdxl_test_t2i_add": (I, [P, P, P, L, I, I, P, P]),
    "sdxl_test_cfg_ddim": (I, [P, P, I, I, I, I, I, I, F, F, F, F, F, F, P]),
    "sdxl_test_inpaint_blend": (I, [P, P, P, P, P, Z, F, F]),
    "sdxl_test_axpby": (I, [P, P, P, Z, F, F]),
    "sdxl_test_cast_f32_to_f16": (I, [P, P, Z, P]),
    "sdxl_test_cast_f16_to_f32": (I, [P, P, Z, P]),
    "sdxl_test_upsample2x": (I, [P, P, I, I, I, I, P]),
    "sdxl_test_phase_split": (I, [P, P, I, I, I, I, P]),
    "sdxl_test_silu_f16": (I, [P, P, I, I, I, I, I, P]),
    "sdxl_test_nhwc_to_nchw_f16": (I, [P, P, I, I, I, I, P]),
    "sdxl_test_nhwc_to_nchw_f32": (I, [P, P, I, I, I, I, P]),
    "sdxl_test_scale_weights": (I, [P, P, Z, P, I, F, P, P]),
    "sdxl_test_vec_add_f32": (I, [P, P, P, I]),
    "sdxl_test_step_coef": (None, [P, I, P, P, I, P]),
    "sdxl_test_guided_step": (I, [P, P, I, I, I, I, I, I, F, F, F, F, F, F, F, F, P, P, P, I, P, P, C.c_uint64, C.c_uint64, C.c_uint64, P, P, F]),
    "sdxl_test_timestep_embedding_f32": (I, [P, P, I, I, F, P]),
    "sdxl_test_cfg_ddim_pred": (I, [P, P, I, I, I, I, I, I, F, F, F, F, F, F, P, I, P]),
    "sdxl_test_guidance_stats_scratch_bytes": (Z, [I]),
    "sdxl_test_guidance_stats_scratch_init": (I, [P, P, I]),
    "sdxl_test_guidance_stats": (I, [P, P, I, I, I, I, I, F, F, F, P, P]),
    "sdxl_test_cfg_ddim_img": (I, [P, P, I, I, I, I, F, F, F, F, F, F, P, I, P]),
    "sdxl_test_guidance_stats_img": (I, [P, P, I, I, I, I, F, F, F, P, P]),
    "sdxl_test_guided_step_img": (I, [P, P, I, I, I, I, F, F, F, F, F, F, F, F, P, P, P, I, P, C.c_uint64, C.c_uint64, I, P, I, P, P, P, P,
                                      I, I]),
    "sdxl_test_guided_step_pred": (I, [P, P, I, I, I, I, I, I, F, F, F, F, F, F, F, F, P, P, P, I, P, P, C.c_uint64, C.c_uint64, C.c_uint64, P,
                                       P, F, I, P]),
    "sdxl_test_guided_step_rows": (I, [P, P, I, I, I, I, I, I, F, F, F, F, F, F, F, F, P, P, P, I, P, P, C.c_uint64, C.c_uint64, C.c_uint64, P,
                                       P, F, I, P, P, P, P, P, I, I]),
    "sdxl_test_step_stages": (I, [P, I, P, I, P, P, I, P]),
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


LORA_KINDS = {"lora": 0, "loha": 1, "lokr": 2, "full": 3, "f32": 4}


def lora_merge_kinds(N, Kd, taps, terms, src, dst, ld, row0=0, col0=0, Ipad=0, geglu_bn=0, delta_out=None) -> None:
    """terms: [(kind, coef, tensors)] with kind a LORA_KINDS key and tensors by kind: lora (up [N, r], down [r, Kd]); loha (up, down,
    up2, down2); lokr (w1 f32 [N / c, I / d], w2 f32 [c, d * taps]); full (diff f16 [N, Kd]); f32 (delta f32 [N, Kd])."""
    n = len(terms)
    ints, ptrs = [], []
    for kind, _, ts in terms:
        z = [None] * 6
        r = r2 = c = d = 0
        if kind in ("lora", "loha"):
            z[0], z[1] = ts[0], ts[1]
            r = ts[0].shape[1]
            if kind == "loha":
                z[2], z[3] = ts[2], ts[3]
                r2 = ts[2].shape[1]
        elif kind == "lokr":
            z[4], z[5] = ts[0], ts[1]
            c, d = ts[1].shape[0], ts[1].shape[1] // taps
        elif kind == "full":
            z[1] = ts[0]
        else:
            z[4] = ts[0]
        ints += [LORA_KINDS[kind], r, r2, c, d]
        ptrs += [_p(x) for x in z]
    coefs = (C.c_float * n)(*[float(cf) for _, cf, _ in terms])
    _call("sdxl_test_lora_merge_kinds", N, Kd, taps, n, (C.c_int * len(ints))(*ints), (C.c_void_p * len(ptrs))(*ptrs), coefs, _p(src),
          _p(dst), int(dst.dtype == torch.float32), ld, row0, col0, Ipad, geglu_bn, _p(delta_out))


def dora_norm(N, Kd, taps, src, ld, dw, axis, norm, row0=0, col0=0, Ipad=0, geglu_bn=0) -> None:
    """norm f64 [N] (axis 0) or [Kd / taps] (axis 1) of W (src through the slot map) + dw f32 [N, Kd]."""
    _call("sdxl_test_dora_norm", N, Kd, taps, _p(src), int(src.dtype == torch.float32), ld, row0, col0, Ipad, geglu_bn, _p(dw), axis,
          _p(norm))


def dora_accum(N, Kd, taps, src, ld, dw, m, norm, axis, s, acc, row0=0, col0=0, Ipad=0, geglu_bn=0) -> None:
    """acc f32 [N, Kd] += s * (m * (W + dw) / norm - W), m f32 and norm f64 along `axis`."""
    _call("sdxl_test_dora_accum", N, Kd, taps, _p(src), int(src.dtype == torch.float32), ld, row0, col0, Ipad, geglu_bn, _p(dw), _p(m),
          _p(norm), axis, float(s), _p(acc))


# latent decoder / encoder (vae_kernels.cu)
def softmax_rows(S, lds, rows, cols, scale, P, ldp) -> None:
    """P f16 [rows, ldp][:, :cols] = softmax(scale * S f32 [rows, lds][:, :cols])."""
    _call("sdxl_test_softmax_rows", _p(S), lds, rows, cols, scale, _p(P), ldp)


def transpose_f16(x, ldx, rows, cols, y, ldy) -> None:
    """y f16 [cols, ldy][:, :rows] = x f16 [rows, ldx][:, :cols] transposed."""
    _call("sdxl_test_transpose_f16", _p(x), ldx, rows, cols, _p(y), ldy)


def post_quant(x, B, C, HW, w, bias, inv_scale, y) -> None:
    _call("sdxl_test_post_quant", _p(x), B, C, HW, _p(w), _p(bias), inv_scale, _p(y))


def quant_out(x, B, Cz, Cout, HW, w, bias, scale, y) -> None:
    _call("sdxl_test_quant_out", _p(x), B, Cz, Cout, HW, _p(w), _p(bias), scale, _p(y))


def image_u8(x, npix, ldx, out) -> None:
    _call("sdxl_test_image_u8", _p(x), npix, ldx, _p(out))


def image_from_u8(inp, B, HW, out) -> None:
    _call("sdxl_test_image_from_u8", _p(inp), B, HW, _p(out))


# text / vision encoders (clip_kernels.cu)
def embed_tokens(tokens, rows, T, C, n_vocab, tok_emb, pos_emb, x, err) -> None:
    _call("sdxl_test_embed_tokens", _p(tokens), rows, T, C, n_vocab, _p(tok_emb), _p(pos_emb), _p(x), _p(err))


def patchify(pixels, N, S, p, Kpad, y) -> None:
    _call("sdxl_test_patchify", _p(pixels), N, S, p, Kpad, _p(y))


def vision_embed_ln(patches, cls, pos, N, T, C, gamma, beta, eps, x) -> None:
    _call("sdxl_test_vision_embed_ln", _p(patches), _p(cls), _p(pos), N, T, C, _p(gamma), _p(beta), eps, _p(x))


def mlp_act(x, n, quick, y) -> None:
    _call("sdxl_test_mlp_act", _p(x), n, int(quick), _p(y))


def ln_gather_f32(x, idx, B, T, C, gamma, beta, eps, y) -> None:
    _call("sdxl_test_ln_gather_f32", _p(x), _p(idx), B, T, C, _p(gamma), _p(beta), eps, _p(y))


# T2I-Adapter (t2i_kernels.cu)
def pixel_unshuffle(x, n, C, H, W, y) -> None:
    _call("sdxl_test_pixel_unshuffle", _p(x), n, C, H, W, _p(y))


def relu_f16(x, n, y) -> None:
    _call("sdxl_test_relu_f16", _p(x), n, _p(y))


def avg_pool2_f16(x, n, H, W, C, y) -> None:
    _call("sdxl_test_avg_pool2_f16", _p(x), n, H, W, C, _p(y))


def t2i_add(x, F, per_img, B, n_hint, t, t_min) -> None:
    """x[b] += F[b % n_hint] unless *t < *t_min; t, t_min: int32 CUDA tensors of one element."""
    _call("sdxl_test_t2i_add", _p(x), _p(F), per_img, B, n_hint, _p(t), _p(t_min))


# sampler, resampling copies and casts (elementwise.cu)
def cfg_ddim(eps, ld, Bimg, C, HW, use_cfg, guidance, sqrt_a, sqrt_1ma, sqrt_ap, sqrt_1map, x, use_pag=False, p_t=0.0) -> None:
    """x f32 NCHW [Bimg, C, HW] updated in place from eps NHWC f32 [(1 + use_cfg + use_pag) * Bimg, HW, ld]; use_pag: the last
    group is the perturbed rows, weighted by p_t."""
    _call("sdxl_test_cfg_ddim", _p(eps), ld, Bimg, C, HW, int(use_cfg), int(use_pag), guidance, p_t, sqrt_a, sqrt_1ma, sqrt_ap, sqrt_1map,
          _p(x))


def cfg_ddim_pred(eps, ld, Bimg, C, HW, use_cfg, guidance, sqrt_a, sqrt_1ma, sqrt_ap, sqrt_1map, x, use_pag=False, p_t=0.0, v=False,
                  factor=None) -> None:
    """cfg_ddim with the v prediction (v) and the per-image guidance-rescale factors (factor: f32 CUDA [Bimg] or None)."""
    _call("sdxl_test_cfg_ddim_pred", _p(eps), ld, Bimg, C, HW, int(use_cfg), int(use_pag), guidance, p_t, sqrt_a, sqrt_1ma, sqrt_ap,
          sqrt_1map, _p(x), int(v), _p(factor))


def guidance_stats_scratch(Bimg, device="cuda") -> torch.Tensor:
    """The statistics kernel's scratch for Bimg images, initialised (its arrival counters zero)."""
    s = torch.empty(int(load().sdxl_test_guidance_stats_scratch_bytes(Bimg)), dtype=torch.uint8, device=device)
    _call("sdxl_test_guidance_stats_scratch_init", _p(s), Bimg)
    return s


def guidance_stats(eps, ld, Bimg, C, HW, use_pag, guidance, p_t, phi, scratch, factor) -> None:
    """factor f32 [Bimg] = phi * std(c_b) / std(g_b) + (1 - phi) of the rows [cond | uncond (| ptb)] of eps (kernels.h)."""
    _call("sdxl_test_guidance_stats", _p(eps), ld, Bimg, C, HW, int(use_pag), guidance, p_t, phi, _p(scratch), _p(factor))


def cfg_ddim_img(eps, ld, Bimg, C, HW, guidance, s_img, sqrt_a, sqrt_1ma, sqrt_ap, sqrt_1map, x, v=False, factor=None) -> None:
    """cfg_ddim_pred with image guidance (DESIGN.md §21): eps rows [cond | img | uncond], e = (u + (c - i) * guidance) + s_img * (i - u)."""
    _call("sdxl_test_cfg_ddim_img", _p(eps), ld, Bimg, C, HW, guidance, s_img, sqrt_a, sqrt_1ma, sqrt_ap, sqrt_1map, _p(x), int(v),
          _p(factor))


def guidance_stats_img(eps, ld, Bimg, C, HW, guidance, s_img, phi, scratch, factor) -> None:
    """guidance_stats of the image-guidance combine of the rows [cond | img | uncond]."""
    _call("sdxl_test_guidance_stats_img", _p(eps), ld, Bimg, C, HW, guidance, s_img, phi, _p(scratch), _p(factor))


def inpaint_blend(x, ref, noise, mask, n, sqrt_a, sqrt_1ma) -> None:
    _call("sdxl_test_inpaint_blend", _p(x), _p(ref), _p(noise), _p(mask), n, sqrt_a, sqrt_1ma)


def axpby(x, noise, n, sa, sb) -> None:
    _call("sdxl_test_axpby", _p(x), _p(noise), n, sa, sb)


def cast_f32_to_f16(x, n, y) -> None:
    _call("sdxl_test_cast_f32_to_f16", _p(x), n, _p(y))


def cast_f16_to_f32(x, n, y) -> None:
    _call("sdxl_test_cast_f16_to_f32", _p(x), n, _p(y))


def upsample2x(x, B, H, W, C, y) -> None:
    _call("sdxl_test_upsample2x", _p(x), B, H, W, C, _p(y))


def phase_split(x, B, H, W, C, y) -> None:
    _call("sdxl_test_phase_split", _p(x), B, H, W, C, _p(y))


def silu_f16(x, B, H, W, C, phase, y) -> None:
    _call("sdxl_test_silu_f16", _p(x), B, H, W, C, int(phase), _p(y))


def nhwc_to_nchw(x, B, HW, C, ldx, y) -> None:
    """f16 or f32 y [B, C, HW] from x f32 [B, HW, ldx][..., :C], by y's dtype."""
    name = "sdxl_test_nhwc_to_nchw_f32" if y.dtype == torch.float32 else "sdxl_test_nhwc_to_nchw_f16"
    _call(name, _p(x), B, HW, C, ldx, _p(y))


def scale_weights(w, nw, b, nb, s, wo, bo) -> None:
    _call("sdxl_test_scale_weights", _p(w), nw, _p(b), nb, s, _p(wo), _p(bo))


def vec_add_f32(dst, src, n) -> None:
    _call("sdxl_test_vec_add_f32", _p(dst), _p(src), n)


def guided_step(eps: Optional[torch.Tensor], ld: int, Bimg: int, Cc: int, HW: int, use_cfg: bool, use_pag: bool, guidance: float, p_t: float,
                sigma: float, coef: Sequence[float], xh: torch.Tensor, x_in: torch.Tensor, hist: Optional[torch.Tensor] = None,
                write_hist: bool = False, z: Optional[torch.Tensor] = None, zb: Optional[torch.Tensor] = None, seed: int = 0,
                z_subseq: int = 0, zb_subseq: int = 0, mask: Optional[torch.Tensor] = None, ref: Optional[torch.Tensor] = None,
                sigma_blend: float = 0.0) -> None:
    """coef = (cx, cd, ch, cn, c_in); xh, x_in and hist are updated in place (kernels.h: GuidedStepParams)."""
    _call("sdxl_test_guided_step", _p(eps), ld, Bimg, Cc, HW, int(use_cfg), int(use_pag), guidance, p_t, sigma, *[float(v) for v in coef],
          _p(xh), _p(x_in), _p(hist), int(write_hist), _p(z), _p(zb), seed, z_subseq, zb_subseq, _p(mask), _p(ref), sigma_blend)


def guided_step_pred(eps, ld, Bimg, Cc, HW, use_cfg, use_pag, guidance, p_t, sigma, coef, xh, x_in, hist=None, write_hist=False, z=None,
                     zb=None, seed=0, z_subseq=0, zb_subseq=0, mask=None, ref=None, sigma_blend=0.0, v=False, factor=None) -> None:
    """guided_step with the v prediction (v: D from schedule.h's d_scale at sigma) and the per-image guidance-rescale factors."""
    _call("sdxl_test_guided_step_pred", _p(eps), ld, Bimg, Cc, HW, int(use_cfg), int(use_pag), guidance, p_t, sigma,
          *[float(c) for c in coef], _p(xh), _p(x_in), _p(hist), int(write_hist), _p(z), _p(zb), seed, z_subseq, zb_subseq, _p(mask),
          _p(ref), sigma_blend, int(v), _p(factor))


def timestep_embedding_f32(t: torch.Tensor, dim: int, max_period: float = 10000.0) -> torch.Tensor:
    out = torch.empty(t.numel(), dim, device=t.device, dtype=torch.float32)
    _call("sdxl_test_timestep_embedding_f32", _p(t), t.numel(), dim, max_period, _p(out))
    return out


def guided_step_rows(eps, ld, Bimg, Cc, HW, use_cfg, use_pag, guidance, p_t, sigma, coef, rows, xh, x_in, hist=None, h2=None, xs=None,
                     write_hist=False, write_xs=False, shift=False, z=None, zb=None, seed=0, z_subseq=0, zb_subseq=0, mask=None, ref=None,
                     sigma_blend=0.0, v=False, factor=None) -> None:
    """The step kernel's two-row form (kernels.h: StepRows): coef = (cx, cs, cd, ch, ch2, cn, c_in), rows = (sx, ss, sd, sh, sh2);
    xh, x_in, xs, hist and h2 are updated in place."""
    cx, cs, cd, ch, ch2, cn, c_in = [float(c) for c in coef]
    rc, sr = (C.c_float * 2)(cs, ch2), (C.c_float * 5)(*[float(c) for c in rows])
    _call("sdxl_test_guided_step_rows", _p(eps), ld, Bimg, Cc, HW, int(use_cfg), int(use_pag), guidance, p_t, sigma, cx, cd, ch, cn, c_in,
          _p(xh), _p(x_in), _p(hist), int(write_hist), _p(z), _p(zb), seed, z_subseq, zb_subseq, _p(mask), _p(ref), sigma_blend, int(v),
          _p(factor), _p(xs), _p(h2), rc, sr, int(write_xs), int(shift))


def guided_step_img(eps, ld, Bimg, Cc, HW, guidance, s_img, sigma, coef, xh, x_in, hist=None, write_hist=False, z=None, seed=0, z_subseq=0,
                    v=False, factor=None, rows=None, h2=None, xs=None, write_xs=False, shift=False) -> None:
    """The step kernel with image guidance on the eps rows [cond | img | uncond]. rows None: the one-row form, coef = (cx, cd, ch, cn,
    c_in); else the two-row form as guided_step_rows, coef = (cx, cs, cd, ch, ch2, cn, c_in), rows = (sx, ss, sd, sh, sh2)."""
    if rows is None:
        cx, cd, ch, cn, c_in = [float(c) for c in coef]
        cs = ch2 = 0.0
        rows = (0.0,) * 5
        use_rows = 0
    else:
        cx, cs, cd, ch, ch2, cn, c_in = [float(c) for c in coef]
        use_rows = 1
    rc, sr = (C.c_float * 2)(cs, ch2), (C.c_float * 5)(*[float(c) for c in rows])
    _call("sdxl_test_guided_step_img", _p(eps), ld, Bimg, Cc, HW, guidance, s_img, sigma, cx, cd, ch, cn, c_in, _p(xh), _p(x_in), _p(hist),
          int(write_hist), _p(z), seed, z_subseq, int(v), _p(factor), use_rows, _p(xs), _p(h2), rc, sr, int(write_xs), int(shift))


STAGE_FIELDS = ("t", "sigma", "sigma_next", "cx", "cs", "cd", "ch", "ch2", "cn", "sx", "ss", "sd", "sh", "sh2", "c_in", "write_xs", "hist")


def step_stages(alphas, schedule_struct, k: int, t, sig, n_hist: int) -> list:
    """schedule.h's step_stages on the host: one dict of STAGE_FIELDS per stage; "hist" is write_hist + 2 * shift. Needs no GPU."""
    import numpy as np
    a = np.ascontiguousarray(alphas, dtype=np.float64)
    t, sig = np.ascontiguousarray(t, dtype=np.float64), np.ascontiguousarray(sig, dtype=np.float64)
    out = (C.c_double * 34)()
    n = load().sdxl_test_step_stages(a.ctypes.data, a.size, C.byref(schedule_struct), k, t.ctypes.data, sig.ctypes.data, n_hist, out)
    return [dict(zip(STAGE_FIELDS, out[17 * i:17 * (i + 1)])) for i in range(n)]
