"""The VAE, text / vision-encoder, T2I-Adapter and sampler kernels, launched one at a time and compared with a float64 reference.

The whole-model tests (test_vae_gpu.py, test_clip_gpu.py, test_t2i_adapter_gpu.py, the sampler goldens) reach these kernels only
after dozens of GEMMs and norms, under tolerances set by network-level f16 error. Here each launcher is reached through the
test-only library (sdxl_b200._testing) at real SDXL shapes and at the edges where such kernels break: both sides of each shared
memory branch, tails that are not a multiple of the vector width, grids capped below the work (the grid-stride loops), pitches
wider than the rows, and the timestep gate and error flag.

Every reference is float64 on the exact operands the kernel reads, and every tolerance is an elementwise bound derived from the
kernel's arithmetic (each test's docstring gives it):
  - u = 2^-24 is the f32 unit roundoff; one rounded f32 operation contributes u times its result's magnitude;
  - one f16 output rounding: 2^-11 relative, 2^-25 absolute below the f16 normal range;
  - nvcc contracts a*b + c into an FMA (-O3 without --fmad=false), so a bound for a*b + c*d covers both evaluation orders.
Copies, layout changes, casts and kernels whose rounding order is fixed (one IEEE operation per element, or a fixed chain) are
compared bit for bit against a float32 replay. Outputs are written into oversized buffers filled with a sentinel (NaN, or 0xAB
bytes for u8), and nothing outside the logical output, pitch padding included, may change.
"""
import math

import numpy as np
import pytest
import torch

from sdxl_b200 import SdxlError
from sdxl_b200 import _testing as T

pytestmark = pytest.mark.gpu

U24 = 2.0 ** -24      # f32 unit roundoff
H11 = 2.0 ** -11      # f16 unit roundoff
H_SUB = 2.0 ** -25    # half the f16 subnormal spacing
LN2 = math.log(2.0)
LOG2E = 1.4426950408889634
CAP8, CAP16 = 132 * 8 * 256, 132 * 16 * 256   # threads of a grid capped at 132 * 8 / 132 * 16 blocks of 256
GUARD = 4096          # sentinel elements after every output
DEV = "cuda"


@pytest.fixture(autouse=True, scope="module")
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def f32(v: float) -> float:
    """The f32 value a ctypes c_float argument carries."""
    return float(np.float32(v))


def gen(seed: int) -> torch.Generator:
    return torch.Generator().manual_seed(seed)


def randn(g, *shape, scale=1.0, shift=0.0) -> torch.Tensor:
    return torch.randn(*shape, generator=g) * scale + shift


def check(out: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor, what: str) -> None:
    err = (out.double() - ref).abs()
    bad = ~(err <= tol)                                     # a NaN output is outside every bound
    worst = float((err / tol.clamp_min(1e-300)).nan_to_num(float("inf")).max())
    print(f"{what}: max err {float(err.max()):.3e}, worst err / bound {worst:.3f}")
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements outside the bound (worst err / bound {worst:.2f})"


def f16_bound(y: torch.Tensor, e32: torch.Tensor) -> torch.Tensor:
    """f32 evaluation error e32 of y, then one f16 rounding of the computed value (|y| + e32)."""
    return e32 + (y.abs() + e32) * H11 + H_SUB


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.view({torch.float16: torch.int16, torch.float32: torch.int32, torch.uint8: torch.uint8}[t.dtype])


def same_bits(out: torch.Tensor, ref: torch.Tensor, what: str) -> None:
    o, r = bits(out.cpu().contiguous()), bits(ref.cpu().contiguous())
    assert o.shape == r.shape, f"{what}: shape {tuple(o.shape)} != {tuple(r.shape)}"
    bad = o != r
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {o.numel()} elements differ, first at {int(bad.view(-1).nonzero()[0])}"
    print(f"{what}: {o.numel()} elements bit-exact")


def buf(n: int, dtype=torch.float32) -> torch.Tensor:
    """An output buffer of n logical elements and GUARD sentinel ones (NaN; 0xAB bytes for u8)."""
    if dtype == torch.uint8:
        return torch.full((n + GUARD,), 0xAB, dtype=dtype, device=DEV)
    return torch.full((n + GUARD,), float("nan"), dtype=dtype, device=DEV)


def untouched(b: torch.Tensor, what: str, mask: torch.Tensor = None) -> None:
    """The sentinel is intact in b (in b[mask] if given)."""
    v = b if mask is None else b[mask]
    ok = (v == 0xAB).all() if b.dtype == torch.uint8 else v.isnan().all()
    assert bool(ok), f"{what}: {int((~(v == 0xAB) if b.dtype == torch.uint8 else ~v.isnan()).sum())} sentinel elements overwritten"


def on_dev(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().to(DEV)


def pad_cols(m: torch.Tensor, ld: int, fill=float("nan")) -> torch.Tensor:
    """[rows, cols] -> [rows, ld] with columns cols.. filled."""
    out = torch.full((m.shape[0], ld), fill, dtype=m.dtype)
    out[:, :m.shape[1]] = m
    return out


# ------------------------------------------------------------------------------------------------------------------------------
# latent decoder / encoder (vae_kernels.cu)
# ------------------------------------------------------------------------------------------------------------------------------
def softmax_logits(g, rows: int, cols: int) -> torch.Tensor:
    """Score rows of the VAE's single-head attention plus the edges: ordinary scores, scores in the thousands (a large
    dynamic range after scaling), a row of equal values, rows with -inf entries, one dominant entry."""
    S = randn(g, rows, cols, scale=20.0)
    S[1] = randn(g, cols, scale=3000.0)
    S[2] = 123.5
    S[3, ::3] = float("-inf")
    S[4, 1::2] = float("-inf")
    S[4, 0] = float("-inf")
    S[5] = randn(g, cols, scale=2.0)
    S[5, cols // 2] = 5000.0
    return S


@pytest.mark.parametrize("cols", [4, 12280, 12284, 12288, 12292, 40960, 40964, 15360, 15808, 16128, 16384])
def test_softmax_rows(cols):
    """softmax_rows at the columns on both sides of its two branches: the row is cached in shared memory when cols * 4 <= 160 KB
    (40960 cached, 40964 not), with the opt-in when the cached row and the kernel's 32-byte reduction buffer exceed the 48 KB
    default (12280 fits without it; 12284 and 12288, the scores of a 96 x 128 latent, need it: the launch used to fail there
    with cudaErrorInvalidValue). S and P have pitches wider than cols (NaN in S's padding: reading it would poison the row);
    scale 1/sqrt(512) as the decoder's attention.

    Bound, per element of a row with max m: the kernel evaluates exp2f(fmaf(s, c', -m c')) with c' = f32(f32(scale) * f32(log2 e))
    (2 roundings) and m c' rounded, so the exponent a = (s - m) c is off by (2^-23 + 2^-24) |a| + 2^-24 |m c|, a relative error
    2^da - 1 of the term, plus exp2f's 2 ulp (2^-22). The f32 sum has depth cols / 1024 + 15 (a thread's float4 chain, 5 shuffle
    levels, 8 warps): the sum's relative error is sum(q d) / sum(q) + depth u. 1 / sum and the product add 2u; then one f16
    rounding. -inf entries must give exactly 0."""
    g = gen(cols)
    rows = 6
    lds, ldp = cols + 8, cols + 12
    S = softmax_logits(g, rows, cols)
    Sd = on_dev(pad_cols(S, lds))
    scale = 1.0 / math.sqrt(512.0)
    P = buf(rows * ldp, torch.float16)
    T.softmax_rows(Sd, lds, rows, cols, scale, P, ldp)
    torch.cuda.synchronize()
    x = S.double()
    c = f32(scale) * LOG2E
    m = x.amax(dim=1, keepdim=True)
    a = (x - m) * c
    q = torch.exp2(a)
    p = q / q.sum(dim=1, keepdim=True)
    fin = torch.isfinite(x)
    a_abs = torch.where(fin, a.abs(), torch.zeros_like(a))
    da = (2.0 ** -23 + U24) * a_abs + U24 * (m.abs() * c)
    d = torch.expm1(LN2 * da) + 2.0 ** -22
    depth = math.ceil(cols / 1024) + 15
    dsum = (q * d).sum(dim=1, keepdim=True) / q.sum(dim=1, keepdim=True) + depth * U24 * (1 + d.amax(dim=1, keepdim=True))
    e32 = p * (d + dsum + 2 * U24) * (1 + 2.0 ** -20)
    tol = torch.where(fin, f16_bound(p, e32), torch.zeros_like(p))
    Pm = P[:rows * ldp].view(rows, ldp).cpu()
    check(Pm[:, :cols], p, tol, f"softmax_rows cols={cols}")
    untouched(Pm[:, cols:], f"softmax_rows cols={cols}: P pitch padding")
    untouched(P[rows * ldp:], f"softmax_rows cols={cols}: after P")


@pytest.mark.parametrize("rows,cols,ldx,ldy", [
    (100, 70, 72, 102),            # neither a multiple of 64, both pitches wider
    (129, 65, 66, 130),            # odd rows (the scalar store tail) and odd cols (the scalar load tail)
    (127, 63, 64, 132),
    (1, 1, 2, 2),
    (64, 64, 64, 64),
    (16384, 512, 512, 16384),      # the decoder's V at 1024 x 1024 (T = 128^2, C = 512)
])
def test_transpose_f16(rows, cols, ldx, ldy):
    """transpose_f16: y[c, r] = x[r, c], bit-exact; y's padding columns r >= rows and everything after y keep the sentinel."""
    g = gen(rows * 7 + cols)
    x = pad_cols(randn(g, rows, cols).half(), ldx, float("nan"))
    y = buf(cols * ldy, torch.float16)
    T.transpose_f16(on_dev(x), ldx, rows, cols, y, ldy)
    torch.cuda.synchronize()
    ym = y[:cols * ldy].view(cols, ldy)
    same_bits(ym[:, :rows], x[:, :cols].t(), f"transpose_f16 {rows}x{cols} ldx={ldx} ldy={ldy}")
    untouched(ym[:, rows:], "transpose_f16: y pitch padding")
    untouched(y[cols * ldy:], "transpose_f16: after y")


@pytest.mark.parametrize("B,C,HW", [(1, 4, 128 * 128), (2, 3, 1000), (5, 4, 256 * 256), (5, 8, 256 * 256)])
def test_post_quant(B, C, HW):
    """post_quant_conv on the rescaled latent: y[b, o] = bias[o] + sum_c w[o, c] (x[b, c] * f32(1 / 0.13025)). B * HW = 5 * 256^2
    exceeds the grid cap (132 * 8 blocks of 256). Bound: the rescale rounds once, the fmaf chain C times, the bias add once:
    (C + 2) u (sum_c |w x s| + |bias|)."""
    g = gen(B * C + HW)
    x = randn(g, B, C, HW, scale=4.0)
    w = randn(g, C, C, scale=0.5)
    b = randn(g, C, scale=0.2)
    s = f32(1.0 / 0.13025)
    y = buf(B * C * HW)
    T.post_quant(on_dev(x), B, C, HW, on_dev(w), on_dev(b), s, y)
    torch.cuda.synchronize()
    xs = x.double() * s
    ref = torch.einsum("oc,bcp->bop", w.double(), xs) + b.double()[None, :, None]
    mag = torch.einsum("oc,bcp->bop", w.double().abs(), xs.abs()) + b.double().abs()[None, :, None]
    check(y[:B * C * HW].view(B, C, HW).cpu(), ref, (C + 2) * U24 * mag, f"post_quant B={B} C={C} HW={HW}")
    untouched(y[B * C * HW:], "post_quant: after y")


@pytest.mark.parametrize("B,Cz,Cout,HW", [(1, 8, 4, 128 * 128), (5, 8, 4, 256 * 256), (5, 16, 4, 256 * 256), (2, 16, 16, 999)])
def test_quant_out(B, Cz, Cout, HW):
    """quant_conv's first Cout channels times the scale factor: y[b, o, p] = (bias[o] + sum_c w[o, c] x[b, p, c]) * f32(0.13025),
    NHWC in, NCHW out; 5 * 256^2 pixels exceed the grid cap. Bound: Cz fmaf roundings, the bias add and the scale product:
    (Cz + 2) u (sum_c |w x| + |bias|) |scale|."""
    g = gen(B * Cz + Cout + HW)
    x = randn(g, B, HW, Cz, scale=3.0)
    w = randn(g, Cz, Cz, scale=0.4)
    b = randn(g, Cz, scale=0.2)
    s = f32(0.13025)
    y = buf(B * Cout * HW)
    T.quant_out(on_dev(x), B, Cz, Cout, HW, on_dev(w), on_dev(b), s, y)
    torch.cuda.synchronize()
    wd = w.double()[:Cout]
    ref = (torch.einsum("oc,bpc->bop", wd, x.double()) + b.double()[:Cout, None]) * s
    mag = (torch.einsum("oc,bpc->bop", wd.abs(), x.double().abs()) + b.double()[:Cout, None].abs()) * s
    check(y[:B * Cout * HW].view(B, Cout, HW).cpu(), ref, (Cz + 2) * U24 * mag, f"quant_out B={B} Cz={Cz} Cout={Cout} HW={HW}")
    untouched(y[B * Cout * HW:], "quant_out: after y")


def image_u8_replay(x: np.ndarray) -> np.ndarray:
    """The reference's conversion replayed in f32: trunc(clamp(((x + 1) / 2) * 255, 0, 255)), NaN -> 0."""
    with np.errstate(invalid="ignore", over="ignore"):
        v = ((x + np.float32(1)) / np.float32(2)) * np.float32(255)
        v = np.where(v >= 0, np.minimum(v, np.float32(255)), np.float32(0))
    return v.astype(np.uint8)


def run_image_u8(vals: np.ndarray, ldx: int = 4):
    """vals f32 [npix, 3] -> (kernel output u8 [npix * 3], replay, the output buffer); channel 3 of the pitch holds NaN."""
    npix = vals.shape[0]
    x = np.full((npix, ldx), np.nan, dtype=np.float32)
    x[:, :3] = vals
    out = buf(npix * 3, torch.uint8)
    T.image_u8(on_dev(torch.from_numpy(x)), npix, ldx, out)
    torch.cuda.synchronize()
    return out[:npix * 3].cpu(), torch.from_numpy(image_u8_replay(vals).reshape(-1)), out


def test_image_u8():
    """image_u8 bit-exact against the f32 replay, ldx = 4 as the decoder calls it, over one 1024 x 1024 image (about 1 M pixels:
    twice the 132 * 16-block grid): the value of every integer boundary k = 2k/255 - 1 and its f32 neighbours, +-1 and the
    values just beyond, +-inf, +-0, huge values, and uniform values over [-1.2, 1.2]."""
    g = gen(8)
    k = np.arange(256, dtype=np.float64)
    edge = (2 * k / 255 - 1).astype(np.float32)
    special = np.concatenate([edge, np.nextafter(edge, np.float32(-2)), np.nextafter(edge, np.float32(2)),
                              np.array([1, -1, np.nextafter(np.float32(1), np.float32(2)), np.nextafter(np.float32(-1), np.float32(-2)),
                                        np.inf, -np.inf, 0.0, -0.0, 1e30, -1e30, 3.4e38, -3.4e38, 1e-40, -1e-40], dtype=np.float32)])
    npix = 1024 * 1024
    vals = (torch.rand(npix * 3, generator=g) * 2.4 - 1.2).numpy().astype(np.float32)
    vals[:special.size] = special
    vals[-special.size:] = special[::-1]
    got, ref, out = run_image_u8(vals.reshape(npix, 3))
    same_bits(got, ref, "image_u8 1024x1024")
    untouched(out[npix * 3:], "image_u8: after the image")


def test_image_u8_nan_is_zero():
    """A NaN channel becomes 0, as the kernel documents (fminf / fmaxf return the non-NaN operand, so a clamp written with them
    alone turns NaN into 255)."""
    vals = np.array([[np.nan, 0.0, 1.0], [1.0, np.nan, -1.0], [-1.0, 1.0, np.nan], [np.nan, np.nan, np.nan]], dtype=np.float32)
    got, ref, out = run_image_u8(vals)
    assert ref.tolist() == [0, 127, 255, 255, 0, 0, 0, 255, 0, 0, 0, 0]
    same_bits(got, ref, "image_u8 NaN pixels")
    untouched(out[vals.size:], "image_u8 NaN: after the image")


@pytest.mark.parametrize("B,HW", [(1, 256), (2, 300_000)])
def test_image_from_u8(B, HW):
    """image_from_u8 bit-exact against the f32 replay ((v / 255) * 2) - 1 for all 256 values; 2 * 300000 pixels exceed the grid
    cap. (A contraction of the last two steps into fmaf(q, 2, -1) is exact: q * 2 is.)"""
    g = gen(B + HW)
    v = torch.randint(0, 256, (B, HW, 3), generator=g, dtype=torch.uint8)
    v.view(-1)[:256] = torch.arange(256, dtype=torch.uint8)
    out = buf(B * 3 * HW)
    T.image_from_u8(on_dev(v), B, HW, out)
    torch.cuda.synchronize()
    vn = v.numpy().astype(np.float32)
    ref = (vn / np.float32(255)) * np.float32(2) - np.float32(1)
    same_bits(out[:B * 3 * HW].view(B, 3, HW), torch.from_numpy(ref).permute(0, 2, 1), f"image_from_u8 B={B} HW={HW}")
    untouched(out[B * 3 * HW:], "image_from_u8: after the output")


# ------------------------------------------------------------------------------------------------------------------------------
# text / vision encoders (clip_kernels.cu)
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [768, 1280])
def test_embed_tokens(C):
    """embed_tokens for both text encoders (n_vocab 49408, 2 prompts of 77 tokens): x = f32(tok[id]) + f32(pos[t]), one IEEE add,
    bit-exact. Valid ids leave *err untouched; ids -1 and n_vocab set it to 1 and read row 0; the flag stays set across later
    launches with valid ids."""
    g = gen(C)
    n_vocab, T_, rows = 49408, 77, 2 * 77
    tok = randn(g, n_vocab, C, scale=0.02).half()
    tok[0] = randn(g, C, scale=30.0).half()                   # large entries: the f32 add rounds
    pos = randn(g, T_, C, scale=0.01).half()
    tok_d, pos_d = on_dev(tok), on_dev(pos)
    ids = torch.randint(0, n_vocab, (rows,), generator=g, dtype=torch.int32)
    ids[0], ids[1], ids[77] = 0, n_vocab - 1, 0

    def run(idv, err):
        x = buf(rows * C)
        T.embed_tokens(on_dev(idv), rows, T_, C, n_vocab, tok_d, pos_d, x, err)
        torch.cuda.synchronize()
        untouched(x[rows * C:], "embed_tokens: after x")
        return x[:rows * C].view(rows, C).cpu()

    def ref(idv):
        safe = torch.where((idv < 0) | (idv >= n_vocab), torch.zeros_like(idv), idv).long()
        return tok[safe].float() + pos[torch.arange(rows) % T_].float()

    err = torch.zeros(1, dtype=torch.int32, device=DEV)
    same_bits(run(ids, err), ref(ids), f"embed_tokens C={C}")
    assert int(err.item()) == 0, "valid ids must leave *err untouched"
    bad = ids.clone()
    bad[5], bad[80] = -1, n_vocab
    same_bits(run(bad, err), ref(bad), f"embed_tokens C={C} with ids -1 and n_vocab (read as id 0)")
    assert int(err.item()) == 1, "an id outside [0, n_vocab) must set *err to 1"
    same_bits(run(ids, err), ref(ids), f"embed_tokens C={C} after an error")
    assert int(err.item()) == 1, "*err must stay set across launches"


@pytest.mark.parametrize("p,Kpad", [(14, 640), (16, 768), (16, 832)])
def test_patchify(p, Kpad):
    """patchify at S = 224 (CLIP ViT-H/14 and a /16 tower), N = 2: row n G^2 + py G + px, column (c, kh, kw), f16 rounded, bit-exact;
    the padding columns K..Kpad are written as zeros."""
    g = gen(p + Kpad)
    N, S = 2, 224
    G, K = S // p, 3 * p * p
    px = randn(g, N, 3, S, S, scale=2.0)
    y = buf(N * G * G * Kpad, torch.float16)
    T.patchify(on_dev(px), N, S, p, Kpad, y)
    torch.cuda.synchronize()
    ref = torch.zeros(N * G * G, Kpad, dtype=torch.float16)
    ref[:, :K] = px.view(N, 3, G, p, G, p).permute(0, 2, 4, 1, 3, 5).reshape(N * G * G, K).half()
    same_bits(y[:N * G * G * Kpad].view(N * G * G, Kpad), ref, f"patchify p={p} Kpad={Kpad}")
    untouched(y[N * G * G * Kpad:], "patchify: after y")


def ln_ref(x: torch.Tensor, ex: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float, depth: int):
    """float64 LayerNorm of the rows of x (exact), and the bound on a two-pass f32 evaluation that reads x with an error <= ex,
    sums with tree depth `depth`, divides by C, and forms (x - mean) * rstd * gamma + beta:
      mean: |dm| <= (sum ex + depth u sum |x|) / C + u |mean|;
      d = x - mean: |dd| <= ex + dm + u |d|;
      sum d^2: |dq| <= sum (2 |d| dd + dd^2) + depth u sum d^2 (fmaf chain and tree);
      rstd = 1 / sqrtf(q / C + eps): relative 0.5 (dq / C) / (var + eps) + 0.5 * 2u (divide, add) + 2u (sqrt, reciprocal);
      y: |gamma| rstd (dd + |d| e_rstd) + 3u (|d rstd gamma| + |beta|)."""
    C = x.shape[-1]
    mean = x.mean(dim=-1, keepdim=True)
    d = x - mean
    var = (d * d).mean(dim=-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    g, b = gamma.double(), beta.double()
    y = d * rstd * g + b
    dm = (ex.sum(dim=-1, keepdim=True) + depth * U24 * x.abs().sum(dim=-1, keepdim=True)) / C + U24 * mean.abs()
    dd = ex + dm + U24 * d.abs()
    dq = (2 * d.abs() * dd + dd * dd).sum(dim=-1, keepdim=True) + depth * U24 * (d * d).sum(dim=-1, keepdim=True)
    er = 0.5 * (dq / C) / (var + eps) + 3 * U24
    tol = g.abs() * rstd * (dd + d.abs() * er) + 3 * U24 * ((d * rstd * g).abs() + b.abs())
    return y, tol * (1 + 2.0 ** -20)


@pytest.mark.parametrize("C", [1280, 1664])
def test_vision_embed_ln(C):
    """vision_embed_ln for the ViT-H (1280) and ViT-bigG (1664) towers, N = 2 images of T = 257 tokens: LayerNorm of
    [class ; patches] + position, with class and position embeddings offset by up to 40 (a one-pass variance would cancel).
    The output is f32: the bound is ln_ref's, with the input sum's rounding (u |cls or patch + pos|) and the block's
    tree depth (C / 256 per thread, 5 shuffle levels, 8 warps)."""
    g = gen(C)
    N, T_ = 2, 257
    patches = randn(g, N * (T_ - 1), C, scale=2.0, shift=-1.0)
    cls = randn(g, C, shift=40.0).half()
    pos = (randn(g, T_, C) + 25.0 * (torch.arange(T_) % 3 - 1.0)[:, None]).half()
    gamma, beta = 1 + 0.2 * randn(g, C), 0.1 * randn(g, C)
    eps = f32(1e-5)
    x = buf(N * T_ * C)
    T.vision_embed_ln(on_dev(patches), on_dev(cls), on_dev(pos), N, T_, C, on_dev(gamma), on_dev(beta), eps, x)
    torch.cuda.synchronize()
    src = torch.cat([cls.double()[None].expand(N, 1, C), patches.double().view(N, T_ - 1, C)], dim=1)
    xin = (src + pos.double()[None]).reshape(N * T_, C)
    y, tol = ln_ref(xin, U24 * xin.abs(), gamma, beta, eps, math.ceil(C / 256) + 13)
    check(x[:N * T_ * C].view(N * T_, C).cpu(), y, tol, f"vision_embed_ln C={C}")
    untouched(x[N * T_ * C:], "vision_embed_ln: after x")


def mlp_act_ref(x: torch.Tensor, quick: bool):
    """float64 activation and the bound on its f32 evaluation (before the f16 rounding).
    quick: x / (1 + __expf(-k x)), k = f32(1.702): __expf's error grows with its argument w = k x (2^-21 + |w| 2^-23 relative),
      w itself rounds (|w| 2^-24), 1 + E and the division round once each: 2^-20 (1 + |w|) relative in all.
    erf: 0.5 x (1 + erf_as(z)), z = f32(x * f32(1/sqrt 2)) (|dz| <= 2u |z|). |erf_as - erf| <= 1.5e-7 (Abramowitz-Stegun
      7.1.26) + 1.8e-6 of f32 evaluation (coefficients rounded to f32, the Horner roundings, rcp.approx through |dP/dt| <= 3.5,
      ex2.approx 2^-22 and its argument's roundings) < 2^-18; erf' <= 1.13 carries dz; 1 + erf and the product round once each."""
    if quick:
        k = f32(1.702)
        y = x * torch.sigmoid(k * x)
        return y, 2.0 ** -20 * (1 + (k * x).abs()) * y.abs()
    z = x / math.sqrt(2.0)
    e = torch.erf(z)
    y = 0.5 * x * (1 + e)
    de = 2.0 ** -18 + 1.13 * torch.exp(-z * z) * 2 * U24 * z.abs()
    return y, 0.5 * x.abs() * (de + U24 * (1 + e).abs()) + U24 * y.abs()


@pytest.mark.parametrize("quick", [0, 1])
def test_mlp_act(quick):
    """mlp_act in both modes (exact-erf GELU for OpenCLIP-bigG, QuickGELU for CLIP-L) over [-60, 60] and normal values, n above
    132 * 8 * 256 * 4 (the grid cap times four elements per thread). Large negatives drive __expf to inf: the result must be
    -0 or 0, never NaN."""
    g = gen(quick)
    n = CAP8 * 4 + 4 * 1003
    half = n // 2
    x = torch.cat([torch.linspace(-60.0, 60.0, half), randn(g, n - half, scale=3.0)]).float()
    y = buf(n, torch.float16)
    T.mlp_act(on_dev(x), n, quick, y)
    torch.cuda.synchronize()
    out = y[:n].cpu()
    assert not bool(out.isnan().any()), "mlp_act produced NaN"
    assert bool((out[x < -20] == 0).all()), "large negative inputs must give (-)0"
    ref, e32 = mlp_act_ref(x.double(), bool(quick))
    check(out, ref, f16_bound(ref, e32), f"mlp_act quick={quick}")
    untouched(y[n:], "mlp_act: after y")


@pytest.mark.parametrize("C", [768, 1280])
def test_ln_gather_f32(C):
    """ln_gather_f32, the pooled end-of-text feature: y[b] = LayerNorm(x[b T + idx[b]]) in f32 with idx at 0, T - 1 and in
    between; the unselected rows hold NaN. Bound: ln_ref with exact f32 inputs and one warp's depth (C / 32 + 5)."""
    g = gen(C)
    B, T_ = 3, 77
    idx = torch.tensor([0, T_ - 1, 40], dtype=torch.int32)
    x = torch.full((B * T_, C), float("nan"))
    rows = torch.arange(B) * T_ + idx
    x[rows] = randn(g, B, C, scale=2.0, shift=3.0)
    gamma, beta = 1 + 0.2 * randn(g, C), 0.1 * randn(g, C)
    eps = f32(1e-5)
    y = buf(B * C)
    T.ln_gather_f32(on_dev(x), on_dev(idx), B, T_, C, on_dev(gamma), on_dev(beta), eps, y)
    torch.cuda.synchronize()
    xs = x[rows].double()
    ref, tol = ln_ref(xs, torch.zeros_like(xs), gamma, beta, eps, C // 32 + 5)
    check(y[:B * C].view(B, C).cpu(), ref, tol, f"ln_gather_f32 C={C}")
    untouched(y[B * C:], "ln_gather_f32: after y")


# ------------------------------------------------------------------------------------------------------------------------------
# T2I-Adapter (t2i_kernels.cu)
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,C,H,W", [(3, 3, 1024, 768), (3, 1, 1024, 768), (4, 3, 1024, 1024), (1, 3, 16, 32)])
def test_pixel_unshuffle(n, C, H, W):
    """PixelUnshuffle(16) of a hint into conv_in's NHWC operand, bit-exact: channel ci * 256 + i * 16 + j of pixel (y, x) is
    f16(hint[ci, 16 y + i, 16 x + j]). A non-square 1024 x 768 hint; 4 x 3 x 1024^2 exceeds the grid cap."""
    g = gen(n * 100 + C + H + W)
    x = randn(g, n, C, H, W, scale=2.0)
    h, w = H // 16, W // 16
    ne = n * h * w * C * 256
    y = buf(ne, torch.float16)
    T.pixel_unshuffle(on_dev(x), n, C, H, W, y)
    torch.cuda.synchronize()
    ref = x.view(n, C, h, 16, w, 16).permute(0, 2, 4, 1, 3, 5).reshape(n, h, w, C * 256).half()
    same_bits(y[:ne].view(n, h, w, C * 256), ref, f"pixel_unshuffle n={n} C={C} {H}x{W}")
    untouched(y[ne:], "pixel_unshuffle: after y")


@pytest.mark.parametrize("n", [4, 1000, 2 * 64 * 64 * 320, 2 * 32 * 32 * 1280 + 4])
def test_relu_f16(n):
    """y = f16(max(x, 0)), bit-exact; 2 x 64^2 x 320 elements exceed the grid cap (132 * 16 blocks of 4 elements per thread)."""
    g = gen(n)
    x = randn(g, n, scale=3.0)
    y = buf(n, torch.float16)
    T.relu_f16(on_dev(x), n, y)
    torch.cuda.synchronize()
    same_bits(y[:n], x.clamp_min(0).half(), f"relu_f16 n={n}")
    untouched(y[n:], "relu_f16: after y")


@pytest.mark.parametrize("n,H,W,C", [(2, 128, 128, 320), (2, 64, 64, 1280), (1, 6, 10, 4)])
def test_avg_pool2_f16(n, H, W, C):
    """2x2 stride-2 average pool, bit-exact against the f32 replay f16((a + b + c + d) * 0.25) in the kernel's order (top-left,
    top-right, bottom-left, bottom-right); both SDXL shapes exceed the grid cap."""
    g = gen(n + H + W + C)
    x = randn(g, n, H, W, C, scale=2.0)
    ne = n * (H // 2) * (W // 2) * C
    y = buf(ne, torch.float16)
    T.avg_pool2_f16(on_dev(x), n, H, W, C, y)
    torch.cuda.synchronize()
    v = x.view(n, H // 2, 2, W // 2, 2, C)
    ref = ((((v[:, :, 0, :, 0] + v[:, :, 0, :, 1]) + v[:, :, 1, :, 0]) + v[:, :, 1, :, 1]) * 0.25).half()
    same_bits(y[:ne].view(n, H // 2, W // 2, C), ref, f"avg_pool2_f16 n={n} {H}x{W} C={C}")
    untouched(y[ne:], "avg_pool2_f16: after y")


@pytest.mark.parametrize("n_hint", [1, 2])
def test_t2i_add_gate(n_hint):
    """The adapter feature add at level 0 (per_img = 128^2 x 320 floats, B = 4, far beyond the grid cap), with its timestep gate:
    t < t_min leaves x bit-identical; t == t_min and t > t_min add F[b % n_hint], bit-exact against the f32 replay."""
    g = gen(n_hint)
    B, per_img = 4, 128 * 128 * 320
    x0 = randn(g, B, per_img)
    Fh = randn(g, n_hint, per_img, scale=0.5)
    F_d = on_dev(Fh)
    x = buf(B * per_img)
    x[:B * per_img] = on_dev(x0).view(-1)
    t_min = torch.tensor([500], dtype=torch.int32, device=DEV)
    expect = x0.clone()
    for t, applied in ((499, False), (500, True), (501, True), (0, False)):
        T.t2i_add(x, F_d, per_img, B, n_hint, torch.tensor([t], dtype=torch.int32, device=DEV), t_min)
        torch.cuda.synchronize()
        if applied:
            expect = expect + Fh[torch.arange(B) % n_hint]
        same_bits(x[:B * per_img].view(B, per_img), expect, f"t2i_add n_hint={n_hint} t={t} t_min=500")
    untouched(x[B * per_img:], "t2i_add: after x")


# ------------------------------------------------------------------------------------------------------------------------------
# sampler (elementwise.cu)
# ------------------------------------------------------------------------------------------------------------------------------
def sdxl_alphas_cumprod() -> np.ndarray:
    betas = np.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=np.float64) ** 2
    return np.cumprod(1.0 - betas)


def ddim_scalars(t: int, t_prev: int):
    """(sqrt a, sqrt(1 - a), sqrt a_prev, sqrt(1 - a_prev)) as the f32 values the sampler passes (a_prev = 1 past t = 0)."""
    ac = sdxl_alphas_cumprod()
    a = ac[t]
    ap = ac[t_prev] if t_prev >= 0 else 1.0
    return f32(math.sqrt(a)), f32(math.sqrt(1 - a)), f32(math.sqrt(ap)), f32(math.sqrt(1 - ap))


@pytest.mark.parametrize("t,t_prev", [(999, 979), (1, -1)])
@pytest.mark.parametrize("use_cfg", [0, 1])
def test_cfg_ddim(use_cfg, t, t_prev):
    """The guided DDIM update, Bimg = 2 latents of 4 x 128^2, eps rows with pitch ld = 8 > C (NaN in the padding columns):
    e = u + (c - u) g (use_cfg) or c; x = ((x - e s1) / sa) sap + e s1p with the alphas_cumprod of t = 999 (sa ~ 0.07: the
    division amplifies the numerator's error 14x) and t = 1. First-order bound, evaluation order free (FMA or not):
      d = c - u: u |d|;  e: |g| u |d| + 2u (|u| + |d g|);  num = x - e s1: s1 de + 2u (|x| + |e s1|);
      p = num / sa: dnum / sa + u |p|;  out = p sap + e s1p: sap dp + s1p de + 2u (|p sap| + |e s1p|);
    times 1 + 2^-20 for the second-order terms."""
    g = gen(t * 2 + use_cfg)
    Bimg, C, HW, ld = 2, 4, 128 * 128, 8
    guidance = 5.0
    sa, s1, sap, s1p = ddim_scalars(t, t_prev)
    rows = (1 + use_cfg) * Bimg
    eps = torch.full((rows, HW, ld), float("nan"))
    eps[..., :C] = randn(g, rows, HW, C)
    x0 = randn(g, Bimg, C, HW)
    x = buf(Bimg * C * HW)
    x[:Bimg * C * HW] = on_dev(x0).view(-1)
    T.cfg_ddim(on_dev(eps), ld, Bimg, C, HW, use_cfg, guidance, sa, s1, sap, s1p, x)
    torch.cuda.synchronize()
    ec = eps[:Bimg, :, :C].double().permute(0, 2, 1)
    if use_cfg:
        eu = eps[Bimg:, :, :C].double().permute(0, 2, 1)
        d = ec - eu
        e = eu + d * guidance
        de = U24 * guidance * d.abs() + 2 * U24 * (eu.abs() + (d * guidance).abs())
    else:
        e, de = ec, torch.zeros_like(ec)
    xd = x0.double()
    num = xd - e * s1
    dnum = s1 * de + 2 * U24 * (xd.abs() + (e * s1).abs())
    p = num / sa
    dp = dnum / sa + U24 * p.abs()
    ref = p * sap + e * s1p
    tol = (sap * dp + s1p * de + 2 * U24 * ((p * sap).abs() + (e * s1p).abs())) * (1 + 2.0 ** -20)
    check(x[:Bimg * C * HW].view(Bimg, C, HW).cpu(), ref, tol, f"cfg_ddim use_cfg={use_cfg} t={t}")
    untouched(x[Bimg * C * HW:], "cfg_ddim: after x")


@pytest.mark.parametrize("t", [999, 1])
def test_inpaint_blend(t):
    """x = mask ? x : ref sa + noise s1 over n = 131079 elements (not a multiple of 256), 0/1 mask: kept elements are
    bit-identical, blended ones within 2u (|ref sa| + |noise s1|) (a product and a sum, or an fmaf and a product)."""
    g = gen(t)
    n = 131079
    sa, s1, _, _ = ddim_scalars(t, -1)
    x0, ref, noise = randn(g, n, scale=2.0), randn(g, n, scale=2.0), randn(g, n)
    mask = (torch.rand(n, generator=g) < 0.4).to(torch.uint8)
    x = buf(n)
    x[:n] = on_dev(x0)
    T.inpaint_blend(x, on_dev(ref), on_dev(noise), on_dev(mask), n, sa, s1)
    torch.cuda.synchronize()
    out = x[:n].cpu()
    keep = mask.bool()
    same_bits(out[keep], x0[keep], f"inpaint_blend t={t}: masked elements")
    r = ref.double() * sa + noise.double() * s1
    tol = 2 * U24 * ((ref.double() * sa).abs() + (noise.double() * s1).abs())
    check(out[~keep], r[~keep], tol[~keep], f"inpaint_blend t={t}: blended elements")
    untouched(x[n:], "inpaint_blend: after x")


def test_axpby():
    """x = x sa + noise sb (the refiner's entry noise) over n = 131079: within 2u (|x sa| + |noise sb|)."""
    g = gen(5)
    n = 131079
    sa, sb, _, _ = ddim_scalars(700, -1)
    x0, noise = randn(g, n, scale=2.0), randn(g, n)
    x = buf(n)
    x[:n] = on_dev(x0)
    T.axpby(x, on_dev(noise), n, sa, sb)
    torch.cuda.synchronize()
    r = x0.double() * sa + noise.double() * sb
    check(x[:n].cpu(), r, 2 * U24 * ((x0.double() * sa).abs() + (noise.double() * sb).abs()), "axpby")
    untouched(x[n:], "axpby: after x")


F16_EDGES = [0.0, -0.0, 65504.0, 65519.99, 65520.0, -65520.0, 2.0 ** -24, 2.0 ** -25, 1.5 * 2.0 ** -25, 2.0 ** -14, 2.0 ** -14 * 0.999,
             1e-30, float("inf"), float("-inf"), 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11]


def test_casts():
    """cast_f32_to_f16 over n above the grid cap with the rounding edges, bit-exact; cast_f16_to_f32 of every f16 bit pattern,
    bit-exact (NaN stays NaN)."""
    g = gen(6)
    n = CAP16 + 777
    x = randn(g, n, scale=1000.0)
    x[:len(F16_EDGES)] = torch.tensor(F16_EDGES)
    y = buf(n, torch.float16)
    T.cast_f32_to_f16(on_dev(x), n, y)
    torch.cuda.synchronize()
    same_bits(y[:n], x.half(), "cast_f32_to_f16")
    untouched(y[n:], "cast_f32_to_f16: after y")
    pats = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.float16).repeat(9)
    m = pats.numel()
    z = buf(m)
    T.cast_f16_to_f32(on_dev(pats), m, z)
    torch.cuda.synchronize()
    got, ref = z[:m].cpu(), pats.float()
    nan = ref.isnan()
    assert bool(got[nan].isnan().all()), "cast_f16_to_f32: NaN must stay NaN"
    same_bits(got[~nan], ref[~nan], "cast_f16_to_f32 (every f16 bit pattern)")
    untouched(z[m:], "cast_f16_to_f32: after y")


# ------------------------------------------------------------------------------------------------------------------------------
# resampling copies (elementwise.cu)
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,C", [(2, 32, 32, 1280), (2, 64, 64, 640), (1, 3, 5, 4)])
def test_upsample2x(B, H, W, C):
    """Nearest-2x upsample of f32 NHWC into f16, bit-exact; the UNet's two upsample shapes exceed the grid cap."""
    g = gen(B + H + W + C)
    x = randn(g, B, H, W, C, scale=3.0)
    ne = B * 4 * H * W * C
    y = buf(ne, torch.float16)
    T.upsample2x(on_dev(x), B, H, W, C, y)
    torch.cuda.synchronize()
    ref = x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2).half()
    same_bits(y[:ne].view(B, 2 * H, 2 * W, C), ref, f"upsample2x B={B} {H}x{W} C={C}")
    untouched(y[ne:], "upsample2x: after y")


def phase_layout(x: torch.Tensor) -> torch.Tensor:
    """[B, H, W, C] -> the stride-2 phase split [4 (ph * 2 + pw), B, H / 2, W / 2, C]: P[ph][pw][i][j] = x[2i + ph][2j + pw]."""
    B, H, W, C = x.shape
    return x.view(B, H // 2, 2, W // 2, 2, C).permute(2, 4, 0, 1, 3, 5).reshape(4, B, H // 2, W // 2, C)


HINT_SHAPES = [(1, 1024, 1024, 16), (1, 512, 512, 32), (2, 256, 256, 96), (1, 2, 6, 4)]   # before the hint encoder's stride-2 convs


@pytest.mark.parametrize("B,H,W,C", HINT_SHAPES)
def test_phase_split(B, H, W, C):
    """The stride-2 phase split of f32 NHWC into f16, bit-exact, at the ControlNet hint encoder's shapes (above the grid cap)."""
    g = gen(B + H + W + C + 1)
    x = randn(g, B, H, W, C, scale=3.0)
    ne = B * H * W * C
    y = buf(ne, torch.float16)
    T.phase_split(on_dev(x), B, H, W, C, y)
    torch.cuda.synchronize()
    same_bits(y[:ne].view(4, B, H // 2, W // 2, C), phase_layout(x).half(), f"phase_split B={B} {H}x{W} C={C}")
    untouched(y[ne:], "phase_split: after y")


@pytest.mark.parametrize("B,H,W,C", HINT_SHAPES)
def test_silu_f16(B, H, W, C):
    """f16(silu(x)) in both forms: phase = 0 within 2^-20 (1 + |x|) |silu| (x / (1 + __expf(-x)), as in test_fused_paths_gpu.py)
    plus the f16 rounding; phase = 1 bit-identical to the phase = 0 values in phase_split's layout."""
    g = gen(B + H + W + C + 2)
    x = randn(g, B, H, W, C, scale=4.0)
    x.view(-1)[:7] = torch.tensor([-60.0, -20.0, -0.0, 0.0, 20.0, 60.0, 1e-30])
    ne = B * H * W * C
    xd = on_dev(x)
    y0, y1 = buf(ne, torch.float16), buf(ne, torch.float16)
    T.silu_f16(xd, B, H, W, C, 0, y0)
    T.silu_f16(xd, B, H, W, C, 1, y1)
    torch.cuda.synchronize()
    x64 = x.double()
    ref = x64 * torch.sigmoid(x64)
    check(y0[:ne].view(B, H, W, C).cpu(), ref, f16_bound(ref, 2.0 ** -20 * (1 + x64.abs()) * ref.abs()),
          f"silu_f16 B={B} {H}x{W} C={C}")
    same_bits(y1[:ne].view(4, B, H // 2, W // 2, C), phase_layout(y0[:ne].view(B, H, W, C).cpu()),
              f"silu_f16 phase=1 vs phase_split layout of phase=0, B={B} {H}x{W} C={C}")
    untouched(y0[ne:], "silu_f16: after y")
    untouched(y1[ne:], "silu_f16 phase: after y")


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("B,HW,C,ldx", [(1, 1024 * 1024, 3, 4), (2, 128 * 128, 4, 8), (3, 77, 5, 5)])
def test_nhwc_to_nchw(dtype, B, HW, C, ldx):
    """NHWC f32 with channel pitch ldx (the decoder's 4-wide image, the UNet's eps) -> NCHW f16 / f32, bit-exact; the pitch
    padding holds NaN, so reading it would show."""
    g = gen(B + HW + C + ldx)
    x = torch.full((B, HW, ldx), float("nan"))
    x[..., :C] = randn(g, B, HW, C, scale=50.0)
    ne = B * C * HW
    y = buf(ne, dtype)
    T.nhwc_to_nchw(on_dev(x), B, HW, C, ldx, y)
    torch.cuda.synchronize()
    same_bits(y[:ne].view(B, C, HW), x[..., :C].permute(0, 2, 1).to(dtype), f"nhwc_to_nchw {dtype} B={B} HW={HW} C={C} ldx={ldx}")
    untouched(y[ne:], "nhwc_to_nchw: after y")


# ------------------------------------------------------------------------------------------------------------------------------
# load-time helpers (elementwise.cu)
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", [1.0, 0.37])
def test_scale_weights(s):
    """The ControlNet scale folded into a zero conv: wo = f16(s * f32(w)), bo = s * b, bit-exact against the f32 replay. s = 1
    keeps every f16 bit pattern (subnormals and -0 included; NaN stays NaN). nw = 20 x 65536 exceeds the grid cap; a second
    launch with nb > nw checks the bias loop on a one-block grid."""
    g = gen(int(s * 100))
    pats = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.float16)
    for nw, nb in ((20 * 65536, 1280), (100, 1000)):
        w = pats.repeat(20)[:nw] if nw > 65536 else randn(g, nw).half()
        b = randn(g, nb, scale=2.0)
        wo, bo = buf(nw, torch.float16), buf(nb)
        T.scale_weights(on_dev(w), nw, on_dev(b), nb, s, wo, bo)
        torch.cuda.synchronize()
        sf = torch.tensor(f32(s), dtype=torch.float32)
        ref_w = (sf * w.float()).half()
        got = wo[:nw].cpu()
        nan = ref_w.isnan()
        assert bool(got[nan].isnan().all()), "scale_weights: NaN weights must stay NaN"
        same_bits(got[~nan], ref_w[~nan], f"scale_weights s={s} nw={nw} weights")
        if s == 1.0:
            same_bits(got[~nan], w[~nan], f"scale_weights s=1 nw={nw} keeps the weight bits")
        same_bits(bo[:nb], sf * b, f"scale_weights s={s} nb={nb} bias")
        untouched(wo[nw:], "scale_weights: after wo")
        untouched(bo[nb:], "scale_weights: after bo")


@pytest.mark.parametrize("n", [77, 1_000_003])
def test_vec_add_f32(n):
    """dst += src, bit-exact against the f32 replay."""
    g = gen(n)
    a, b = randn(g, n, scale=10.0), randn(g, n)
    dst = buf(n)
    dst[:n] = on_dev(a)
    T.vec_add_f32(dst, on_dev(b), n)
    torch.cuda.synchronize()
    same_bits(dst[:n], a + b, f"vec_add_f32 n={n}")
    untouched(dst[n:], "vec_add_f32: after dst")


# ------------------------------------------------------------------------------------------------------------------------------
# refusals
# ------------------------------------------------------------------------------------------------------------------------------
def refusal_cases(x32, o16, o32, t1):
    """name -> (status, launch) for each documented precondition; every launch is given real buffers."""
    return {
        "softmax_cols": (6001, lambda: T.softmax_rows(x32, 8, 2, 6, 1.0, o16, 8)),
        "softmax_lds": (6001, lambda: T.softmax_rows(x32, 10, 2, 8, 1.0, o16, 8)),
        "softmax_ldp": (6001, lambda: T.softmax_rows(x32, 8, 2, 8, 1.0, o16, 10)),
        "softmax_rows0": (6001, lambda: T.softmax_rows(x32, 8, 0, 8, 1.0, o16, 8)),
        "transpose_ldx": (6002, lambda: T.transpose_f16(o16, 9, 4, 4, o16, 8)),
        "transpose_ldy": (6002, lambda: T.transpose_f16(o16, 8, 4, 4, o16, 9)),
        "transpose_rows0": (6002, lambda: T.transpose_f16(o16, 8, 0, 4, o16, 8)),
        "transpose_cols0": (6002, lambda: T.transpose_f16(o16, 8, 4, 0, o16, 8)),
        "post_quant_C9": (6003, lambda: T.post_quant(x32, 1, 9, 16, x32, x32, 1.0, o32)),
        "post_quant_C0": (6003, lambda: T.post_quant(x32, 1, 0, 16, x32, x32, 1.0, o32)),
        "quant_out_Cz17": (6004, lambda: T.quant_out(x32, 1, 17, 4, 16, x32, x32, 1.0, o32)),
        "quant_out_Cout_gt_Cz": (6004, lambda: T.quant_out(x32, 1, 4, 8, 16, x32, x32, 1.0, o32)),
        "quant_out_Cout0": (6004, lambda: T.quant_out(x32, 1, 4, 0, 16, x32, x32, 1.0, o32)),
        "upsample_C": (2003, lambda: T.upsample2x(x32, 1, 4, 4, 6, o16)),
        "phase_split_C": (2004, lambda: T.phase_split(x32, 1, 4, 4, 6, o16)),
        "phase_split_H": (2004, lambda: T.phase_split(x32, 1, 5, 4, 4, o16)),
        "phase_split_W": (2004, lambda: T.phase_split(x32, 1, 4, 5, 4, o16)),
        "silu_C": (2005, lambda: T.silu_f16(x32, 1, 4, 4, 6, 0, o16)),
        "silu_phase_H": (2005, lambda: T.silu_f16(x32, 1, 5, 4, 4, 1, o16)),
        "silu_phase_W": (2005, lambda: T.silu_f16(x32, 1, 4, 5, 4, 1, o16)),
        "unshuffle_H": (2101, lambda: T.pixel_unshuffle(x32, 1, 1, 24, 16, o16)),
        "unshuffle_W": (2101, lambda: T.pixel_unshuffle(x32, 1, 1, 16, 8, o16)),
        "unshuffle_n0": (2101, lambda: T.pixel_unshuffle(x32, 0, 1, 16, 16, o16)),
        "unshuffle_C0": (2101, lambda: T.pixel_unshuffle(x32, 1, 0, 16, 16, o16)),
        "relu_n": (2102, lambda: T.relu_f16(x32, 6, o16)),
        "avg_pool_C": (2103, lambda: T.avg_pool2_f16(x32, 1, 4, 4, 6, o16)),
        "avg_pool_H": (2103, lambda: T.avg_pool2_f16(x32, 1, 5, 4, 4, o16)),
        "avg_pool_W": (2103, lambda: T.avg_pool2_f16(x32, 1, 4, 5, 4, o16)),
        "avg_pool_n0": (2103, lambda: T.avg_pool2_f16(x32, 0, 4, 4, 4, o16)),
        "t2i_add_per_img": (2104, lambda: T.t2i_add(o32, x32, 6, 2, 1, t1, t1)),
        "t2i_add_B_mod_n_hint": (2104, lambda: T.t2i_add(o32, x32, 8, 3, 2, t1, t1)),
        "t2i_add_n_hint0": (2104, lambda: T.t2i_add(o32, x32, 8, 2, 0, t1, t1)),
        "t2i_add_B0": (2104, lambda: T.t2i_add(o32, x32, 8, 0, 1, t1, t1)),
        "embed_C_odd": (7101, lambda: T.embed_tokens(t1, 1, 1, 7, 10, o16, o16, o32, t1)),
        "mlp_act_n": (7103, lambda: T.mlp_act(x32, 6, 0, o16)),
        "patchify_S_mod_p": (7105, lambda: T.patchify(x32, 1, 15, 2, 16, o16)),
        "patchify_Kpad": (7105, lambda: T.patchify(x32, 1, 16, 2, 11, o16)),
        "patchify_p0": (7105, lambda: T.patchify(x32, 1, 16, 0, 16, o16)),
    }


REFUSALS = list(refusal_cases(None, None, None, None))


@pytest.mark.parametrize("case", REFUSALS)
def test_refusal(case):
    """Each launcher's documented precondition returns its status before any launch: nothing is written."""
    x32 = torch.zeros(4096, device=DEV)
    o16, o32 = buf(0, torch.float16), buf(0)
    t1 = torch.zeros(1, dtype=torch.int32, device=DEV)
    code, launch = refusal_cases(x32, o16, o32, t1)[case]
    with pytest.raises(SdxlError, match=rf"\({code}\)"):
        launch()
    torch.cuda.synchronize()
    untouched(o16, f"{case}: f16 output")
    untouched(o32, f"{case}: f32 output")
    assert int(t1.item()) == 0 and not bool(x32.any()), f"{case}: an input was written"
