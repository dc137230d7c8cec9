"""Every implicit-GEMM form of the VAE, the ControlNet hint encoder, the T2I-Adapter, the text / vision encoders and the IP-Adapter
Plus Resampler, bit for bit on exactly representable operands at the models' real extents.

test_igemm_forms_gpu.py pins the UNet plan's forms. The other models run the same igemm_kernel with parameter sets the UNet never
uses: outputs narrower than any tile (N = 4, 8, 16, 32, 96), K = 16384 (P V of the VAE attention), N = 16384 with an activation
matrix as the weights (q k^T), the VAE encoder's asymmetric stride-2 conv, 1x1 conv taps, 16- and 32-channel inputs of which TMA
zero-fills most of each 64-channel K block, and 77 B / 257 N / 273 n rows. Each test builds its form as the named call site does
(build_vae_plan / build_vae_enc_plan and VaeStage in vae.cu, embed_hint / conv3x3_direct, t2i_forward / conv_nhwc and ip_resample
in engine.cu, clip_block_ops and vision_run in clip.cu): the same repack_conv / repack_upconv / transpose_linear layouts, segment
lists, pitches, output dtypes, and out aliasing res or not. The one tap list with its own geometry, the encoder's PaddedConv2d
downsample, is derived here from the operation's definition rather than copied from the plan.

Extents: the 1024 x 1024 image (latent 128 x 128, VAE attention T = 16384) and the 1216 x 832 bucket (latent 152 x 104,
T = 15808: a ragged last M tile, and an N that only 64-wide tiles divide). More than one image wherever the call site has a batch
offset.

Exact arithmetic, as in test_igemm_forms_gpu.py: activations on the 2^-3 grid, weights on 2^-6, biases and residuals on 2^-9, and
assert_exact_range on every case, so every partial sum is exact in f32 whatever the summation order: f32 outputs must equal the
exact value and f16 outputs its round-to-nearest-even rounding, with zero tolerance. The reference is float64 on the GPU, one
matmul per tap, built in row chunks (at most CHUNK_BYTES each) where the whole of it would not fit beside the operands. Outputs
are pre-filled with NaN and followed by a NaN guard. Three controls show the checks can tell near misses apart: the UNet's
symmetric stride-2 taps on the encoder downsample, image 0's k used for image 1's scores, and P V without its last K block must
all fail the exact comparison.

The file runs in about 15 s on an H100 80GB HBM3 at its 700 W power limit. It catches kernel faults the UNet forms cannot see:
an igemm_kernel that drops a segment's last K block once the segment has more than 128 of them (only P V has), or that skips the
phase-split taps at a positive row / column offset (only PaddedConv2d has them), passes test_igemm_forms_gpu.py and fails here.
"""
import pytest
import torch
import torch.nn.functional as F

from sdxl_b200 import _testing as T
from harness import (DEV, GRID_B, GRID_W, GRID_X, assert_exact, assert_exact_range, bias_f32, conv_bound, conv_taps, gen, grid,
                     guarded, in_place_residual, lin_weights, linear, pad64, plan_upconv, repack3, stride2_taps)

pytestmark = pytest.mark.gpu

CHUNK_BYTES = 256 << 20     # float64 reference rows built at a time
EXTENTS = [(128, 128), (152, 104)]   # latent h x w of the 1024^2 image and of the 1216 x 832 bucket
VAE_C = 512                 # SDXL_VAE mid width: the attention's d


def lean_grid(g, shape, step, lim, dtype=torch.float16) -> torch.Tensor:
    """harness.grid's values (integers in [-lim, lim] times step) without its int64 / float64 intermediates, for operands of up
    to 2^29 elements: int8 / int32 draws, exact in dtype, scaled by a power of two."""
    idt = torch.int8 if lim < 128 else torch.int32
    return torch.randint(-lim, lim + 1, tuple(shape), generator=g, device=DEV, dtype=idt).to(dtype).mul_(step)


def gx(g, *shape):
    return lean_grid(g, shape, GRID_X, 8)


def gw(g, *shape):
    return lean_grid(g, shape, GRID_W, 8)


def gf(g, *shape):
    """f32 residual values on the 2^-9 grid, magnitude <= 2^11."""
    return lean_grid(g, shape, GRID_B, 2 ** 20, torch.float32)


# ------------------------------------------------------------------------------------------------------------------------------
# chunked float64 references
# ------------------------------------------------------------------------------------------------------------------------------
def conv_rows(x, w, r0, r1, stride=1, pad=None, up=False):
    """Output rows [r0, r1) of the exact float64 conv of x [B, H, W, I] (nearest-2x upsampled first when up) with w [O, I, k, k]
    at `stride`, zero padding pad = (top, bottom, left, right) (default k // 2 on every side): conv_ref's one matmul per tap
    over shifted views, of only the input rows the chunk reads. [B, r1 - r0, Wo, O]."""
    B, H, W, _ = x.shape
    if up:
        H, W = 2 * H, 2 * W
    O, _, k, _ = w.shape
    pt, pb, pl, pr = pad if pad is not None else (k // 2,) * 4
    Wo = (W + pl + pr - k) // stride + 1
    lo, hi = r0 * stride - pt, (r1 - 1) * stride - pt + k       # padded input rows [lo, hi) in image coordinates
    a, b = max(lo, 0), min(hi, H)
    if up:
        xs = x[:, a // 2:(b - 1) // 2 + 1].repeat_interleave(2, dim=1)[:, a % 2:a % 2 + b - a].repeat_interleave(2, dim=2)
    else:
        xs = x[:, a:b]
    xp = F.pad(xs.double(), (0, 0, pl, pr, a - lo, hi - b))
    wd = w.double()
    n = r1 - r0
    out = torch.zeros(B, n, Wo, O, dtype=torch.float64, device=x.device)
    for kh in range(k):
        for kw in range(k):
            out += xp[:, kh:kh + stride * (n - 1) + 1:stride, kw:kw + stride * (Wo - 1) + 1:stride] @ wd[:, :, kh, kw].t()
    return out


def inexact(out, ref_fn, rows, dim=0):
    """How many elements of out differ from ref_fn(r0, r1) (the exact float64 value of out.narrow(dim, r0, r1 - r0)) rounded
    once to out's dtype, taken `rows` at a time along dim; and the first such (index, value, exact value)."""
    n_bad, first = 0, None
    for r0 in range(0, out.shape[dim], rows):
        r1 = min(out.shape[dim], r0 + rows)
        o = out.narrow(dim, r0, r1 - r0)
        ref = ref_fn(r0, r1)
        want = ref.float() if o.dtype == torch.float32 else ref.float().half()
        bad = o != want
        nb = int(bad.sum())
        if nb and first is None:
            idx = bad.nonzero()[0].tolist()
            first = (tuple(idx[:dim] + [idx[dim] + r0] + idx[dim + 1:]), float(o[bad][0]), float(want[bad][0]))
        n_bad += nb
        del ref, want, bad
    return n_bad, first


def assert_exact_rows(out, ref_fn, guard, what, rows, dim=0) -> None:
    """harness.assert_exact with the reference built `rows` at a time along dim."""
    n_bad, first = inexact(out, ref_fn, rows, dim)
    print(f"{what}: {out.numel() - n_bad} / {out.numel()} exact")
    assert n_bad == 0, f"{what}: {n_bad} elements differ from the exact value, first at {first[0]}: {first[1]} != {first[2]}"
    assert guard is None or bool(guard.isnan().all()), f"{what}: elements after the output were written"


def assert_control_fails(out, ref_fn, what, rows, dim=0) -> None:
    """A control launch (an in-bounds near miss of the real form) must not match the exact value of the real form."""
    n_bad, _ = inexact(out, ref_fn, rows, dim)
    print(f"{what} (control): {n_bad} / {out.numel()} differ from the exact value")
    assert n_bad > 0, f"{what}: the control matches the reference, so the test cannot tell the two forms apart"


def conv_chunk_rows(out, convs) -> int:
    """Output rows per chunk so that the float64 output and each conv's padded input chunk stay under CHUNK_BYTES."""
    B, _, Wo, O = out.shape
    per_row = B * Wo * O
    for x, _, kw in convs:
        s, up = kw.get("stride", 1), kw.get("up", False)
        per_row = max(per_row, B * (x.shape[2] * (2 if up else 1) + 2) * x.shape[3] * s)
    return max(1, CHUNK_BYTES // (8 * per_row))


def assert_exact_conv(out, guard, what, convs, extra=None) -> None:
    """out [B, Ho, Wo, O] equals sum of conv_rows(x, w, **kw) over convs = [(x, w, kw)] plus extra(r0, r1) (bias / residual),
    built in row chunks."""
    def ref(r0, r1):
        r = sum(conv_rows(x, w, r0, r1, **kw) for x, w, kw in convs)
        return r if extra is None else r + extra(r0, r1)
    assert_exact_rows(out, ref, guard, what, conv_chunk_rows(out, convs), dim=1)


def conv_form(g, a, Cout, ks=3, res=None):
    """One conv launch as PlanBuilder::conv3 / conv_nhwc issue it: a [B, H, W, I] f16, weights repack_conv [Cout, ks^2 Ipad],
    conv_taps(ks) (one 1x1 segment for ks = 1), f32 out (ldo = Cout) + bias_to_f32 bias; with res, the output is pre-filled with
    res and is the residual too (out == res, ldr = ldo). Returns (out, guard, w, b16)."""
    B, H, W, I = a.shape
    w = gw(g, Cout, I, ks, ks)
    b16, b32 = bias_f32(g, Cout)
    Ktot = ks * ks * pad64(I)
    wt = repack3(w, Ktot)
    out, guard = guarded((B, H, W, Cout), fill=res)
    if res is not None:
        res = out
    assert_exact_range("conv", conv_bound(a, w), b16.abs().max(), 0 if res is None else res.abs().max())
    segs = conv_taps(pad64(I) // 64) if ks == 3 else [(0, 0, 0, 0, pad64(I) // 64)]
    T.igemm(a, (B, H, W, I), wt, Cout, Ktot, (W, H, B), segs, out, Cout, bias=b32, res=res, ldr=Cout if res is not None else 0)
    return out, guard, w, b16


def bias_rows(b16, res=None):
    """extra() of assert_exact_conv: the bias, plus the residual's rows when there is one."""
    if res is None:
        return lambda r0, r1: b16.double()
    return lambda r0, r1: b16.double() + res[:, r0:r1].double()


# ------------------------------------------------------------------------------------------------------------------------------
# VAE decoder and encoder
# ------------------------------------------------------------------------------------------------------------------------------
# (scale of the latent extent, Cin, Cout) of the ResnetBlocks: decoder mid / blocks 0..3 (512@1x, 512@2x, 512->256 and 256@4x,
# 256->128 and 128@8x), then the encoder's own width changes (128->256 @4x, 256->512 @2x; its 128@8x and 512@1x are the decoder's)
VAE_RES = [(1, 512, 512), (2, 512, 512), (4, 512, 256), (4, 256, 256), (8, 256, 128), (8, 128, 128), (4, 128, 256), (2, 256, 512)]


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(B, h * s, w * s, ci, co) for h, w in EXTENTS for s, ci, co in VAE_RES for B in (1, 2)])
def test_vae_resblock(ctx, B, H, W, Cin, Cout):
    """VaeStage::vres: conv1 (3x3 Cin -> Cout + bias into s_h), then conv2. With a width change (has_skip) conv2 carries the
    nin_shortcut 1x1 as one more K segment on map 1 (s_raw, GroupNorm's raw f16 copy of the block input): weights
    [Cout, 9 Ipad | I2pad], bias conv2 + nin_shortcut (bias_to_f32, then accumulate). Without, the block input x() is the f32
    residual of a launch writing the other stream buffer (out != res, ldr = ldo = Cout)."""
    g = gen(B, H, W, Cin, Cout, 11)
    a1 = gx(g, B, H, W, Cin)
    out, guard, w1, b1 = conv_form(g, a1, Cout)
    assert_exact_conv(out, guard, f"vae resblock conv1 {B}x{H}x{W} {Cin}->{Cout}", [(a1, w1, {})], bias_rows(b1))
    del a1, out, guard
    a2 = gx(g, B, H, W, Cout)
    w2 = gw(g, Cout, Cout, 3, 3)
    b2, bias = bias_f32(g, Cout)
    Ipad = pad64(Cout)
    out, guard = guarded((B, H, W, Cout))
    if Cin != Cout:
        raw = gx(g, B, H, W, Cin)
        ws = gw(g, Cout, Cin, 1, 1)
        bs = grid(g, (Cout,), GRID_B, 2047)
        T.bias_to_f32(bs, Cout, bias, accumulate=True)
        Ktot = 9 * Ipad + pad64(Cin)
        wt = repack3(w2, Ktot)
        repack3(ws, Ktot, wt, 9 * Ipad)
        assert_exact_range("conv2 + nin_shortcut", conv_bound(a2, w2), conv_bound(raw, ws), b2.abs().max(), bs.abs().max())
        T.igemm(a2, (B, H, W, Cout), wt, Cout, Ktot, (W, H, B), conv_taps(Ipad // 64) + [(1, 0, 0, 0, pad64(Cin) // 64)], out, Cout,
                a1=raw, a1_shape=(B, H, W, Cin), bias=bias)
        assert_exact_conv(out, guard, f"vae resblock conv2 + nin_shortcut {B}x{H}x{W} {Cin}->{Cout}",
                          [(a2, w2, {}), (raw, ws, {})], lambda r0, r1: b2.double() + bs.double())
    else:
        res = gf(g, B, H, W, Cout)
        wt = repack3(w2, 9 * Ipad)
        assert_exact_range("conv2 + identity", conv_bound(a2, w2), b2.abs().max(), res.abs().max())
        T.igemm(a2, (B, H, W, Cout), wt, Cout, 9 * Ipad, (W, H, B), conv_taps(Ipad // 64), out, Cout, bias=bias, res=res, ldr=Cout)
        assert_exact_conv(out, guard, f"vae resblock conv2 + identity into the other buffer {B}x{H}x{W}x{Cout}", [(a2, w2, {})],
                          bias_rows(b2, res))


@pytest.mark.parametrize("B,H,W,C", [(B, h * s, w * s, c) for h, w in EXTENTS for s, c in ((1, 512), (2, 512), (4, 256))
                                     for B in (1, 2)])
def test_vae_upsample_conv(ctx, B, H, W, C):
    """build_vae_plan, each decoder block but the last: PlanBuilder::upconv, the nearest-2x upsample and 3x3 conv as four 2x2
    phase convolutions of the source image (repack_upconv), one launch per output parity through opix: 512@128^2 -> 256^2,
    512@256^2 -> 512^2 and 256@512^2 -> 1024^2."""
    g = gen(B, H, W, C, 12)
    x = gx(g, B, H, W, C)
    w = gw(g, C, C, 3, 3)
    b16, b32 = bias_f32(g, C)
    assert_exact_range("upsample conv", conv_bound(x, w), b16.abs().max())
    out, _ = plan_upconv(x, w, b32)      # NaN-filled, every pixel written by one of the four parity launches
    assert_exact_conv(out, None, f"vae upsample conv {B}x{H}x{W}x{C} -> {2 * H}x{2 * W}", [(x, w, {"up": True})], bias_rows(b16))


def padded_conv_taps(Bn: int, nkb: int):
    """PaddedConv2d(3x3, stride 2, padding right / bottom by one) on the phase split [4][Bn][H/2][W/2][C] of its input (phase
    (h % 2, w % 2) of image b at batch index (2 (h % 2) + w % 2) Bn + b): output (i, j) tap (kh, kw) reads input pixel
    (2 i + kh, 2 j + kw) = phase (kh % 2, kw % 2) at phase pixel (i + kh // 2, j + kw // 2); past the bottom / right edge TMA
    reads zeros."""
    return [(0, kw // 2, kh // 2, (2 * (kh % 2) + kw % 2) * Bn, nkb) for kh in range(3) for kw in range(3)]


@pytest.mark.parametrize("B,H,W,C", [(B, h * s, w * s, c) for h, w in EXTENTS for s, c in ((8, 128), (4, 256), (2, 512))
                                     for B in (1, 2)])
def test_vae_encoder_downsample(ctx, B, H, W, C):
    """build_vae_enc_plan, each encoder block but the last: OP_PHASE (phase_split of the f32 stream) then the 3x3 stride-2 conv
    with the asymmetric padding of PaddedConv2d, as 9 segments with batch offsets phase * Bn. Control: the UNet's Downsample taps
    (stride2_taps, padding 1 on every side) on the same phase split must not match."""
    g = gen(B, H, W, C, 13)
    x = gx(g, B, H, W, C).float()
    w = gw(g, C, C, 3, 3)
    b16, b32 = bias_f32(g, C)
    ph = torch.empty(4 * B, H // 2, W // 2, C, dtype=torch.float16, device=DEV)
    T.phase_split(x, B, H, W, C, ph)
    Ktot = 9 * pad64(C)
    wt = repack3(w, Ktot)
    H2, W2 = H // 2, W // 2
    assert_exact_range("encoder downsample", conv_bound(x, w), b16.abs().max())
    convs = [(x, w, {"stride": 2, "pad": (0, 1, 0, 1)})]
    outs = {}
    for name, segs in (("padded", padded_conv_taps(B, pad64(C) // 64)), ("symmetric", stride2_taps(B, pad64(C) // 64))):
        outs[name] = guarded((B, H2, W2, C))
        T.igemm(ph, (4 * B, H2, W2, C), wt, C, Ktot, (W2, H2, B), segs, outs[name][0], C, bias=b32)
    what = f"vae encoder downsample {B}x{H}x{W}x{C}"
    assert_exact_conv(*outs["padded"], what, convs, bias_rows(b16))
    rows = conv_chunk_rows(outs["symmetric"][0], convs)
    assert_control_fails(outs["symmetric"][0], lambda r0, r1: conv_rows(x, w, r0, r1, **convs[0][2]) + b16.double(),
                         f"{what} with the UNet's symmetric stride2_taps", rows, dim=1)


@pytest.mark.parametrize("h,w", EXTENTS)
def test_vae_mid_attention(ctx, h, w):
    """VaeStage::attn at B = 2 (two images with different q, k, v, P), T = h w, d = 512:
    - q / k / v: 1x1 convs as Linears (lin_from_conv1x1: repack_conv with ks = 1), f16 out + bias, M = 2T;
    - per image b, S = q k^T: A = q rows of image b, the weights the k rows at k16 + b T C (N = T, K = 512), f32 out, ldo = T;
    - per image, P V: A = P [T, T] f16, weights vT = transpose_f16 of image b's v ([512, T], K = T: T / 64 K blocks), f16 out at
      ao + b T C (image 1's rows stay NaN after image 0's launch);
    - proj_out: f32 out + bias + the stream x() as residual, into the other buffer.
    Controls: image 1's scores with image 0's k, and P V without its last K block, must not match."""
    B, C, Tn = 2, VAE_C, h * w
    M = B * Tn
    g = gen(h, w, 14)
    Kp = pad64(C)
    x = gx(g, M, C)
    for name in ("q", "k", "v"):
        wc = gw(g, C, C, 1, 1)
        wt = repack3(wc, Kp)
        b16, b32 = bias_f32(g, C)
        out, guard = guarded((M, C), torch.float16)
        assert_exact_range(name, conv_bound(x, wc), b16.abs().max())
        linear(x, wt, C, Kp, out, C, bias=b32)
        assert_exact(out, x.double() @ wc.view(C, C).double().t() + b16.double(), guard, f"vae attention {name} M={M} (f16)")
    del x, out, guard

    # S = q k^T per image, into one [T, T] f32 buffer the plan reuses
    q, k = gx(g, B, Tn, C), gw(g, B, Tn, C)
    assert_exact_range("q k^T", conv_bound(q, k.view(M, C)))
    S, guard = guarded((Tn, Tn))
    rows = CHUNK_BYTES // (8 * Tn)
    for b in range(B):
        S.fill_(float("nan"))
        T.igemm(q[b], (1, 1, Tn, C), k[b], Tn, Kp, (Tn, 1, 1), [(0, 0, 0, 0, Kp // 64)], S, Tn)
        kd = k[b].double().t()
        assert_exact_rows(S, lambda r0, r1: q[b, r0:r1].double() @ kd, guard, f"vae attention S = q k^T image {b} T={Tn} (f32)", rows)
    S.fill_(float("nan"))
    T.igemm(q[1], (1, 1, Tn, C), k[0], Tn, Kp, (Tn, 1, 1), [(0, 0, 0, 0, Kp // 64)], S, Tn)
    assert_control_fails(S, lambda r0, r1: q[1, r0:r1].double() @ kd, f"vae attention S image 1 with image 0's k T={Tn}", rows)
    del q, k, kd, S, guard

    # O = P v per image, K = T
    v = gw(g, B, Tn, C)
    vT = torch.full((C, Tn), float("nan"), dtype=torch.float16, device=DEV)
    ao, guard = guarded((B, Tn, C), torch.float16)
    rows = CHUNK_BYTES // (8 * Tn)
    for b in range(B):
        P = gx(g, Tn, Tn)
        T.transpose_f16(v[b], C, Tn, C, vT, Tn)
        assert_exact_range("P v", conv_bound(P, vT))
        T.igemm(P, (1, 1, Tn, Tn), vT, C, Tn, (Tn, 1, 1), [(0, 0, 0, 0, Tn // 64)], ao[b], C)
        if b == 0:
            assert bool(ao[1].isnan().all()), "vae attention P v: image 0's launch wrote into image 1's rows"
        vd = v[b].double()
        assert_exact_rows(ao[b], lambda r0, r1: P[r0:r1].double() @ vd, guard if b == B - 1 else None,
                          f"vae attention P v image {b} K={Tn} (f16)", rows)
    short, _ = guarded((Tn, C), torch.float16)
    T.igemm(P, (1, 1, Tn, Tn), vT, C, Tn, (Tn, 1, 1), [(0, 0, 0, 0, Tn // 64 - 1)], short, C)
    assert_control_fails(short, lambda r0, r1: P[r0:r1].double() @ vd, f"vae attention P v without its last K block K={Tn}", rows)
    del v, vT, P, vd, short

    # proj_out: x + proj_out(ao), f32 into the other stream buffer
    wc = gw(g, C, C, 1, 1)
    wt = repack3(wc, Kp)
    b16, b32 = bias_f32(g, C)
    res = gf(g, M, C)
    out, guard = guarded((M, C))
    a = ao.view(M, C)
    assert_exact_range("proj_out", conv_bound(a, wc), b16.abs().max(), res.abs().max())
    linear(a, wt, C, Kp, out, C, bias=b32, res=res)
    assert_exact(out, a.double() @ wc.view(C, C).double().t() + b16.double() + res.double(), guard,
                 f"vae attention proj_out M={M} (f32 + bias + residual)")


@pytest.mark.parametrize("B,H,W", [(B, 8 * h, 8 * w) for h, w in EXTENTS for B in (1, 2)])
def test_vae_decoder_conv_out(ctx, B, H, W):
    """build_vae_plan head: the 3x3 conv 128 -> 3 with O padded to 4 as Loader::conv(Opad = 4) pads it (zero weight row, zero
    bias), N = 4, f32, ldo = 4: column 3 must be exactly the padded bias, 0, and nothing may be written past the last pixel."""
    g = gen(B, H, W, 15)
    Cf = 128
    a = gx(g, B, H, W, Cf)
    w = gw(g, 3, Cf, 3, 3)
    Ktot = 9 * pad64(Cf)
    wt = repack3(w, Ktot, torch.zeros(4 * Ktot, dtype=torch.float16, device=DEV))
    b16 = grid(g, (3,), GRID_B, 2047)
    b32 = torch.zeros(4, dtype=torch.float32, device=DEV)
    T.bias_to_f32(b16, 3, b32)
    w4 = torch.cat([w, torch.zeros_like(w[:1])])
    b4 = torch.cat([b16.double(), torch.zeros(1, dtype=torch.float64, device=DEV)])
    out, guard = guarded((B, H, W, 4))
    assert_exact_range("decoder conv_out", conv_bound(a, w), b16.abs().max())
    T.igemm(a, (B, H, W, Cf), wt, 4, Ktot, (W, H, B), conv_taps(pad64(Cf) // 64), out, 4, bias=b32)
    assert_exact_conv(out, guard, f"vae decoder conv_out {B}x{H}x{W} 128 -> 3 (+1 padded)", [(a, w4, {})], lambda r0, r1: b4)
    assert bool((out[..., 3] == 0).all()), "vae decoder conv_out: the padded column must be exactly 0"


@pytest.mark.parametrize("B,h,w", [(B, h, w) for h, w in EXTENTS for B in (1, 2)])
def test_vae_encoder_conv_out(ctx, B, h, w):
    """build_vae_enc_plan head: conv3(econv_out) 512 -> enc_z_channels = 8 at the latent extent, N = 8, f32 + bias."""
    g = gen(B, h, w, 16)
    a = gx(g, B, h, w, VAE_C)
    out, guard, wc, b16 = conv_form(g, a, 8)
    assert_exact_conv(out, guard, f"vae encoder conv_out {B}x{h}x{w} 512 -> 8", [(a, wc, {})], bias_rows(b16))


# ------------------------------------------------------------------------------------------------------------------------------
# ControlNet hint encoder
# ------------------------------------------------------------------------------------------------------------------------------
def silu_exact_input(g, shape):
    """f32 activations whose silu_f16 is exact: x = 17 + i / 8 (i in [0, 32]), where 1 + __expf(-x) rounds to 1 so silu(x) = x,
    or, a quarter of them, x = -100, where __expf(100) overflows and silu(x) = -0. Returns x and silu(x) in f16."""
    x = torch.randint(0, 33, tuple(shape), generator=g, device=DEV, dtype=torch.int32).float().mul_(0.125).add_(17)
    neg = torch.randint(0, 4, tuple(shape), generator=g, device=DEV) == 0
    x[neg] = -100.0
    return x, torch.where(neg, torch.zeros_like(x), x).half()


# SDXL_CONTROLNET hint_block_channels (16, 32, 96, 256) at the hint's full extent (8x the latent), halving at each stride-2 conv:
# (scale of the latent extent, Cin, Cout, stride)
HINT_CONVS = [(8, 16, 16, 1), (8, 16, 32, 2), (4, 32, 32, 1), (4, 32, 96, 2), (2, 96, 96, 1), (2, 96, 256, 2), (1, 256, 320, 1)]


@pytest.mark.parametrize("n,H,W,Cin,Cout,stride", [(n, h * s, w * s, ci, co, st) for h, w in EXTENTS for s, ci, co, st in HINT_CONVS
                                                   for n in (1, 2)])
def test_hint_encoder_conv(ctx, n, H, W, Cin, Cout, stride):
    """embed_hint -> conv3x3_direct on silu_f16's output: stride 1 (conv_taps) on the plain NHWC image, stride 2 (stride2_taps,
    batch offsets phase * n) on the phase split silu_f16(phase = 1) writes; f32 out + bias, ldo = Cout. Cin = 16 / 32: TMA
    zero-fills 48 / 32 of the 64 channels of each K block."""
    g = gen(n, H, W, Cin, Cout, stride, 17)
    x, s = silu_exact_input(g, (n, H, W, Cin))
    w = gw(g, Cout, Cin, 3, 3)
    b16, b32 = bias_f32(g, Cout)
    Ktot = 9 * pad64(Cin)
    wt = repack3(w, Ktot)
    Ho, Wo = H // stride, W // stride
    a = torch.full((n * H * W * Cin,), float("nan"), dtype=torch.float16, device=DEV)
    T.silu_f16(x, n, H, W, Cin, stride == 2, a)
    if stride == 2:
        a = a.view(2, 2, n, Ho, Wo, Cin)
        assert torch.equal(a, s.view(n, Ho, 2, Wo, 2, Cin).permute(2, 4, 0, 1, 3, 5)), "silu_f16 phase split of exact inputs"
        a, a_shape, segs = a.view(4 * n, Ho, Wo, Cin), (4 * n, Ho, Wo, Cin), stride2_taps(n, pad64(Cin) // 64)
    else:
        a = a.view(n, H, W, Cin)
        assert torch.equal(a, s), "silu_f16 of exact inputs"
        a_shape, segs = (n, H, W, Cin), conv_taps(pad64(Cin) // 64)
    out, guard = guarded((n, Ho, Wo, Cout))
    assert_exact_range("hint conv", conv_bound(s, w), b16.abs().max())
    T.igemm(a, a_shape, wt, Cout, Ktot, (Wo, Ho, n), segs, out, Cout, bias=b32)
    assert_exact_conv(out, guard, f"hint encoder conv {n}x{H}x{W} {Cin}->{Cout} stride {stride}", [(s, w, {"stride": stride})],
                      bias_rows(b16))


# ------------------------------------------------------------------------------------------------------------------------------
# T2I-Adapter
# ------------------------------------------------------------------------------------------------------------------------------
# SDXL_T2I_ADAPTER (in_channels 3, widths 320 / 640 / 1280 / 1280) at latent h x w: features at h / 2 (levels 0, 1) and h / 4
# (levels 2, 3). (form, scale divisor of the latent extent, Cin, Cout, ks, residual in place)
T2I_CONVS = [("conv_in", 2, 768, 320, 3, False), ("in_conv1", 2, 320, 640, 1, False), ("in_conv2", 4, 640, 1280, 1, False),
             ("block1", 2, 320, 320, 3, False), ("block1", 2, 640, 640, 3, False), ("block1", 4, 1280, 1280, 3, False),
             ("block2", 2, 320, 320, 1, True), ("block2", 2, 640, 640, 1, True), ("block2", 4, 1280, 1280, 1, True)]


@pytest.mark.parametrize("n,H,W,form,Cin,Cout,ks,in_place", [(n, h // d, w // d, f, ci, co, ks, ip) for h, w in EXTENTS
                                                             for f, d, ci, co, ks, ip in T2I_CONVS for n in (1, 2)])
def test_t2i_adapter_conv(ctx, n, H, W, form, Cin, Cout, ks, in_place):
    """t2i_forward -> conv_nhwc: conv_taps(ks) (one 1x1 segment for the in_convs and block2), f32 out + bias, ldo = Cout. conv_in
    reads pixel_unshuffle's f16 image of the hint [n, 3, 16 H, 16 W] (checked against F.pixel_unshuffle); block2 adds the
    residual in place (out == res == F[k])."""
    g = gen(n, H, W, Cin, Cout, ks, 18)
    if form == "conv_in":
        hint = gx(g, n, 3, 16 * H, 16 * W).float()
        a = torch.full((n, H, W, Cin), float("nan"), dtype=torch.float16, device=DEV)
        T.pixel_unshuffle(hint, n, 3, 16 * H, 16 * W, a)
        assert torch.equal(a, F.pixel_unshuffle(hint, 16).permute(0, 2, 3, 1).half()), "pixel_unshuffle of the hint"
    else:
        a = gx(g, n, H, W, Cin)
    res = gf(g, n, H, W, Cout) if in_place else None
    out, guard, w, b16 = conv_form(g, a, Cout, ks, res=res)
    assert_exact_conv(out, guard, f"t2i {form} {n}x{H}x{W} {Cin}->{Cout} {ks}x{ks}" + (" residual in place" if in_place else ""),
                      [(a, w, {})], bias_rows(b16, res))


# ------------------------------------------------------------------------------------------------------------------------------
# text and vision encoders, IP-Adapter Plus Resampler
# ------------------------------------------------------------------------------------------------------------------------------
# (M, C, mlp): CLIP-L and OpenCLIP bigG text towers at M = 77 B, B = 1..3; ViT-H and ViT-bigG vision towers at M = 257 N, N = 1, 2
ENC_BLOCKS = ([(77 * B, C, mlp) for C, mlp in ((768, 3072), (1280, 5120)) for B in (1, 2, 3)]
              + [(257 * N, C, mlp) for C, mlp in ((1280, 5120), (1664, 8192)) for N in (1, 2)])


@pytest.mark.parametrize("M,C,mlp", ENC_BLOCKS)
def test_encoder_block_linears(ctx, M, C, mlp):
    """clip_block_ops (text and vision towers): the fused QKV (three transpose_linear slices at rows 0, C, 2C of one [3C, Cpad]
    matrix, three bias_to_f32 slices; f16 out, ldo = 3C), attn out (K = C) and fc2 (K = mlp) adding into the f32 stream in place
    and, at the captured block, into the other buffer (in_place_residual runs both), and fc1 (f32 out + bias, ldo = mlp)."""
    g = gen(M, C, mlp, 19)
    x = gx(g, M, C)
    wqkv = torch.empty(3 * C * pad64(C), dtype=torch.float16, device=DEV)
    bqkv = torch.empty(3 * C, dtype=torch.float32, device=DEV)
    ws, bs = [], []
    for j in range(3):
        ws.append(lin_weights(g, C, C, wt=wqkv, row0=j * C)[0])
        bs.append(grid(g, (C,), GRID_B, 2047))
        T.bias_to_f32(bs[j], C, bqkv[j * C:])
    w, b16 = torch.cat(ws, dim=1), torch.cat(bs)
    out, guard = guarded((M, 3 * C), torch.float16)
    assert_exact_range("qkv", conv_bound(x, w.t()), b16.abs().max())
    linear(x, wqkv, 3 * C, pad64(C), out, 3 * C, bias=bqkv)
    assert_exact(out, x.double() @ w.double() + b16.double(), guard, f"encoder qkv M={M} C={C} (f16 + bias)")
    for name, K in (("attn out", C), ("fc2", mlp)):
        a = gx(g, M, K)
        w, wt = lin_weights(g, K, C)
        b16, b32 = bias_f32(g, C)
        in_place_residual(g, a, w, wt, b16, b32, f"encoder {name} M={M} C={C} K={K}")
    w, wt = lin_weights(g, C, mlp)
    b16, b32 = bias_f32(g, mlp)
    out, guard = guarded((M, mlp))
    assert_exact_range("fc1", conv_bound(x, w.t()), b16.abs().max())
    linear(x, wt, mlp, pad64(C), out, mlp, bias=b32)
    assert_exact(out, x.double() @ w.double() + b16.double(), guard, f"encoder fc1 M={M} C={C} N={mlp}")


@pytest.mark.parametrize("N", [1, 2])
@pytest.mark.parametrize("C", [1280, 1664])
def test_vision_patch_gemm(ctx, N, C):
    """vision_run: patchify's rows (N 256 patches of 14 x 14 x 3 pixels, K = 588 real columns zero-padded to Kpad = 640) times
    the patch conv weight rows copied into a zero-padded [C, 640] matrix; f32 out, no bias, ldo = C. Against the stride-14 conv
    of the pixels: the patch order and the column order (c, kh, kw) must match the conv's."""
    g = gen(N, C, 20)
    S, p, Kp = 224, 14, 640
    K, rows = 3 * p * p, N * (S // p) ** 2
    px = gx(g, N, 3, S, S).float()
    a = torch.full((rows, Kp), float("nan"), dtype=torch.float16, device=DEV)
    T.patchify(px, N, S, p, Kp, a)
    w = gw(g, C, 3, p, p)
    wt = torch.zeros(C, Kp, dtype=torch.float16, device=DEV)
    wt[:, :K] = w.view(C, K)
    out, guard = guarded((rows, C))
    assert_exact_range("patch", conv_bound(px, w))
    T.igemm(a, (1, 1, rows, Kp), wt, C, Kp, (rows, 1, 1), [(0, 0, 0, 0, Kp // 64)], out, C)
    ref = F.conv2d(px.double(), w.double(), stride=p).permute(0, 2, 3, 1).reshape(rows, C)
    assert_exact(out, ref, guard, f"vision patch GEMM N={N} C={C} K={K} (Kpad {Kp})")


@pytest.mark.parametrize("n", [1, 2])
def test_resampler_linears(ctx, n):
    """ip_resample for h94's SDXL Plus adapters (20 heads: W = 1280, D = 1280 ViT-H features of L = 257 tokens, Q = 16 latents,
    context 2048): proj_in (M = 257 n, f32 + bias), to_q (M = 16 n, f16), to_kv (M = 273 n over [LN1(x); LN2(latents)], f16, N = 2W),
    to_out and fc2 (K = 4W) adding into the f32 latent stream in place, fc1 (f32, N = 4W) and proj_out (f32 + bias, N = 2048)."""
    W, D, Q, L, ctx_dim = 1280, 1280, 16, 257, 2048
    g = gen(n, 21)
    for name, M, K, N, bias, f16_out, in_place in (
            ("proj_in", L * n, D, W, True, False, False), ("to_q", Q * n, W, W, False, True, False),
            ("to_kv", (L + Q) * n, W, 2 * W, False, True, False), ("to_out", Q * n, W, W, False, False, True),
            ("fc1", Q * n, W, 4 * W, False, False, False), ("fc2", Q * n, 4 * W, W, False, False, True),
            ("proj_out", Q * n, W, ctx_dim, True, False, False)):
        a = gx(g, M, K)
        w, wt = lin_weights(g, K, N)
        b16, b32 = bias_f32(g, N) if bias else (None, None)
        what = f"resampler {name} M={M} K={K} N={N}"
        if in_place:
            res = gf(g, M, N)
            assert_exact_range(what, conv_bound(a, w.t()), res.abs().max())
            out, guard = guarded((M, N), fill=res)
            linear(a, wt, N, pad64(K), out, N, res=out)
            assert_exact(out, a.double() @ w.double() + res.double(), guard, f"{what} (f32, residual in place)")
            continue
        out, guard = guarded((M, N), torch.float16 if f16_out else torch.float32)
        assert_exact_range(what, conv_bound(a, w.t()), 0 if b16 is None else b16.abs().max())
        linear(a, wt, N, pad64(K), out, N, bias=b32)
        assert_exact(out, a.double() @ w.double() + (0 if b16 is None else b16.double()), guard, what)
