"""The flash-attention kernel per element against a float64 statement of its rounding, at every attention shape the plans build
and at adversarial scores; attention_small at the encoders' shapes.

attention_kernel (attention.cu) streams 128-key blocks. For key block j a query row takes the running max m_j (the maximum of
its scores over blocks 0..j, the ragged last block included), computes p = ex2.approx(fmaf(s, sl2e, -f32(m_j sl2e))) in f32,
rounds p to f16 for the P V tensor-core product, adds the unrounded p to l, and rescales O and l by alpha = ex2.approx((m_{j-1}
- m_j) sl2e) when the max grows. out = f16(O / l).

Operands. q and k are f16 multiples of 2^-3 (|entry| <= 2, or wider for the large-logit inputs). Every partial sum of q . k is
then a multiple of 2^-6 below 2^18, exact in f32, so the scores the tensor cores produce equal the float64 scores in any
summation order and the score error drops out. v is on the same grid (or holds one outlier channel near 3e4).

attn_emul states that arithmetic in float64: p = 2^((s - m_j) sl2e) with sl2e the f32 value the kernel reads, P16 = p rounded
to f16 (round to nearest, subnormals included), w_j = 2^((m_j - m_last) sl2e), O = sum_j w_j P16_j V_j, l = sum_j w_j sum(p_j)
(unrounded p), x = O / l. With image sources (kIp) x = O_txt / l_txt + sum_k w_k O_k / l_k, w_k = f32(scale_k mask_k[t]).

Bound. out must lie within half an f16 ulp (of |x| + e) of x, plus e, where e, with u = 2^-24, is the sum of:
  - ambiguous roundings. The kernel's f32 p is within delta_p p of the exact p, where delta_p = E_EX2 + ln2 u (|m_j sl2e| +
    |arg|): E_EX2 = 2^-21 bounds ex2.approx's relative error (as attn_ref does), f32(m_j sl2e) is one rounding of |m_j sl2e|,
    and the fmaf rounds its exact product-minus-difference once, |arg| = |s - m_j| sl2e (a change D in the argument moves p by
    2^D - 1 = ln2 D + O(D^2) relative; D <= 2^-15 here, so the square is below 2^-30 and inside the 2^-21 ex2 allowance). Where
    f16(p (1 - delta_p)) != f16(p (1 + delta_p)) the kernel's P16 may be either; the difference of the two, times |v| and
    w_j, over l, is added. Everywhere else the kernel's P16 equals the emulation's bit for bit. This term grows with |m|: the
    large-logit inputs exercise that.
  - l. f32 sum of unrounded p: a thread adds its 32 columns of a block as 16 pair sums into a chain (at most 17 roundings), l =
    l alpha + sum per block (2 roundings), then two shuffles: every p passes at most 2 nblk + 20 roundings, (2 nblk + 20) u
    relative for a sum of non-negative terms. The kernel's p differ from the exact ones by delta_p each: sum delta_p w p / l.
    x moves by |x| times l's relative error.
  - P V in f32: every addition of the accumulation chain (the S products of P16 V, and one alpha rescale per block) counted
    as one f32 ulp, (S + nblk) 2^-23 sum_j w_j P16_j |V_j| / l. This is the worst case; the tensor cores' internal order is not
    assumed.
  - alpha. O and l are multiplied by the same f32 alpha, so a rescale error common to all blocks cancels in O / l. What does
    not cancel is the difference between blocks: block j's weight carries the errors eps_j of the rescales after it, eps_j =
    sum_{i > j, m_i > m_{i-1}} (E_EX2 + ln2 u |(m_{i-1} - m_i) sl2e|) (the difference m_{i-1} - m_i of two grid scores is exact,
    its product with sl2e rounds once), and x moves by sum_j eps_j w_j |O_j - x l_j| / (l (1 - eps_0)), O_j and l_j block j's
    own sums.
  - final scaling: the reciprocal of l and the multiply by it, 2 u |x|.
  - image sources: each source's own e (times |w_k|), and the f32 fmaf chain that combines them, n_src u (|x_txt| + sum_k |w_k
    x_k|) (the f32 product scale * mask is the w_k the emulation uses).
These are first-order terms; the second-order ones are below 2^-40 relative.

Controls. At S in {77, 129, 257, 1024} the kernel's output falls outside the bound of each of these references: (a) P
truncated toward zero, (b) P unrounded, (c) P rounded against the row's final max instead of its block's running max (S > 128:
with one key block the two maxima are the same), (d) image 0's K / V used for image 1, (e) the ragged last key block dropped
(S = 129 and 257, the sizes that have one). (a) to (c) use the coherent input (coherent_gap): a rising max, and every other
key of a block at the one score gap whose p rounds up to f16 by the most, so P's rounding shifts x in one direction instead
of averaging out, and truncation lands a whole f16 ulp of p below round-to-nearest. At S = 4096 the P V term alone is as wide as P's whole f16 rounding (4096 2^-23 = 2^-11): there (a)
is still rejected and (b), (c) are not (test_controls_at_4096).

Shapes: every self- and cross-attention of block_program(SDXL_BASE) and block_program(SDXL_REFINER) at the 1024^2 latent and the
1216x832 bucket, in the layouts PlanBuilder::strans / attn / attn_ip give them (fused QKV [B T, 3C] with windows 0, C, 2C and
output pitch C; q [B T, C] against the hoisted KV [B n_ctx, 2C] with windows 0 and C), B in {1, 2, 3} and 8 rows, PAG's
attention over the first Bf - Bp rows of a Bf-row buffer, and image sources through attention and attention_multi with masks
from ip_mask_resize. Outputs are NaN-filled and followed by a NaN guard.

attention_small (clip_kernels.cu) keeps P in f32 (32-key chunks with a running max of the same kind), so attn_ref(p_f16=False)
is its bound: the CLIP-L and OpenCLIP-G text encoders, the ViT-H and bigG vision towers and the IP-Adapter Plus Resampler.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from sdxl_b200 import SDXL_BASE, SDXL_REFINER
from sdxl_b200 import _testing as T
from sdxl_b200.config import block_program
from sdxl_b200.ip_adapter import SDXL_PLUS
from harness import DEV, U23, U24, attn_ref, check, f16_round_bound, grid, guarded, heads, to_rows

pytestmark = pytest.mark.gpu

SL2E = float(torch.tensor(1.4426950408889634 / 8.0, dtype=torch.float32))   # the f32 scale_log2e the kernel reads
E_EX2 = 2.0 ** -21
LN2 = math.log(2.0)
EMUL_ELEMS = 2 ** 23          # scores per emulation chunk (a few hundred MB of float64 temporaries)
STEP = 2.0 ** -3              # the q / k / v grid


def cdiv(a, b):
    return (a + b - 1) // b


# ------------------------------------------------------------------------------------------------------------------------------
# the float64 statement of attention_kernel's arithmetic, and its bound
# ------------------------------------------------------------------------------------------------------------------------------
def f16_rn(p: torch.Tensor) -> torch.Tensor:
    return p.half().double()


def f16_rz(p: torch.Tensor) -> torch.Tensor:
    """p >= 0 rounded to f16 toward zero."""
    h = p.half()
    down = (h.view(torch.int16) - 1).view(torch.float16)
    return torch.where(h.double() > p, down, h).double()


def half_ulp16(a: torch.Tensor) -> torch.Tensor:
    """Half an f16 ulp at magnitude a (2^-25 below the normal range)."""
    return torch.exp2(torch.floor(torch.log2(a.clamp_min(2.0 ** -14))) - 11)


def attn_emul(q, k, v, p_round="rn", running_max=True, drop_ragged=False):
    """q [G, T, d], k / v [G, S, d] float64 holding grid f16 values -> (x, e) [G, T, d]: the module docstring's emulation and
    its bound before the output rounding. p_round: "rn" (the kernel), "rz" (truncated P) or "none" (unrounded P);
    running_max=False rounds P against the row's final max; drop_ragged drops the last key block when it is partial."""
    if drop_ragged:
        k, v = k[:, :k.shape[1] // 128 * 128], v[:, :v.shape[1] // 128 * 128]
    G, Tq, d = q.shape
    S = k.shape[1]
    nb = cdiv(S, 128)
    pad = nb * 128 - S
    kp, vp = F.pad(k, (0, 0, 0, pad)), F.pad(v, (0, 0, 0, pad))
    va = vp.abs()
    rnd = {"rn": f16_rn, "rz": f16_rz, "none": None}[p_round]
    x = torch.empty(G, Tq, d, dtype=torch.float64, device=q.device)
    e = torch.empty_like(x)
    tq = max(1, EMUL_ELEMS // (G * nb * 128))
    for t0 in range(0, Tq, tq):
        n = min(tq, Tq - t0)
        s = q[:, t0:t0 + n] @ kp.transpose(1, 2)
        if pad:
            s[..., S:] = float("-inf")
        s = s.view(G, n, nb, 128)
        bm = s.amax(-1)                                        # block maxima
        m = bm.cummax(-1).values if running_max else bm.amax(-1, keepdim=True).expand_as(bm).contiguous()
        live = s.isfinite()
        arg = (s - m[..., None]) * SL2E
        del s
        p = torch.exp2(arg)
        dp = (arg.abs_() + (m * SL2E).abs()[..., None]).mul_(LN2 * U24).add_(E_EX2).masked_fill_(~live, 0.0)
        del arg, live
        w = torch.exp2((m - m[..., -1:]) * SL2E)               # block j's weight against the last block
        lj = p.sum(-1)
        l = (w * lj).sum(-1)                                   # [G, n]
        l_rel = (dp * p).sum(-1).mul_(w).sum(-1) / l + (2 * nb + 20) * U24
        if rnd is None:
            p16, amb = p, None
        else:
            p16 = rnd(p)
            amb = rnd(p * (1 + dp)) - rnd(p * (1 - dp))
        del p, dp
        pw = p16 * w[..., None]
        O = pw.view(G, n, -1) @ vp
        Mabs = pw.view(G, n, -1) @ va
        del pw
        xc = O / l[..., None]
        ec = (S + nb) * U23 * Mabs / l[..., None] + xc.abs() * (l_rel + 2 * U24)[..., None]
        del O, Mabs
        if amb is not None:
            ec += (amb.mul_(w[..., None]).view(G, n, -1) @ va) / l[..., None]
            del amb
        if running_max and nb > 1:
            da = torch.where(m[..., 1:] > m[..., :-1], E_EX2 + LN2 * U24 * ((m[..., 1:] - m[..., :-1]) * SL2E).abs(),
                             torch.zeros_like(m[..., 1:]))
            eps = torch.cat([da.flip(-1).cumsum(-1).flip(-1), torch.zeros_like(m[..., :1])], dim=-1)   # sum over i > j
            Oj = torch.einsum("gtbk,gbkd->gtbd", p16, vp.view(G, nb, 128, d))
            dev = (Oj - xc[:, :, None, :] * lj[..., None]).abs_()
            ec += (dev.mul_((eps * w)[..., None]).sum(-2)) / (l * (1 - eps[..., 0]))[..., None]
            del Oj, dev
        x[:, t0:t0 + n], e[:, t0:t0 + n] = xc, ec
    return x, e


def bound(x, e):
    return half_ulp16(x.abs() + e) + e


def emul_rows(q, k, v, **kw):
    """q [B, nh, T, d], k / v [B, nh, S, d] -> (x, e) as [B T, nh d] rows."""
    B, nh = q.shape[:2]
    x, e = attn_emul(q.flatten(0, 1), k.flatten(0, 1), v.flatten(0, 1), **kw)
    return to_rows(x.view(B, nh, *x.shape[1:])), to_rows(e.view(B, nh, *e.shape[1:]))


def ip_emul(q, kv_txt, srcs, Tq):
    """kIp: x = x_txt + sum_k w_k x_k. kv_txt = (k, v) heads; srcs = [(k, v, scale f32 tensor [1], mask f32 [T] or None)]."""
    x, e = emul_rows(q, *kv_txt)
    mag = x.abs()
    B = q.shape[0]
    for k, v, scale, mask in srcs:
        w = scale.expand(Tq) if mask is None else scale * mask            # f32 product, as the kernel forms it
        w = w.double().repeat(B)[:, None]
        xk, ek = emul_rows(q, k, v)
        x = x + w * xk
        e = e + w.abs() * ek
        mag = mag + (w * xk).abs()
    return x, e + len(srcs) * U24 * mag


def check_emul(out, x, e, what):
    assert bool(torch.isfinite(out).all()), f"{what}: non-finite output"
    return check(out, x, bound(x, e), what)


def outside(out, x, e) -> float:
    """Share of elements of out outside the bound of the reference (x, e)."""
    return float((~((out.double() - x).abs() <= bound(x, e))).double().mean())


# ------------------------------------------------------------------------------------------------------------------------------
# inputs: [B, nh, rows, 64] float64 heads holding f16 grid values
# ------------------------------------------------------------------------------------------------------------------------------
def gridh(g, *shape, lim=16):
    return grid(g, shape, STEP, lim).double()


def coherent_gap() -> float:
    """The raw score gap D (a multiple of 2^-4 in [2, 8]) whose p = 2^(-D sl2e) in (1/4, 3/4) rounds up to f16 by the most:
    on the coherent input every non-max key carries that same rounding error, so P's rounding moves x in one direction (it
    does not average out over the keys). Rounding up puts round-to-nearest close to one f16 ulp of p above truncation and
    half an ulp above the unrounded p; a p that rounds down would make truncation and round-to-nearest the same value."""
    D = torch.arange(32, 129, dtype=torch.float64) / 16
    p = torch.exp2(-D * SL2E)
    r = torch.where((p > 0.25) & (p < 0.75), (f16_rn(p) - p) / p, torch.zeros_like(p))
    return float(D[int(r.argmax())])


def make_qkv(kind, B, nh, Tq, S, g, d=64, chunk=128):
    """q [B, nh, Tq, d], k, v [B, nh, S, d] of one of the score patterns below; chunk is the kernel's key-block size (the
    rising max steps at every chunk)."""
    big = {"grid": 16, "outlier_v": 16, "offset+300": 16, "offset-300": 16}.get(kind, 8)
    q, k, v = gridh(g, B, nh, Tq, d, lim=big), gridh(g, B, nh, S, d, lim=big), gridh(g, B, nh, S, d)
    if kind.startswith("dominant"):              # one key 64 logits (at d = 64) above every other (others within +-8)
        kappa = int(kind[8:]) if kind[8:] != "last" else S - 1
        q[..., 0], k[..., 0] = 32.0, 0.0
        k[..., kappa, 0] = 16.0
    elif kind == "rising":                       # every chunk's max 4 logits (at d = 64) above the previous one's
        q[..., 0] = 2.0
        k[..., 0] = 16.0 * (torch.arange(S, device=DEV) // chunk).double()
    elif kind == "equal":                        # q = 0: x is the mean of V
        q.zero_()
    elif kind.startswith("offset"):              # +-300 on every logit
        q[..., 0] = 40.0
        k[..., 0] = 60.0 if kind[6] == "+" else -60.0
    elif kind == "large_ties":                   # |logits| up to ~1e3; identical keys mirrored around every block boundary
        q = gridh(g, B, nh, Tq, d, lim=128)
        k = gridh(g, B, nh, S, d, lim=32)
        q[..., 0] = torch.where(torch.rand(B, nh, Tq, generator=g, device=DEV) < 0.5, -16.0, 16.0).double()
        k[..., 0] = 0.0
        for b0 in range(chunk, S, chunk):
            for i in range(4):
                if b0 + i < S:
                    k[:, :, b0 - 1 - i, 0] = 500.0
                    k[:, :, b0 + i] = k[:, :, b0 - 1 - i]
    elif kind == "coherent":                     # rising max; every other key of a block exactly D below the block's max
        q.zero_()
        q[..., 0] = 1.0
        k[..., 0] = (torch.arange(S, device=DEV) // chunk).double()
        k[..., ::chunk, 0] += coherent_gap()
        v = 1.5 + gridh(g, B, nh, S, d, lim=3).abs()
    elif kind == "outlier_v":                    # one channel near +3e4 and one near -3e4
        v[..., 5] = 16.0 * torch.randint(1850, 1900, (B, nh, S), generator=g, device=DEV).double()
        v[..., 6] = -16.0 * torch.randint(1850, 1900, (B, nh, S), generator=g, device=DEV).double()
    else:
        assert kind == "grid", kind
    return q, k, v


def rows16(*hs):
    """Heads [B, nh, rows, d] -> one f16 matrix [B rows, sum nh d] with the heads' windows side by side."""
    return torch.cat([to_rows(h) for h in hs], dim=1).half().contiguous()


def run_cross(q, k, v, out_pitch=None):
    """attention on q [B T, C] and the KV matrix [B S, 2C] (windows 0 and C): the plan's cross-attention layout."""
    B, nh, Tq, _ = q.shape
    S, C = k.shape[2], nh * 64
    qm, kvm = rows16(q), rows16(k, v)
    out, guard = guarded((B * Tq, C), torch.float16)
    T.attention(qm, C, 0, kvm, 2 * C, 0, C, B, Tq, S, nh, out, C)
    return out, guard


def assert_guard(guard, what):
    assert bool(guard.isnan().all()), f"{what}: elements after the output were written"


# ------------------------------------------------------------------------------------------------------------------------------
# adversarial scores
# ------------------------------------------------------------------------------------------------------------------------------
ADVERSARIAL = ([("grid", S) for S in (77, 129, 257, 1024, 4096)]
               + [("dominant0", S) for S in (77, 129, 257, 1024, 4096)]
               + [(f"dominant{kk}", S) for kk in (127, 128) for S in (129, 257, 1024, 4096)]
               + [("dominantlast", S) for S in (77, 129, 257, 1024, 4096)]
               + [(r, S) for r in ("rising", "coherent") for S in (129, 257, 1024, 4096)]
               + [("equal", S) for S in (77, 257, 4096)]
               + [(f"offset{o}300", S) for o in "+-" for S in (77, 257, 1024)]
               + [("large_ties", S) for S in (129, 257, 1024, 4096)]
               + [("outlier_v", S) for S in (77, 257, 4096)])


@pytest.mark.parametrize("kind,S", ADVERSARIAL)
def test_adversarial_scores(kind, S):
    """B = 2, 2 heads, T = 129 (a ragged query tile) in the cross-attention layout."""
    g = torch.Generator(device=DEV).manual_seed(sum(map(ord, kind)) * 7 + S)
    q, k, v = make_qkv(kind, 2, 2, 129, S, g)
    s = q @ k.transpose(-1, -2) / 8
    if kind.startswith("dominant"):
        top = s.amax(-1, keepdim=True)
        assert bool(((s == top).sum(-1) == 1).all()) and float((s.masked_fill(s == top, -1e9) - top).amax()) <= -30
    if kind in ("rising", "coherent") and S > 128:
        bm = F.pad(s, (0, cdiv(S, 128) * 128 - S), value=-1e9).unflatten(-1, (-1, 128)).amax(-1)
        assert bool((bm[..., 1:] > bm[..., :-1]).all()), "the rising input's block maxima must grow at every block"
    if kind == "large_ties":
        assert float(s.abs().amax()) > 900
    out, guard = run_cross(q, k, v)
    x, e = emul_rows(q, k, v)
    check_emul(out, x, e, f"flash {kind} S={S}")
    assert_guard(guard, kind)
    if kind == "equal":                   # every p is 1: x is the mean of V (two float64 sums in different orders)
        mean = to_rows(v.mean(dim=2, keepdim=True).expand(-1, -1, 129, -1))
        assert float((x - mean).abs().max()) <= 2.0 ** -40, "equal logits: the emulation must give the mean of V"
    if kind.startswith("dominant"):       # every other p underflows f16: x is the dominant key's v
        kappa = int(kind[8:]) if kind[8:] != "last" else S - 1
        vk = v[:, :, kappa:kappa + 1].expand(-1, -1, 129, -1)
        assert torch.equal(out, rows16(vk)), f"dominant key {kappa}: the output must be its v"


# ------------------------------------------------------------------------------------------------------------------------------
# controls: references the kernel's output must fall outside of
# ------------------------------------------------------------------------------------------------------------------------------
def control_refs(q, k, v, S):
    """(input, (x, e)) of each control reference; q, k, v map the input kind to its heads."""
    qc, kc, vc = q["coherent"], k["coherent"], v["coherent"]
    qg, kg, vg = q["grid"], k["grid"], v["grid"]
    refs = {"(a) P truncated": ("coherent", emul_rows(qc, kc, vc, p_round="rz")),
            "(b) P unrounded": ("coherent", emul_rows(qc, kc, vc, p_round="none")),
            "(d) image 0 K/V for image 1": ("grid image 1", emul_rows(qg[1:], kg[:1], vg[:1]))}
    if S > 128:
        refs["(c) final max"] = ("coherent", emul_rows(qc, kc, vc, running_max=False))
    if S % 128 and S > 128:
        refs["(e) ragged block dropped"] = ("grid", emul_rows(qg, kg, vg, drop_ragged=True))
    return refs


def run_controls(S):
    """Kernel outputs at S for the grid and coherent inputs (B = 2, 4 heads, T = 512), each checked against its own bound,
    and the share of each output outside each control's bound."""
    Tq, B, nh = 512, 2, 4
    q, k, v, outs = {}, {}, {}, {}
    for kind in ("grid", "coherent"):
        g = torch.Generator(device=DEV).manual_seed(S * 3 + len(kind))
        q[kind], k[kind], v[kind] = make_qkv(kind, B, nh, Tq, S, g)
        outs[kind], _ = run_cross(q[kind], k[kind], v[kind])
        x, e = emul_rows(q[kind], k[kind], v[kind])
        check_emul(outs[kind], x, e, f"controls: kernel S={S} {kind}")
    shares = {}
    for name, (inp, ref) in control_refs(q, k, v, S).items():
        out = outs["grid"][Tq:] if inp == "grid image 1" else outs[inp]
        shares[name] = outside(out, *ref)
        print(f"controls S={S} {name}: {100 * shares[name]:.3f} % of elements outside its bound")
    return shares


@pytest.mark.parametrize("S", [77, 129, 257, 1024])
def test_controls_rejected(S):
    shares = run_controls(S)
    for name, share in shares.items():
        assert share > 0, f"S={S}: the bound does not tell the kernel from the reference {name}"


def test_controls_at_4096():
    """At S = 4096 the P V term is as wide as P's rounding: truncated P and the wrong image's K / V are still rejected."""
    shares = run_controls(4096)
    assert shares["(a) P truncated"] > 0 and shares["(d) image 0 K/V for image 1"] > 0


# ------------------------------------------------------------------------------------------------------------------------------
# every plan attention shape
# ------------------------------------------------------------------------------------------------------------------------------
def latent_hws(h, w, n_levels):
    hw = []
    for _ in range(n_levels):
        hw.append(h * w)
        h, w = (h + 1) // 2, (w + 1) // 2
    return hw


def attn_shapes(cfg, hws):
    """(T, n_head) of every transformer block of a UNet of cfg, with hws[level] tokens at each level."""
    ins, mid, outs = block_program(cfg)
    shapes = set()
    level = 0
    for blk in ins[1:]:
        if blk.kind == "downsample":
            level += 1
        elif blk.depth:
            shapes.add((hws[level], blk.n_head))
    if mid.depth:
        shapes.add((hws[-1], mid.n_head))
    level = len(hws) - 1
    for blk in outs:
        if blk.depth:
            shapes.add((hws[level], blk.n_head))
        if blk.kind.endswith("upsample"):
            level -= 1
    return shapes


PLAN_SHAPES = sorted(attn_shapes(SDXL_BASE, latent_hws(128, 128, 3)) | attn_shapes(SDXL_BASE, latent_hws(152, 104, 3))
                     | attn_shapes(SDXL_REFINER, latent_hws(128, 128, 4)) | attn_shapes(SDXL_REFINER, latent_hws(152, 104, 4)))
PLAN_CASES = [(T_, nh, 1 + i % 3) for i, (T_, nh) in enumerate(PLAN_SHAPES)]


def test_plan_shapes_cover_the_levels():
    assert {(4096, 10), (1024, 20), (3952, 10), (988, 20), (4096, 12), (1024, 24), (256, 24), (3952, 12), (988, 24),
            (247, 24)} == set(PLAN_SHAPES)
    assert {B for _, _, B in PLAN_CASES} == {1, 2, 3}


def self_attention(T_, nh, B, g, Bf=None):
    """strans' self-attention over the first B of Bf rows of a fused QKV buffer; checks the attended rows and that the others
    and the guard stay NaN."""
    Bf = Bf or B
    C = nh * 64
    qkv = grid(g, (Bf * T_, 3 * C), STEP, 16)
    out, guard = guarded((Bf * T_, C), torch.float16)
    T.attention(qkv, 3 * C, 0, qkv, 3 * C, C, 2 * C, B, T_, T_, nh, out, C)
    hv = [heads(qkv[:B * T_], B, T_, c0, nh, 64) for c0 in (0, C, 2 * C)]
    x, e = emul_rows(*hv)
    what = f"self-attention B={B}/{Bf} T={T_} heads={nh}"
    check_emul(out[:B * T_], x, e, what)
    assert bool(out[B * T_:].isnan().all()), f"{what}: rows past the attended ones were written"
    assert_guard(guard, what)


@pytest.mark.parametrize("T_,nh,B", PLAN_CASES)
def test_self_attention_plan(T_, nh, B):
    self_attention(T_, nh, B, torch.Generator(device=DEV).manual_seed(T_ * 31 + nh + B))


@pytest.mark.parametrize("T_,nh,B", PLAN_CASES)
@pytest.mark.parametrize("n_ctx", [77, 154])
def test_cross_attention_plan(T_, nh, B, n_ctx):
    g = torch.Generator(device=DEV).manual_seed(T_ * 17 + nh + B + n_ctx)
    q, k, v = make_qkv("grid", B, nh, T_, n_ctx, g)
    out, guard = run_cross(q, k, v)
    x, e = emul_rows(q, k, v)
    check_emul(out, x, e, f"cross-attention B={B} T={T_} n_ctx={n_ctx} heads={nh}")
    assert_guard(guard, "cross-attention")


def test_self_attention_eight_rows():
    """Eight rows (four images under classifier-free guidance) at the base's level 2."""
    self_attention(1024, 20, 8, torch.Generator(device=DEV).manual_seed(8))


@pytest.mark.parametrize("T_,nh,Bf,Bp", [(1024, 20, 3, 1), (4096, 10, 6, 2), (247, 24, 3, 1)])
def test_pag_self_attention(T_, nh, Bf, Bp):
    """PAG: softmax attention over the first Bf - Bp rows; the perturbed rows' output is left to pag_identity."""
    self_attention(T_, nh, Bf - Bp, torch.Generator(device=DEV).manual_seed(T_ + Bf + Bp), Bf=Bf)


@pytest.mark.parametrize("T_,nh,B,S_ip", [(4096, 10, 2, 4), (1024, 20, 3, 16), (988, 24, 1, 16), (247, 24, 2, 4)])
def test_ip_source(T_, nh, B, S_ip):
    """One image source through attention, in attn_ip's layout (KV [B S_ip, 2C], windows 0 and C)."""
    g = torch.Generator(device=DEV).manual_seed(T_ + nh + B + S_ip)
    C = nh * 64
    q, k, v = make_qkv("grid", B, nh, T_, 77, g)
    _, ki, vi = make_qkv("grid", B, nh, 1, S_ip, g)
    scale = torch.tensor([0.7], device=DEV)
    out, guard = guarded((B * T_, C), torch.float16)
    T.attention(rows16(q), C, 0, rows16(k, v), 2 * C, 0, C, B, T_, 77, nh, out, C, kip=rows16(ki, vi), kip_pitch=2 * C,
                k_ip_col0=0, v_ip_col0=C, S_ip=S_ip, ip_scale=scale)
    x, e = ip_emul(q, (k, v), [(ki, vi, scale, None)], T_)
    check_emul(out, x, e, f"IP attention B={B} T={T_} S_ip={S_ip} heads={nh}")
    assert_guard(guard, "IP attention")


def soft_mask(H, W, left):
    """A [H, W] f32 region mask: 1 on one side of a vertical edge, 0 on the other, a linear ramp between."""
    xs = torch.linspace(0.0, 1.0, W, device=DEV)
    ramp = ((xs - 0.4) / 0.2).clamp(0, 1)
    return (1 - ramp if left else ramp).expand(H, W).contiguous()


@pytest.mark.parametrize("h,w,n_levels,level,nh", [(152, 104, 3, 1, 10), (152, 104, 3, 2, 20), (152, 104, 4, 3, 24)])
def test_masked_image_sources(h, w, n_levels, level, nh):
    """Three image sources through attention_multi at the bucket's level extents: two masked by ip_mask_resize'd regions
    (S_ip 16 and 4), one unmasked."""
    g = torch.Generator(device=DEV).manual_seed(h * level + nh)
    mh, mw = h >> level, w >> level
    T_, B, C = mh * mw, 2, nh * 64
    q, k, v = make_qkv("grid", B, nh, T_, 77, g)
    srcs, launch = [], []
    for S_ip, scale, mask in ((16, 0.6, soft_mask(96, 64, True)), (4, 0.9, soft_mask(h, w, False)), (16, 0.45, None)):
        _, ki, vi = make_qkv("grid", B, nh, 1, S_ip, g)
        sc = torch.tensor([scale], device=DEV)
        mk = None if mask is None else T.ip_mask_resize(mask, mh, mw, T_)
        srcs.append((ki, vi, sc, mk))
        launch.append((rows16(ki, vi), 2 * C, 0, C, S_ip, sc, mk))
    out, guard = guarded((B * T_, C), torch.float16)
    T.attention_multi(rows16(q), C, 0, rows16(k, v), 2 * C, 0, C, B, T_, 77, nh, out, C, launch)
    x, e = ip_emul(q, (k, v), srcs, T_)
    check_emul(out, x, e, f"masked image sources {mh}x{mw} heads={nh}")
    assert_guard(guard, "masked image sources")


# ------------------------------------------------------------------------------------------------------------------------------
# attention_small at the encoders' shapes
# ------------------------------------------------------------------------------------------------------------------------------
SMALL = {"clip-l": (64, 12, 77, 77, True), "openclip-g": (64, 20, 77, 77, True), "vit-h": (80, 16, 257, 257, False),
         "vit-bigg": (104, 16, 257, 257, False), "resampler": (64, SDXL_PLUS.heads, SDXL_PLUS.tokens, 257 + SDXL_PLUS.tokens, False)}


@pytest.mark.parametrize("kind", ["grid", "dominantlast", "rising"])
@pytest.mark.parametrize("enc", list(SMALL))
def test_attention_small_encoders(enc, kind):
    """The text encoders (causal, fused QKV pitch 3C), the vision towers (fused QKV, T = S = 257) and the Resampler (Q latents
    against L + Q keys: q pitch W, KV pitch 2W with windows 0 and W), B = 2."""
    d, nh, Tq, S, causal = SMALL[enc]
    g = torch.Generator(device=DEV).manual_seed(d * nh + Tq + len(kind))
    B, C = 2, nh * d
    q, k, v = make_qkv(kind, B, nh, Tq, S, g, d=d, chunk=32)
    out, guard = guarded((B * Tq, C), torch.float16)
    if enc == "resampler":
        kv = rows16(k, v)
        T.attention_small(rows16(q), C, 0, kv, kv, 2 * C, 0, C, B, Tq, S, nh, None, False, out, C, d)
    else:
        qkv = rows16(q, k, v)
        T.attention_small(qkv, 3 * C, 0, qkv, qkv, 3 * C, C, 2 * C, B, Tq, S, nh, None, causal, out, C, d)
    ref, tol = attn_ref(q, k, v, 1.0 / math.sqrt(d), causal=causal, p_f16=False)
    ref, tol = to_rows(ref), to_rows(tol)
    assert bool(torch.isfinite(out).all())
    check(out, ref, tol + f16_round_bound(ref), f"attention_small {enc} {kind}")
    assert_guard(guard, enc)
