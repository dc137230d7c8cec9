"""The edit workload of tests/test_edit_gpu.py's fill / graph / PDL check, saved to the file given on the command line: a DPM++ 2M
Karras sample of the tiny edit UNet with image guidance and guidance rescale 0.7, on a fresh model so that its plan, its per-row
first-conv condition and the sampler buffers are fresh. The library reads its switches once per process, so the test runs this once per
configuration.

    python edit_invariance_worker.py OUT.pt"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, os.path.join(ROOT, "stable-diffusion-xl-burn_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from sdxl_b200 import TINY_EDIT, Conditioning, Context, Diffuser, synth_weights  # noqa: E402
from sdxl_b200.schedulers import Schedule  # noqa: E402
from harness import tiny_conditioning  # noqa: E402


def main(out_path):
    ctx = Context(0)
    g = torch.Generator().manual_seed(0)
    noise, L = torch.randn(2, 4, 16, 16, generator=g), torch.randn(1, 4, 16, 16, generator=g)
    d = Diffuser(ctx, TINY_EDIT, synth_weights(TINY_EDIT, seed=0))
    d.set_edit_image(L, 1.5)
    d.set_prediction("epsilon", 0.7)
    out = {"dpmpp_2m": d.sample_latent(Conditioning(**tiny_conditioning(cfg=TINY_EDIT)), 5.0, 6, noise=noise,
                                       schedule=Schedule("dpmpp_2m", "karras", 6)).cpu()}
    d.close()
    torch.save(out, out_path)
    ctx.close()


if __name__ == "__main__":
    main(sys.argv[1])
