"""DeepCache workloads of tests/test_deepcache_gpu.py's fill / graph / PDL check, every output saved to the file given on the command
line: an interval-3 DDIM sample and an interval-3 DPM++ 2M Karras sample of the tiny UNet with FreeU and a ControlNet attached,
each on a fresh model so that its plan and sampler buffers are fresh. The library reads its switches once per process, so the test
runs this once per configuration.

    python deepcache_invariance_worker.py OUT.pt"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, os.path.join(ROOT, "stable-diffusion-xl-burn_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from sdxl_b200 import TINY, TINY_CONTROLNET, Conditioning, Context, ControlNet, Diffuser, synth_weights  # noqa: E402
from sdxl_b200.schedulers import Schedule  # noqa: E402
import freeu_oracle as FO  # noqa: E402
from harness import tiny_conditioning  # noqa: E402


def main(out_path):
    ctx = Context(0)
    w = synth_weights(TINY, seed=0)
    net = ControlNet(ctx, TINY_CONTROLNET, synth_weights(TINY_CONTROLNET, seed=1))
    hint = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(2))
    noise = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(0))
    out = {}
    for name, sch in (("ddim", None), ("dpmpp_2m", Schedule("dpmpp_2m", "karras", 7))):
        d = Diffuser(ctx, TINY, w)
        d.set_controls([(net, hint, 0.8)])
        d.set_freeu(*FO.RECOMMENDED_SDXL)
        d.set_deepcache(3, 4)
        out[name] = d.sample_latent(Conditioning(**tiny_conditioning()), 7.5, 7, noise=noise, seed=9, schedule=sch).cpu()
        d.close()
    net.close()
    torch.save(out, out_path)
    ctx.close()


if __name__ == "__main__":
    main(sys.argv[1])
