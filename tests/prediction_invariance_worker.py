"""v-prediction workloads of tests/test_prediction_gpu.py's fill / graph / PDL check, every output saved to the file given on the
command line: a DDIM and a DPM++ 2M trailing sample of the tiny UNet as a v model on the zero-terminal-SNR table with guidance rescale
0.7 and PAG, each on a fresh model so that its plan and sampler buffers (the statistics kernel's scratch among them) are fresh. The
library reads its switches once per process, so the test runs this once per configuration.

    python prediction_invariance_worker.py OUT.pt"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, os.path.join(ROOT, "stable-diffusion-xl-burn_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from sdxl_b200 import TINY, Conditioning, Context, Diffuser, synth_weights  # noqa: E402
from sdxl_b200.schedulers import Schedule  # noqa: E402
from harness import tiny_conditioning  # noqa: E402


def main(out_path):
    ctx = Context(0)
    w = synth_weights(TINY, seed=0)
    noise = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(0))
    out = {}
    for name, sch in (("ddim", None), ("dpmpp_2m", Schedule("dpmpp_2m", "trailing", 7))):
        d = Diffuser(ctx, TINY, w)
        d.set_pag("mid", 3.0)
        d.set_prediction("v_prediction", 0.7, zero_terminal_snr=True)
        out[name] = d.sample_latent(Conditioning(**tiny_conditioning()), 7.5, 7, noise=noise, seed=9, schedule=sch).cpu()
        d.close()
    torch.save(out, out_path)
    ctx.close()


if __name__ == "__main__":
    main(sys.argv[1])
