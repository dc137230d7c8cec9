"""Adapter merges of tests/test_lora_formats_gpu.py's fill check, every output saved to the file given on the command line: a tiny
UNet forward with a LoHa + LoKr + full-delta set and with a DoRA (row and column) set merged, each on a fresh model, so the merge
scratch, the LoKr factors and the DoRA norms all sit in fresh memory. The library reads its switches once per process, so the test
runs this once per configuration.

    python lora_formats_worker.py OUT.pt"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, os.path.join(ROOT, "stable-diffusion-xl-burn_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from sdxl_b200 import TINY, Context, Diffuser, synth_weights  # noqa: E402
from harness import arb, h16f  # noqa: E402
from lora_cases import layer_paths  # noqa: E402
from lora_family_cases import add_dora, make_family  # noqa: E402


def main(out_path):
    ctx = Context(0)
    w = synth_weights(TINY, seed=0)
    paths = layer_paths(TINY)
    exact = [p for p in paths if "/upsample/" not in p]
    x, c, y = arb(2, 4, 16, 16), h16f(arb(2, 7, TINY.context_dim)), h16f(arb(2, TINY.adm_in_channels))
    sets = {
        "families": [(make_family(TINY, paths, "loha", seed=1, dyadic=False), 0.7), (make_family(TINY, paths, "lokr", seed=2, dyadic=False), 0.6),
                     (make_family(TINY, paths[::3], "full", seed=3, dyadic=False), 1.0)],
        "dora": [(add_dora(TINY, make_family(TINY, exact[::2], "loha", seed=4, dyadic=False), w, 0, seed=5), 0.8),
                 (add_dora(TINY, make_family(TINY, exact[1::2], "lora", seed=6, dyadic=False), w, 1, seed=7), 1.0),
                 (make_family(TINY, paths, "lora", seed=8, dyadic=False), 0.5)],
    }
    out = {}
    for name, s in sets.items():
        d = Diffuser(ctx, TINY, w)
        d.set_adapters(s)
        out[name] = d.unet_forward(x, [499], c, y).cpu()
        d.close()
    torch.save(out, out_path)
    ctx.close()


if __name__ == "__main__":
    main(sys.argv[1])
