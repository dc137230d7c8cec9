"""Float64 statement of DESIGN.md §21 (instruction-based editing, diffusers' StableDiffusionXLInstructPix2PixPipeline), importing
nothing from the engine: the three-group image-guidance combine in diffusers' order of terms, guidance rescale of that combine
(tests/prediction_oracle.py's rescale_noise_cfg), and the model rows [cond | img | uncond] as oracle/unet_oracle.py's forward with the
source latent L concatenated to the latent (Attach(concat=L)), zeros for the unconditional group. The chains are
tests/prediction_oracle.py's DDIM loop and samplers and tests/scheduler2_oracle.py's sample2, driven by `model_fn`."""
import torch

from oracle import unet_oracle as O
import prediction_oracle as PR


def combine(c, i, u, s, s_img):
    """g = u + s (c - i) + s_img (i - u), evaluated as (u + s (c - i)) + s_img (i - u)."""
    return (u + s * (c - i)) + s_img * (i - u)


def guided(cfg, w, latent, timestep, c, L, s, s_img, phi=0.0, no_cfg=False, cache=None):
    """The guided model output of one evaluation: rows [cond | img | uncond] with context / pooled [c | n | n] and first-conv condition
    [L | L | 0] (row b reads L[b % n]), combined and, for phi > 0, rescaled against the conditional rows. no_cfg: the conditional rows
    alone. cache (tests/deepcache_oracle.py's Cache): each row group's forward goes through it, as the engine's DeepCache runs them."""
    n = latent.shape[0]
    ctx, y = c.context_full, c.channel_context
    uctx, uy = c.unconditional_context_full.unsqueeze(0).repeat(n, 1, 1), c.unconditional_channel_context.unsqueeze(0).repeat(n, 1)
    with_l, zero = O.Attach(concat=L), O.Attach(concat=torch.zeros_like(L))

    def fwd(group, context, label, att):
        if cache is None:
            return O.unet_forward(cfg, w, latent, timestep, context, label, att)
        return cache.forward(group, w, latent, timestep, context, label, att)
    cond = fwd("cond", ctx, y, with_l)
    if no_cfg:
        out = cond
    else:
        img = fwd("img", uctx, uy, with_l)
        unc = fwd("uncond", uctx, uy, zero)
        out = combine(cond.double(), img.double(), unc.double(), s, s_img)
        if phi > 0:
            out = PR.rescale_noise_cfg(out, cond.double(), phi)
    if cache is not None:
        cache.step()
    return out


def model_fn(cfg, w, c, L, s, s_img, phi=0.0, no_cfg=False, cache=None):
    """g(x_in, t) of `guided` with the timestep as the engine passes it (an int for the DDIM loop, a float for the schedules)."""
    def f(x_in, t):
        ts = torch.tensor([float(t)], dtype=torch.float32)
        return guided(cfg, w, x_in.float(), ts, c, L, s, s_img, phi, no_cfg, cache)
    return f
