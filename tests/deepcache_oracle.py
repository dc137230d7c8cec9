"""f32 oracle of DeepCache (sdxl_unet_set_deepcache, DESIGN.md §17), built from oracle/unet_oracle.py's pieces and a literal
restatement of the header's semantics: for branch b and e = 3 * n_levels - 1 - b, a full forward is unet_forward and keeps the
backbone input of output block e (before FreeU); a cached forward runs the embeddings, the first conv, input blocks 1..b (T2I
features there), the ControlNets in full with only their residuals 0..b taken, then output blocks e.. on the kept feature and the
head. The chains take `interval`: evaluation j of a call is full when j % interval == 0."""
import dataclasses
import math

import torch

from oracle import unet_oracle as O


def n_branches(cfg) -> int:
    return 3 * len(cfg.channel_mults)


def unet_forward(cfg, w, x, timesteps, context, label, att=None, branch=0, feature=None):
    """(eps, feature). feature None: the full forward, which returns the feature it keeps; else the cached forward on it."""
    att = att or O.NOTHING
    n = x.shape[0]
    latent = x
    if att.concat is not None:
        x = torch.cat([x, O._rows(att.concat, n)], dim=1)
    emb = O._emb(cfg, w, timesteps, label)
    ins, mid, outs = O.unet_blocks(cfg)
    e = len(outs) - 1 - branch
    adds = {}
    if att.t2i is not None and int(timesteps[0]) >= att.t2i[1]:
        adds = {p: O._rows(f, n) for p, f in zip(O.injection_blocks(cfg) + ["middle_block"], att.t2i[0])}
    if feature is None:
        x, saved = O.encoder(cfg, w, x, emb, context, att, adds)
    else:
        saved = []
        for kind, p, nh, d in ins[:branch + 1]:
            x = O._run_block(kind, p, nh, d, x, emb, context, w, att)
            if p in adds:
                x = x + adds[p]
            saved.append(x)
    for ncfg, wc, hint, scale in att.controls:
        res, r_mid = O.controlnet_forward(ncfg, wc, latent, timesteps, context, label, O.hint_embedding(ncfg, wc, hint))
        saved = [s + scale * r for s, r in zip(saved, res)]
        if feature is None:
            x = x + scale * r_mid
    kept = None
    for i, (kind, p, nh, d) in enumerate(outs):
        if feature is not None and i < e:
            continue
        if i == e:
            if feature is None:
                kept = x
            else:
                x = feature
        skip = saved.pop()
        if O.freeu_enabled(att.freeu) and i // 3 < 2:
            x, skip = O.apply_freeu(i // 3, x, skip, att.freeu)
        x = torch.cat([x, skip], dim=1)
        x = O._run_block(kind, p, nh, d, x, emb, context, w, att)
    x = O.group_norm(x, w["norm_out/weight"], w["norm_out/bias"])
    return O.conv2d(O.silu(x), w, "conv_out"), kept


class Cache:
    """One sampling call's DeepCache state: the evaluation count and the kept feature of each row group."""

    def __init__(self, cfg, interval: int, branch: int):
        self.cfg, self.interval, self.branch = cfg, interval, branch
        self.j = 0
        self.features = {}

    def forward(self, group, w, x, timesteps, context, label, att):
        full = self.j % self.interval == 0
        eps, kept = unet_forward(self.cfg, w, x, timesteps, context, label, att, self.branch, None if full else self.features[group])
        if full:
            self.features[group] = kept
        return eps

    def step(self):
        self.j += 1


def forward_diffuser(cfg, w, latent, timestep, c, guidance, att, cache: Cache):
    """oracle/unet_oracle.py's forward_diffuser with each row group's UNet run through the cache."""
    n_batch = latent.shape[0]
    att = att or O.NOTHING
    if not cfg.is_refiner:
        uctx, ctx, uy, y = c.unconditional_context_full, c.context_full, c.unconditional_channel_context, c.channel_context
    else:
        uctx, ctx, uy, y = (c.unconditional_context_open_clip, c.context_open_clip,
                            c.unconditional_channel_context_refiner, c.channel_context_refiner)
    cond = dataclasses.replace(att, prompts=[(wa, O._rows(t, n_batch), s, m) for wa, t, s, m in att.prompts], pag_layers=())
    conditional = cache.forward("cond", w, latent, timestep, ctx, y, cond)
    if att.pag_layers:
        perturbed = cache.forward("ptb", w, latent, timestep, ctx, y, dataclasses.replace(cond, pag_layers=att.pag_layers))
        p_t = att.pag_scale(int(timestep[0]))
    if cfg.is_refiner:
        out = conditional + p_t * (conditional - perturbed) if att.pag_layers else conditional
    else:
        unc = dataclasses.replace(cond, prompts=[(wa, O._rows(t, n_batch), s, m)
                                                 for (wa, _, s, m), t in zip(att.prompts, att.uncond_tokens, strict=True)])
        unconditional = cache.forward("uncond", w, latent, timestep, uctx.unsqueeze(0).repeat(n_batch, 1, 1),
                                      uy.unsqueeze(0).repeat(n_batch, 1), unc)
        out = unconditional + (conditional - unconditional) * guidance
        if att.pag_layers:
            out = out + p_t * (conditional - perturbed)
    cache.step()
    return out


def diffuse_latent(cfg, w, alphas, latent, c, step_start, n_steps, guidance, interval, branch, att=None):
    """oracle/unet_oracle.py's diffuse_latent (DDIM, no inpainting blend) with DeepCache."""
    cache = Cache(cfg, interval, branch)
    step_size = cfg.n_steps // n_steps
    for t in range(cfg.n_steps - step_start - 1, -1, -step_size):
        a = O.get_alpha(alphas, t)
        ap = O.get_alpha(alphas, t - step_size) if t >= step_size else 1.0
        eps = forward_diffuser(cfg, w, latent, torch.tensor([t], dtype=torch.int32), c, guidance, att, cache)
        latent = (latent - eps * math.sqrt(1.0 - a)) / math.sqrt(a) * math.sqrt(ap) + eps * math.sqrt(1.0 - ap)
    return latent


def sample_latent(cfg, w, alphas, noise, c, guidance, n_steps, interval, branch, att=None):
    return diffuse_latent(cfg, w, alphas, noise, c, 0, n_steps, guidance, interval, branch, att)


def refine_latent(cfg, w, alphas, latent, c, guidance, step_start, n_steps, noise, interval, branch, att=None):
    a0 = O.get_alpha(alphas, cfg.n_steps - step_start)
    noised = latent * math.sqrt(a0) + noise * math.sqrt(1.0 - a0)
    return diffuse_latent(cfg, w, alphas, noised, c, step_start, n_steps, guidance, interval, branch, att)


def eps_fn(cfg, w, c, guidance, interval, branch, att=None, no_cfg=False):
    """A scheduled chain's eps(x, t) (tests/scheduler_oracle.py: sample) with DeepCache over the chain's evaluations."""
    cache = Cache(cfg, interval, branch)

    def f(x_in, t):
        ts = torch.tensor([float(t)], dtype=torch.float32)
        if no_cfg:
            eps = cache.forward("cond", w, x_in.float(), ts, c.context_full, c.channel_context, att)
            cache.step()
            return eps
        return forward_diffuser(cfg, w, x_in.float(), ts, c, guidance, att, cache)
    return f
