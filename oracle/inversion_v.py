"""ORACLE (test infrastructure) — the v-prediction form of the reference's DDIM inversion and reconstruction loops.

The reference has no v-prediction support (its preprocess.py would treat the model output as eps).  This restatement
keeps the structure, grids and dtype flow of oracle/inversion.py (0-dim fp32 CPU alphas, `step_alphas`), and replaces
the update by the v-branch of diffusers' DDIMInverseScheduler.step (inversion) and DDIMScheduler.step
(reconstruction), eta = 0: from the level (mu_from, sigma_from) of the sample x to the level (mu_to, sigma_to),

    pred_x0 = mu_from * x - sigma_from * v      pred_eps = mu_from * v + sigma_from * x
    x'      = mu_to * pred_x0 + sigma_to * pred_eps

with the sample of an inversion step at the level of `prev`, as in the reference's eps loop (preprocess.py:211-225).
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch

from .inversion import _eps, step_alphas


def v_expression(x: torch.Tensor, v: torch.Tensor, direction: str, alphas) -> torch.Tensor:
    """One step's v update, with the alphas of `step_alphas`."""
    mu, sigma, mu_prev, sigma_prev = alphas
    if direction == "inversion":
        return mu * (mu_prev * x - sigma_prev * v) + sigma * (mu_prev * v + sigma_prev * x)
    return mu_prev * (mu * x - sigma * v) + sigma_prev * (mu * v + sigma * x)


@torch.no_grad()
def ddim_inversion_v(unet, scheduler, cond: torch.Tensor, latent_frames: torch.Tensor, batch_size: int,
                     timesteps_to_save=None, n_steps: Optional[int] = None) -> Tuple[torch.Tensor, Dict[int, torch.Tensor]]:
    """oracle/inversion.py's `ddim_inversion` for a v-prediction UNet: `latent_frames` updated in place; returns the
    latents and the saved {t: latents} (every t in `timesteps_to_save`, default all, and the last t)."""
    timesteps = reversed(scheduler.timesteps.cpu())
    timesteps_to_save = timesteps_to_save if timesteps_to_save is not None else timesteps
    saved = {}
    for i, t in enumerate(timesteps[:n_steps]):
        alphas = step_alphas(scheduler, "inversion", i)
        for b in range(0, latent_frames.shape[0], batch_size):
            x_batch = latent_frames[b:b + batch_size]
            v = _eps(unet, x_batch, t, cond)
            latent_frames[b:b + batch_size] = v_expression(x_batch, v, "inversion", alphas)
        if t in timesteps_to_save:
            saved[int(t)] = latent_frames.clone()
    saved[int(t)] = latent_frames.clone()
    return latent_frames, saved


@torch.no_grad()
def ddim_sample_v(unet, scheduler, x: torch.Tensor, cond: torch.Tensor, batch_size: int,
                  n_steps: Optional[int] = None) -> torch.Tensor:
    """oracle/inversion.py's `ddim_sample` for a v-prediction UNet (`x` updated in place)."""
    timesteps = scheduler.timesteps.cpu()
    for i, t in enumerate(timesteps[:n_steps]):
        alphas = step_alphas(scheduler, "reconstruction", i)
        for b in range(0, x.shape[0], batch_size):
            x_batch = x[b:b + batch_size]
            v = _eps(unet, x_batch, t, cond)
            x[b:b + batch_size] = v_expression(x_batch, v, "reconstruction", alphas)
    return x
