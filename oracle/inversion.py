"""ORACLE (test infrastructure) — the reference's DDIM inversion and reconstruction loops, restated with its dtype flow
(omerbt/TokenFlow preprocess.py:199-261, `Preprocess.ddim_inversion` / `Preprocess.ddim_sample`, plain SD UNet: no
depth or ControlNet conditioning).

The dtype flow is the reference's: the latents and the UNet are whatever the caller passes (fp16 on the GPU in the
reference), the timesteps come from `scheduler.timesteps` on the CPU, and the alphas are 0-dim fp32 CPU tensors
(`scheduler.alphas_cumprod[t]`), so `alpha ** 0.5` and `1 - alpha` are fp32 tensor operations and each latent
expression is evaluated as written: ATen multiplies the fp16 latents by the 0-dim fp32 scalars and divides by one
(`/ mu_prev`) as a multiply by its fp32 reciprocal, rounding every intermediate to fp16.

`n_steps` stops the loop after that many steps of the grid (timing and comparisons over part of a schedule); the
reference runs the whole grid.  The reference writes the saved latents to `noisy_latents_<t>.pt`; here they are
returned as {t: clone}.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch


def _eps(unet, x_batch, t, cond):
    cond_batch = cond.repeat(x_batch.shape[0], 1, 1)                                          # :206
    out = unet(x_batch, t, encoder_hidden_states=cond_batch)                                  # :222
    return out["sample"] if isinstance(out, dict) else out.sample


@torch.no_grad()
def ddim_inversion(unet, scheduler, cond: torch.Tensor, latent_frames: torch.Tensor, batch_size: int,
                   timesteps_to_save=None, n_steps: Optional[int] = None) -> Tuple[torch.Tensor, Dict[int, torch.Tensor]]:
    """preprocess.py:199-230 on `latent_frames` (updated in place, as the reference does).  Returns the latents and
    the saved {t: latents}: every t in `timesteps_to_save` (default: all) and the last t."""
    timesteps = reversed(scheduler.timesteps.cpu())                                           # :200
    timesteps_to_save = timesteps_to_save if timesteps_to_save is not None else timesteps     # :201
    saved = {}
    for i, t in enumerate(timesteps[:n_steps]):                                               # :202
        for b in range(0, latent_frames.shape[0], batch_size):                                # :203
            x_batch = latent_frames[b:b + batch_size]
            alpha_prod_t = scheduler.alphas_cumprod[t]                                        # :211
            alpha_prod_t_prev = (scheduler.alphas_cumprod[timesteps[i - 1]]
                                 if i > 0 else scheduler.final_alpha_cumprod)                 # :212-215
            mu = alpha_prod_t ** 0.5                                                          # :217-220
            mu_prev = alpha_prod_t_prev ** 0.5
            sigma = (1 - alpha_prod_t) ** 0.5
            sigma_prev = (1 - alpha_prod_t_prev) ** 0.5
            eps = _eps(unet, x_batch, t, cond)
            pred_x0 = (x_batch - sigma_prev * eps) / mu_prev                                  # :224
            latent_frames[b:b + batch_size] = mu * pred_x0 + sigma * eps                      # :225
        if t in timesteps_to_save:                                                            # :227-228
            saved[int(t)] = latent_frames.clone()
    saved[int(t)] = latent_frames.clone()                                                     # :229
    return latent_frames, saved


@torch.no_grad()
def ddim_sample(unet, scheduler, x: torch.Tensor, cond: torch.Tensor, batch_size: int,
                n_steps: Optional[int] = None) -> torch.Tensor:
    """preprocess.py:232-261 on `x` (updated in place, as the reference does)."""
    timesteps = scheduler.timesteps.cpu()                                                     # :234
    for i, t in enumerate(timesteps[:n_steps]):                                               # :235
        for b in range(0, x.shape[0], batch_size):                                            # :236
            x_batch = x[b:b + batch_size]
            alpha_prod_t = scheduler.alphas_cumprod[t]                                        # :245
            alpha_prod_t_prev = (scheduler.alphas_cumprod[timesteps[i + 1]]
                                 if i < len(timesteps) - 1 else scheduler.final_alpha_cumprod)   # :246-250
            mu = alpha_prod_t ** 0.5                                                          # :251-254
            sigma = (1 - alpha_prod_t) ** 0.5
            mu_prev = alpha_prod_t_prev ** 0.5
            sigma_prev = (1 - alpha_prod_t_prev) ** 0.5
            eps = _eps(unet, x_batch, t, cond)                                                # :256
            pred_x0 = (x_batch - sigma * eps) / mu                                            # :259
            x[b:b + batch_size] = mu_prev * pred_x0 + sigma_prev * eps                        # :260
    return x


def step_alphas(scheduler, direction: str, i: int):
    """(mu, sigma, mu_prev, sigma_prev) of step i of `direction` ("inversion" or "reconstruction") as the reference
    computes them: 0-dim fp32 tensors (:211-220 / :245-254)."""
    if direction == "inversion":
        timesteps = reversed(scheduler.timesteps.cpu())
        a_p = scheduler.alphas_cumprod[timesteps[i - 1]] if i > 0 else scheduler.final_alpha_cumprod
    else:
        timesteps = scheduler.timesteps.cpu()
        a_p = (scheduler.alphas_cumprod[timesteps[i + 1]] if i < len(timesteps) - 1
               else scheduler.final_alpha_cumprod)
    a_t = scheduler.alphas_cumprod[timesteps[i]]
    return a_t ** 0.5, (1 - a_t) ** 0.5, a_p ** 0.5, (1 - a_p) ** 0.5


def step_coefficients(scheduler, direction: str, i: int):
    """The fp32 values (s1, inv_s2, s3, s4) with which the reference's step i evaluates
    `s3 * ((x - s1 * eps) * inv_s2) + s4 * eps`: inv_s2 is the fp32 reciprocal ATen multiplies by when it divides a
    CUDA tensor by a 0-dim CPU tensor."""
    mu, sigma, mu_prev, sigma_prev = step_alphas(scheduler, direction, i)
    if direction == "inversion":
        return sigma_prev, 1 / mu_prev, mu, sigma
    return sigma, 1 / mu, mu_prev, sigma_prev


def ddim_expression(x: torch.Tensor, eps: torch.Tensor, direction: str, alphas) -> torch.Tensor:
    """One step's update as the reference writes it (:224-225 / :259-260), with the alphas of `step_alphas`."""
    mu, sigma, mu_prev, sigma_prev = alphas
    if direction == "inversion":
        return mu * ((x - sigma_prev * eps) / mu_prev) + sigma * eps
    return mu_prev * ((x - sigma * eps) / mu) + sigma_prev * eps
