"""ORACLE (test infrastructure) — the reference's DDIM inversion and reconstruction loops with its ControlNet branch
(omerbt/TokenFlow preprocess.py:199-261 with `sd_version == 'ControlNet'`): every UNet call is `controlnet_pred`
(:129-149) on the batch's slice of the Canny conditioning (:222-223, :256-257).

The dtype flow is that of oracle/inversion.py, which restates the same loops for the plain UNet: timesteps from
`scheduler.timesteps` on the CPU, the alphas 0-dim fp32 CPU tensors, every latent expression evaluated as written.
`n_steps` stops the loop after that many steps of the grid; the saved latents are returned as {t: clone}.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch


def controlnet_pred(controlnet, unet, latent_model_input, t, text_embed_input, controlnet_cond):
    down_block_res_samples, mid_block_res_sample = controlnet(                               # :130-137
        latent_model_input,
        t,
        encoder_hidden_states=text_embed_input,
        controlnet_cond=controlnet_cond,
        conditioning_scale=1,
        return_dict=False,
    )
    return unet(                                                                              # :140-148
        latent_model_input,
        t,
        encoder_hidden_states=text_embed_input,
        cross_attention_kwargs={},
        down_block_additional_residuals=down_block_res_samples,
        mid_block_additional_residual=mid_block_res_sample,
        return_dict=False,
    )[0]


@torch.no_grad()
def ddim_inversion(unet, controlnet, scheduler, cond: torch.Tensor, canny_cond: torch.Tensor,
                   latent_frames: torch.Tensor, batch_size: int, timesteps_to_save=None,
                   n_steps: Optional[int] = None) -> Tuple[torch.Tensor, Dict[int, torch.Tensor]]:
    """preprocess.py:199-230 on `latent_frames` (updated in place), `canny_cond` [N, 3, H, W] the conditioning of the
    N frames.  Returns the latents and the saved {t: latents}: every t in `timesteps_to_save` (default: all) and the
    last t."""
    timesteps = reversed(scheduler.timesteps.cpu())                                           # :200
    timesteps_to_save = timesteps_to_save if timesteps_to_save is not None else timesteps     # :201
    saved = {}
    for i, t in enumerate(timesteps[:n_steps]):                                               # :202
        for b in range(0, latent_frames.shape[0], batch_size):                                # :203
            x_batch = latent_frames[b:b + batch_size]
            cond_batch = cond.repeat(x_batch.shape[0], 1, 1)                                  # :206
            alpha_prod_t = scheduler.alphas_cumprod[t]                                        # :211
            alpha_prod_t_prev = (scheduler.alphas_cumprod[timesteps[i - 1]]
                                 if i > 0 else scheduler.final_alpha_cumprod)                 # :212-215
            mu = alpha_prod_t ** 0.5                                                          # :217-220
            mu_prev = alpha_prod_t_prev ** 0.5
            sigma = (1 - alpha_prod_t) ** 0.5
            sigma_prev = (1 - alpha_prod_t_prev) ** 0.5
            eps = controlnet_pred(controlnet, unet, x_batch, t, cond_batch,
                                  torch.cat([canny_cond[b: b + batch_size]]))                 # :222-223
            pred_x0 = (x_batch - sigma_prev * eps) / mu_prev                                  # :224
            latent_frames[b:b + batch_size] = mu * pred_x0 + sigma * eps                      # :225
        if t in timesteps_to_save:                                                            # :227-228
            saved[int(t)] = latent_frames.clone()
    saved[int(t)] = latent_frames.clone()                                                     # :229
    return latent_frames, saved


@torch.no_grad()
def ddim_sample(unet, controlnet, scheduler, x: torch.Tensor, cond: torch.Tensor, canny_cond: torch.Tensor,
                batch_size: int, n_steps: Optional[int] = None) -> torch.Tensor:
    """preprocess.py:232-261 on `x` (updated in place)."""
    timesteps = scheduler.timesteps.cpu()                                                     # :234
    for i, t in enumerate(timesteps[:n_steps]):                                               # :235
        for b in range(0, x.shape[0], batch_size):                                            # :236
            x_batch = x[b:b + batch_size]
            cond_batch = cond.repeat(x_batch.shape[0], 1, 1)                                  # :239
            alpha_prod_t = scheduler.alphas_cumprod[t]                                        # :245
            alpha_prod_t_prev = (scheduler.alphas_cumprod[timesteps[i + 1]]
                                 if i < len(timesteps) - 1 else scheduler.final_alpha_cumprod)   # :246-250
            mu = alpha_prod_t ** 0.5                                                          # :251-254
            sigma = (1 - alpha_prod_t) ** 0.5
            mu_prev = alpha_prod_t_prev ** 0.5
            sigma_prev = (1 - alpha_prod_t_prev) ** 0.5
            eps = controlnet_pred(controlnet, unet, x_batch, t, cond_batch,
                                  torch.cat([canny_cond[b: b + batch_size]]))                 # :256-257
            pred_x0 = (x_batch - sigma * eps) / mu                                            # :259
            x[b:b + batch_size] = mu_prev * pred_x0 + sigma_prev * eps                        # :260
    return x
