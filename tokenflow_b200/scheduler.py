"""Minimal DDIM scheduler with the surface the reference drivers use
(run_tokenflow_pnp.py:55-56, 190, 217, 257): `set_timesteps`, `timesteps`, `alphas_cumprod`,
`add_noise`, `step(...)['prev_sample']`.

Stable-Diffusion settings: 1000 train steps, scaled-linear betas 0.00085→0.012, "leading"
timestep spacing with steps_offset=1 (50 steps → 981, 961, …, 1), eta=0, no sample clipping,
set_alpha_to_one=False (final alpha = alphas_cumprod[0]).
"""
from __future__ import annotations

import torch


class DDIMScheduler:
    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085,
                 beta_end: float = 0.012, steps_offset: int = 1):
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.final_alpha_cumprod = self.alphas_cumprod[0]
        self.num_train_timesteps = num_train_timesteps
        self.steps_offset = steps_offset
        self.num_inference_steps = None
        self.timesteps = torch.arange(num_train_timesteps - 1, -1, -1)

    def set_timesteps(self, num_inference_steps: int, device=None):
        self.num_inference_steps = num_inference_steps
        ratio = self.num_train_timesteps // num_inference_steps
        ts = (torch.arange(0, num_inference_steps) * ratio).flip(0) + self.steps_offset
        self.timesteps = ts.to(device) if device is not None else ts

    def _alpha(self, t: int) -> torch.Tensor:
        return self.alphas_cumprod[t] if t >= 0 else self.final_alpha_cumprod

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor):
        """eta = 0 DDIM update.  The alphas enter as host scalars (the table lives on the CPU), so the
        update enqueues device work only — no host<->device copy and no stream synchronisation."""
        t = int(timestep)
        prev_t = t - self.num_train_timesteps // self.num_inference_steps
        a_t = float(self._alpha(t))
        a_prev = float(self._alpha(prev_t))
        pred_x0 = (sample - (1 - a_t) ** 0.5 * model_output) / a_t ** 0.5
        prev = a_prev ** 0.5 * pred_x0 + (1 - a_prev) ** 0.5 * model_output
        return {"prev_sample": prev}

    def add_noise(self, original: torch.Tensor, noise: torch.Tensor, timestep):
        """diffusers' arithmetic (the edit's start, reference run_tokenflow_pnp.py:257): the alpha is taken in the
        samples' dtype, and its square roots are tensor ops in that dtype."""
        alphas = self.alphas_cumprod.to(device=original.device, dtype=original.dtype)
        t = torch.as_tensor(timestep).to(original.device)
        a = alphas[t].flatten().view((-1,) + (1,) * (original.dim() - 1))
        return a ** 0.5 * original + (1 - a) ** 0.5 * noise
