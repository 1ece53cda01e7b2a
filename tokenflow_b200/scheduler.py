"""Minimal DDIM scheduler with the surface the reference drivers use
(run_tokenflow_pnp.py:55-56, 190, 217, 257): `set_timesteps`, `timesteps`, `alphas_cumprod`,
`add_noise`, `step(...)['prev_sample']`.

Stable-Diffusion settings: 1000 train steps, scaled-linear betas 0.00085→0.012, "leading"
timestep spacing with steps_offset=1 (50 steps → 981, 961, …, 1), eta=0, no sample clipping,
set_alpha_to_one=False (final alpha = alphas_cumprod[0]).

The model may predict the noise ("epsilon", SD 1.x and the 512² SD 2.x checkpoints) or the velocity
v = sqrt(a) * eps - sqrt(1 - a) * x0 ("v_prediction", the 768² SD 2.x checkpoints); `from_config` reads which from a
diffusers `scheduler_config.json` and refuses any setting this scheduler does not compute.
"""
from __future__ import annotations

import torch

PREDICTION_TYPES = ("epsilon", "v_prediction")

# diffusers DDIMScheduler config keys that change the arithmetic.  A key missing from a config takes diffusers' default
# (the second column), as `DDIMScheduler.from_pretrained` would.  The first group is read; the second must hold the one
# value this scheduler computes.  Every other key (_class_name, _diffusers_version, skip_prk_steps, ...) changes nothing.
_READ_KEYS = {"num_train_timesteps": 1000, "beta_start": 0.0001, "beta_end": 0.02, "steps_offset": 0,
              "prediction_type": "epsilon"}
_FIXED_KEYS = {  # key: (diffusers' default, the value computed here)
    "beta_schedule": ("linear", "scaled_linear"), "set_alpha_to_one": (True, False), "clip_sample": (True, False),
    "thresholding": (False, False), "timestep_spacing": ("leading", "leading"),
    "rescale_betas_zero_snr": (False, False), "trained_betas": (None, None),
}


class DDIMScheduler:
    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085,
                 beta_end: float = 0.012, steps_offset: int = 1, prediction_type: str = "epsilon"):
        if prediction_type not in PREDICTION_TYPES:
            raise ValueError(f"prediction_type={prediction_type!r} is not supported (one of {PREDICTION_TYPES})")
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.final_alpha_cumprod = self.alphas_cumprod[0]
        self.num_train_timesteps = num_train_timesteps
        self.steps_offset = steps_offset
        self.prediction_type = prediction_type
        self.num_inference_steps = None
        self.timesteps = torch.arange(num_train_timesteps - 1, -1, -1)

    @classmethod
    def from_config(cls, config: dict) -> "DDIMScheduler":
        """The scheduler a diffusers `scheduler_config.json` describes (its dict, e.g. `json.load(f)`).  Raises
        ValueError, naming the key and the value, on any setting whose arithmetic this scheduler does not compute:
        a beta schedule other than scaled_linear, set_alpha_to_one, sample clipping, thresholding, timestep spacing
        other than leading, zero-SNR rescaling, trained betas, or a prediction type other than epsilon and
        v_prediction.  Keys that change nothing are ignored; a missing key takes diffusers' default."""
        for key, (default, supported) in _FIXED_KEYS.items():
            value = config.get(key, default)
            if value != supported:
                raise ValueError(f"scheduler config {key}={value!r} is not supported (only {supported!r})")
        c = {key: config.get(key, default) for key, default in _READ_KEYS.items()}
        if c["prediction_type"] not in PREDICTION_TYPES:
            raise ValueError(f"scheduler config prediction_type={c['prediction_type']!r} is not supported "
                             f"(one of {PREDICTION_TYPES})")
        return cls(num_train_timesteps=int(c["num_train_timesteps"]), beta_start=float(c["beta_start"]),
                   beta_end=float(c["beta_end"]), steps_offset=int(c["steps_offset"]),
                   prediction_type=c["prediction_type"])

    def set_timesteps(self, num_inference_steps: int, device=None):
        self.num_inference_steps = num_inference_steps
        ratio = self.num_train_timesteps // num_inference_steps
        ts = (torch.arange(0, num_inference_steps) * ratio).flip(0) + self.steps_offset
        self.timesteps = ts.to(device) if device is not None else ts

    def _alpha(self, t: int) -> torch.Tensor:
        return self.alphas_cumprod[t] if t >= 0 else self.final_alpha_cumprod

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor):
        """eta = 0 DDIM update (diffusers' DDIMScheduler.step, both branches in its operation order).  The alphas enter
        as host scalars (the table lives on the CPU), so the update enqueues device work only — no host<->device copy
        and no stream synchronisation."""
        t = int(timestep)
        prev_t = t - self.num_train_timesteps // self.num_inference_steps
        a_t = float(self._alpha(t))
        a_prev = float(self._alpha(prev_t))
        if self.prediction_type == "v_prediction":
            pred_x0 = a_t ** 0.5 * sample - (1 - a_t) ** 0.5 * model_output
            pred_eps = a_t ** 0.5 * model_output + (1 - a_t) ** 0.5 * sample
        else:
            pred_x0 = (sample - (1 - a_t) ** 0.5 * model_output) / a_t ** 0.5
            pred_eps = model_output
        prev = a_prev ** 0.5 * pred_x0 + (1 - a_prev) ** 0.5 * pred_eps
        return {"prev_sample": prev}

    def add_noise(self, original: torch.Tensor, noise: torch.Tensor, timestep):
        """diffusers' arithmetic (the edit's start, reference run_tokenflow_pnp.py:257): the alpha is taken in the
        samples' dtype, and its square roots are tensor ops in that dtype.  The same for both prediction types: the
        noise comes from the latents (`preprocess.ddim_eps`), not from the model."""
        alphas = self.alphas_cumprod.to(device=original.device, dtype=original.dtype)
        t = torch.as_tensor(timestep).to(original.device)
        a = alphas[t].flatten().view((-1,) + (1,) * (original.dim() - 1))
        return a ** 0.5 * original + (1 - a) ** 0.5 * noise
