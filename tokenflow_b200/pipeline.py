"""The reference's two driver stages on this package's native paths: `preprocess` (preprocess.py:264-330, `prep` /
`extract_latents`) and `edit` (run_tokenflow_pnp.py:251-273, run_tokenflow_sdedit.py:195-216, `edit_video`).

Both take the loaded models (`Parts`, `load_parts`) and uint8 frames, and hold only the drivers' control flow; every
step is a stage function of this package, the chain INTEGRATION.md §6 writes out:

    preprocess: resize_frames -> encode_imgs [-> canny_cond] -> LatentInverter.ddim_inversion / ddim_sample ->
                decode_latents
    edit:       resize_frames -> encode_imgs [-> canny_cond] -> ddim_eps -> add_noise -> TokenFlowEditor.sample_loop ->
                decode_latents

With a CUDA fp16 UNet the inversion runs its captured step (`tf_ddim` / `tf_ddim_v`) and the edit its fused, captured
step (`tf_ext_attn*`, `tf_nn_field`, `tf_propagate`, `tf_cfg_ddim` / `tf_cfg_ddim_v`); with `load_parts` the models are
channels_last fp16, so their GroupNorm sites run `tf_group_norm_nhwc`.  `python -m tokenflow_b200.run` is the
command line around them.
"""
from __future__ import annotations

import copy
import os
from dataclasses import dataclass
from pathlib import Path
from typing import Any, Dict, Optional, Sequence, Tuple

import torch

from . import checkpoint
from . import lora
from . import tokenflow_utils
from .editor import TokenFlowEditor
from .preprocess import (LatentInverter, canny_cond, ddim_eps, decode_latents, encode_imgs, resize_frames,
                         write_inversion_prompt)


@dataclass
class Parts:
    """The models of one checkpoint.  `scheduler` is copied by each stage, which sets its own grid."""
    unet: Any
    vae: Any
    scheduler: Any
    tokenizer: Any
    text_encoder: Any
    controlnet: Any = None

    @property
    def device(self) -> torch.device:
        return next(self.unet.parameters()).device


def load_parts(model_dir: str, device="cuda", dtype=torch.float16, controlnet_dir: Optional[str] = None,
               variant: Optional[str] = None, weights: Optional[str] = None,
               loras: Optional[Sequence[Tuple[str, float]]] = None) -> Parts:
    """Every model of a diffusers checkpoint directory (and a ControlNet folder), as `checkpoint` loads them.

    With `weights`, a single-file SD checkpoint in the LDM layout, the UNet, VAE and text encoder take its weights,
    on the architectures, tokenizer and scheduler of `model_dir` (`checkpoint.load_single_file_models`).  A
    `controlnet_dir` that is a file is a cldm ControlNet (`checkpoint.load_controlnet_file`).  `variant` names the
    weight files of the folders that are read for weights.  `loras`, `[(LoRA file, scale), ...]`, are merged into the
    loaded UNet and text encoder (`lora.merge`), whichever way their weights were read."""
    if weights is None:
        tokenizer, text_encoder = checkpoint.load_text_encoder(model_dir, device, dtype)
        unet = checkpoint.load_unet(model_dir, device, dtype, variant)
        vae = checkpoint.load_vae(model_dir, device, dtype, variant)
    else:
        unet, vae, tokenizer, text_encoder = checkpoint.load_single_file_models(weights, model_dir, device, dtype)
    controlnet = None
    if controlnet_dir and os.path.isfile(controlnet_dir):
        controlnet = checkpoint.load_controlnet_file(controlnet_dir, model_dir, device, dtype)
    elif controlnet_dir:
        controlnet = checkpoint.load_controlnet(controlnet_dir, device, dtype, variant)
    if loras:
        lora.merge(unet, text_encoder, loras)
    return Parts(unet=unet, vae=vae, scheduler=checkpoint.load_scheduler(model_dir), tokenizer=tokenizer,
                 text_encoder=text_encoder, controlnet=controlnet)


def _opt(opt, key: str, default=None):
    return opt.get(key, default) if isinstance(opt, dict) else getattr(opt, key, default)


def latents_dir(opt, n_frames: int) -> str:
    """The reference's latents directory of a preprocess run (preprocess.py:305-309):
    <save_dir>/sd_<sd_version>/<data_path stem>/steps_<steps>/nframes_<n_frames>."""
    return os.path.join(_opt(opt, "save_dir"), f"sd_{_opt(opt, 'sd_version')}", Path(_opt(opt, "data_path")).stem,
                        f"steps_{_opt(opt, 'steps')}", f"nframes_{n_frames}")


@torch.no_grad()
def preprocess(parts: Parts, frames_u8: torch.Tensor, opt, world_size: int = 1, rank: int = 0, group=None,
               comm=None) -> Tuple[Dict[int, torch.Tensor], torch.Tensor]:
    """uint8 frames [N, H_in, W_in, 3] -> ({t: inverted latents [N, 4, h, w]}, reconstruction uint8 [N, H, W, 3]).

    `opt` (an argparse namespace or a dict) has the reference's preprocess flags: H, W, steps, batch_size, save_steps,
    inversion_prompt, and, to write the reference's latents directory (`latents_dir`: latents/noisy_latents_<t>.pt and
    inversion_prompt.txt), save_dir, sd_version and data_path; without save_dir nothing is written.  Square frames are
    resized to 512², others to (H, W), as the reference does.  The latents of the `save_steps` sampling timesteps and of
    the last inversion step are kept, as `get_timesteps(..., strength=1.0)` selects them (preprocess.py:17-24,
    :297-301)."""
    device = parts.device
    frames = frames_u8.to(device)
    square = frames.shape[1] == frames.shape[2]
    frames = resize_frames(frames, 512 if square else (int(_opt(opt, "H")), int(_opt(opt, "W"))))
    latents = encode_imgs(parts.vae, frames)
    edges = canny_cond(frames) if parts.controlnet is not None else None
    sampling = copy.deepcopy(parts.scheduler)
    sampling.set_timesteps(int(_opt(opt, "save_steps")))
    save_path = None
    if _opt(opt, "save_dir") is not None:
        save_path = latents_dir(opt, frames.shape[0])
        if rank == 0:
            write_inversion_prompt(save_path, _opt(opt, "inversion_prompt"))
    inv = LatentInverter(parts.unet, copy.deepcopy(parts.scheduler), int(_opt(opt, "steps")), world_size, rank, group,
                         controlnet=parts.controlnet, controlnet_cond=edges)
    if comm is not None:
        inv.attach_communicator(comm)
    prompt = _opt(opt, "inversion_prompt")
    cond = checkpoint.text_embeds(parts.tokenizer, parts.text_encoder, prompt, "")[1:]
    batch_size = int(_opt(opt, "batch_size"))
    inverted = inv.ddim_inversion(cond, latents, save_path, batch_size=batch_size,
                                  timesteps_to_save=[int(t) for t in sampling.timesteps])
    reconstruction = inv.ddim_sample(inverted, cond, batch_size=batch_size)
    return inv.saved_latents(), decode_latents(parts.vae, reconstruction)


def edit_mode(config: Dict) -> str:
    """The editing method of a config: its `mode`, else "pnp" when it has pnp_attn_t, else "sdedit"."""
    return config.get("mode", "pnp" if "pnp_attn_t" in config else "sdedit")


@torch.no_grad()
def edit(parts: Parts, frames_u8: torch.Tensor, config: Dict, source_latents: Dict[int, torch.Tensor],
         world_size: int = 1, rank: int = 0, group=None, comm=None, vae_recon: bool = False):
    """uint8 frames [N, H_in, W_in, 3] and the inverted latents of their preprocess ({t: [>= N, 4, h, w]}) -> the
    edited uint8 frames [N, 8h, 8w, 3]; with `vae_recon`, (edited frames, the VAE reconstruction of the source
    frames [N, 8h, 8w, 3]), which is `decode_latents` of the latents the edit starts from (the reference's
    `save_vae_recon`, run_tokenflow_pnp.py:242-246).

    `config` has the keys of the reference's configs/config_pnp.yaml or config_sdedit.yaml (prompt, negative_prompt,
    guidance_scale, n_timesteps, batch_size, pnp_attn_t, pnp_f_t / start, use_ddim_noise), `inversion_prompt` (the
    reference reads it from the latents directory), `mode` ("pnp" when pnp_attn_t is given, else "sdedit", unless
    set), and this package's keys (frames_per_pass, controlnet_conditioning_scale, ...).  The editor runs the fused
    step, captured into CUDA graphs on a CUDA UNet, unless the config says otherwise.  The frames are resized to the
    latents' size times 8 (square ones come out of preprocess at 512²).  SDEdit with `use_ddim_noise: False` draws
    one noise latent from the global generator and repeats it over the frames (run_tokenflow_sdedit.py:198); the
    keyframes come from the global CPU generator too, as in the reference, so seed before calling.

    With several ranks every rank resizes, encodes (and runs Canny on) all N frames, since the editor holds the
    latents of all frames, and decodes all N edited frames; only the denoising work is split.  The same holds for
    `preprocess`'s encode and reconstruction decode.  These stages take about 3 % of a single-GPU C2 run."""
    device = parts.device
    n = frames_u8.shape[0]
    # on the device once: the graphed step reads the timestep's source latents every step, and a host tensor would
    # cost a synchronising copy per step
    source = {int(t): v[:n].to(device) for t, v in source_latents.items()}
    h, w = next(iter(source.values())).shape[-2:]
    frames = resize_frames(frames_u8.to(device), (8 * h, 8 * w))
    latents = encode_imgs(parts.vae, frames)
    edges = canny_cond(frames) if parts.controlnet is not None else None
    cfg = dict(config)
    cfg["mode"] = edit_mode(cfg)
    cfg.setdefault("fused_pass", True)
    cfg.setdefault("cuda_graph", device.type == "cuda")
    tok, enc = parts.tokenizer, parts.text_encoder
    text = checkpoint.text_embeds(tok, enc, cfg["prompt"], cfg["negative_prompt"])
    inv_prompt = cfg["inversion_prompt"]
    pnp = checkpoint.text_embeds(tok, enc, inv_prompt, inv_prompt).chunk(2)[0]
    editor = TokenFlowEditor(parts.unet, copy.deepcopy(parts.scheduler), tokenflow_utils, cfg, text, pnp,
                             source_latents=source.__getitem__, world_size=world_size, rank=rank, group=group,
                             controlnet=parts.controlnet, controlnet_cond=edges)
    if comm is not None:
        editor.attach_communicator(comm)
    eps = ddim_eps(latents, source, editor.scheduler)
    if cfg["mode"] == "sdedit" and not cfg.get("use_ddim_noise", True):
        eps = torch.randn_like(eps[[0]]).repeat(n, 1, 1, 1)
    x = editor.scheduler.add_noise(latents, eps, editor.scheduler.timesteps[0])
    editor.init_method()
    edited = decode_latents(parts.vae, editor.sample_loop(x))
    return (edited, decode_latents(parts.vae, latents)) if vae_recon else edited
