"""Load Stable Diffusion from a diffusers model folder on disk: the models the pipeline runs, with real weights.

A diffusers checkpoint directory holds one folder per model:

    <model_dir>/unet/config.json + weights          -> load_unet        (sd_unet.UNet2DConditionModel)
    <model_dir>/vae/config.json + weights           -> load_vae         (vae.AutoencoderKL)
    <model_dir>/scheduler/scheduler_config.json     -> load_scheduler   (scheduler.DDIMScheduler)
    <model_dir>/text_encoder/, <model_dir>/tokenizer/ -> load_text_encoder (transformers' CLIPTextModel / CLIPTokenizer)
    <controlnet_dir>/config.json + weights          -> load_controlnet  (controlnet.ControlNetModel, its own folder)

Each model is built from its `config.json` by the class's `from_config` (which refuses, with a ValueError naming the
key, any setting the restatement does not compute) on the `meta` device, so no parameter is initialised, and the
weights are assigned with `strict=True`: every name and shape must match.  The module is then cast to `dtype`, moved to
`device`, and made channels_last when it is CUDA fp16, the layout in which its GroupNorm sites run
`tf_group_norm_nhwc` rather than ATen.

Weights are read from diffusers' file names: `diffusion_pytorch_model.safetensors`, the `fp16` variant
`diffusion_pytorch_model.fp16.safetensors`, a sharded `diffusion_pytorch_model.safetensors.index.json`, and the same
for `.bin` files (read with `torch.load(weights_only=True)`).  Single-file `.ckpt` checkpoints are not read.

The text side is the reference's (preprocess.py:53-55, :151-160): transformers' own CLIP classes, loaded from the local
folders only, and `text_embeds` is its `get_text_embeds`.
"""
from __future__ import annotations

import json
import os
from typing import Callable, Dict, Optional

import torch
import torch.nn as nn

WEIGHTS_NAME = "diffusion_pytorch_model"


def read_config(folder: str, name: str = "config.json") -> dict:
    with open(os.path.join(folder, name)) as f:
        return json.load(f)


def _with_variant(name: str, variant: Optional[str]) -> str:
    """diffusers' variant file name: the variant goes before the last suffix (x.safetensors -> x.fp16.safetensors,
    x.safetensors.index.json -> x.safetensors.index.fp16.json)."""
    if not variant:
        return name
    head, tail = name.rsplit(".", 1)
    return f"{head}.{variant}.{tail}"


def _read_file(path: str) -> Dict[str, torch.Tensor]:
    if path.endswith(".safetensors"):
        from safetensors.torch import load_file
        return load_file(path)
    return torch.load(path, map_location="cpu", weights_only=True)


def load_weights(folder: str, variant: Optional[str] = None) -> Dict[str, torch.Tensor]:
    """The state dict stored in a diffusers model folder, in diffusers' order of preference: one safetensors file, a
    sharded safetensors index, one .bin file, a sharded .bin index.  `variant="fp16"` reads the fp16 files."""
    tried = []
    for suffix in ("safetensors", "bin"):
        single = os.path.join(folder, _with_variant(f"{WEIGHTS_NAME}.{suffix}", variant))
        if os.path.isfile(single):
            return _read_file(single)
        index = os.path.join(folder, _with_variant(f"{WEIGHTS_NAME}.{suffix}.index.json", variant))
        if os.path.isfile(index):
            with open(index) as f:
                shards = sorted(set(json.load(f)["weight_map"].values()))
            state = {}
            for shard in shards:
                state.update(_read_file(os.path.join(folder, shard)))
            return state
        tried += [single, index]
    raise FileNotFoundError(f"no weights in {folder}: tried {', '.join(os.path.basename(p) for p in tried)}")


# diffusers' AttentionBlock before 0.14 (the name every SD 1.x / 2.x VAE on the hub was saved with) -> its `Attention`
_DEPRECATED_ATTENTION = {"query": "to_q", "key": "to_k", "value": "to_v", "proj_attn": "to_out.0"}


def renamed_vae_attention(state: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """The state dict with the VAE mid-block attentions' deprecated names (`query`, `key`, `value`, `proj_attn`) renamed
    to `to_q`, `to_k`, `to_v`, `to_out.0`, as diffusers' `_convert_deprecated_attention_blocks` does when it loads
    such a file.  Other keys are kept as they are."""
    out = {}
    for key, value in state.items():
        head, sep, tail = key.partition(".attentions.0.")
        if sep and "mid_block" in head:
            name, dot, param = tail.partition(".")
            tail = f"{_DEPRECATED_ATTENTION.get(name, name)}{dot}{param}"
        out[head + sep + tail] = value
    return out


def load_model(build: Callable[[dict], nn.Module], folder: str, device="cpu", dtype=torch.float32,
               variant: Optional[str] = None,
               rename: Optional[Callable[[Dict[str, torch.Tensor]], Dict[str, torch.Tensor]]] = None) -> nn.Module:
    """`build(config)` on the meta device, the folder's weights (after `rename`) assigned with strict=True, then cast,
    moved, and made channels_last when CUDA fp16."""
    config = read_config(folder)
    with torch.device("meta"):
        net = build(config)
    state = load_weights(folder, variant)
    net.load_state_dict(rename(state) if rename is not None else state, strict=True, assign=True)
    net = net.to(device=device, dtype=dtype)
    if torch.device(device).type == "cuda" and dtype == torch.float16:
        net = net.to(memory_format=torch.channels_last)
    return net.eval()


def load_unet(model_dir: str, device="cpu", dtype=torch.float32, variant: Optional[str] = None):
    from .sd_unet import UNet2DConditionModel
    return load_model(UNet2DConditionModel.from_config, os.path.join(model_dir, "unet"), device, dtype, variant)


def load_vae(model_dir: str, device="cpu", dtype=torch.float32, variant: Optional[str] = None):
    """The VAE, whether its mid-block attentions carry today's names or the deprecated ones the SD 1.x / 2.x VAE
    files were published with (`renamed_vae_attention`)."""
    from .vae import AutoencoderKL
    return load_model(AutoencoderKL.from_config, os.path.join(model_dir, "vae"), device, dtype, variant,
                      rename=renamed_vae_attention)


def load_controlnet(controlnet_dir: str, device="cpu", dtype=torch.float32, variant: Optional[str] = None):
    """A standalone ControlNet folder (`config.json` and the weights at its top level, as lllyasviel/sd-controlnet-canny
    is published)."""
    from .controlnet import ControlNetModel
    return load_model(ControlNetModel.from_config, controlnet_dir, device, dtype, variant)


def load_scheduler(model_dir: str):
    """`DDIMScheduler.from_config` of the checkpoint's `scheduler/scheduler_config.json`: the parameterisation (eps or
    v) is read from the checkpoint, never assumed."""
    from .scheduler import DDIMScheduler
    return DDIMScheduler.from_config(read_config(os.path.join(model_dir, "scheduler"), "scheduler_config.json"))


def load_text_encoder(model_dir: str, device="cpu", dtype=torch.float32):
    """(tokenizer, text encoder): transformers' CLIPTokenizer and CLIPTextModel from the checkpoint's `tokenizer/` and
    `text_encoder/` folders, local files only, the encoder in `dtype` on `device` (reference preprocess.py:53-55)."""
    from transformers import CLIPTextModel, CLIPTokenizer
    tokenizer = CLIPTokenizer.from_pretrained(model_dir, subfolder="tokenizer", local_files_only=True)
    encoder = CLIPTextModel.from_pretrained(model_dir, subfolder="text_encoder", local_files_only=True, dtype=dtype)
    return tokenizer, encoder.to(device).eval()


@torch.no_grad()
def text_embeds(tokenizer, encoder, prompt: str, negative_prompt: str) -> torch.Tensor:
    """[2, L, C] = [uncond, cond]: the reference's `get_text_embeds` (preprocess.py:151-160, run_tokenflow_pnp.py:
    128-142).  Both prompts are padded to the tokenizer's `model_max_length`; the prompt is truncated to it and the
    negative prompt is not, so a negative prompt longer than the encoder's positions raises the ValueError the
    encoder raises for the reference's call.

    The inversion's condition is `text_embeds(tok, enc, inversion_prompt, "")[1:]` (preprocess.py:271) and the edit's
    PnP guidance `text_embeds(tok, enc, inversion_prompt, inversion_prompt).chunk(2)[0]` (run_tokenflow_pnp.py:68)."""
    device = next(encoder.parameters()).device
    ids = tokenizer(prompt, padding="max_length", max_length=tokenizer.model_max_length, truncation=True,
                    return_tensors="pt").input_ids
    cond = encoder(ids.to(device))[0]
    ids = tokenizer(negative_prompt, padding="max_length", max_length=tokenizer.model_max_length,
                    return_tensors="pt").input_ids
    uncond = encoder(ids.to(device))[0]
    return torch.cat([uncond, cond])
