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
for `.bin` files (read with `torch.load(weights_only=True)`).

A single-file checkpoint in the original LDM layout (`.safetensors`, or a `.ckpt` / `.pth` read with
`weights_only=True`) supplies the weights of the same models: `load_single_file_models` renames
`model.diffusion_model.*`, `first_stage_model.*` and `cond_stage_model.*` to diffusers' names (`unet_state`,
`vae_state`, `text_state`), and `load_controlnet_file` renames a cldm ControlNet's `control_model.*`
(`controlnet_state`).  The architectures, the tokenizer and the scheduler still come from a diffusers folder of the
same family, since a single file holds no config, no vocabulary and no prediction type.

The text side is the reference's (preprocess.py:53-55, :151-160): transformers' own CLIP classes, loaded from the local
folders only, and `text_embeds` is its `get_text_embeds`.
"""
from __future__ import annotations

import json
import os
import pickle
import re
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


def assign_model(build: Callable[[dict], nn.Module], config: dict, state: Dict[str, torch.Tensor], device="cpu",
                 dtype=torch.float32) -> nn.Module:
    """`build(config)` on the meta device, `state` assigned with strict=True, then cast, moved, and made channels_last
    when CUDA fp16."""
    with torch.device("meta"):
        net = build(config)
    net.load_state_dict(state, strict=True, assign=True)
    net = net.to(device=device, dtype=dtype)
    if torch.device(device).type == "cuda" and dtype == torch.float16:
        net = net.to(memory_format=torch.channels_last)
    return net.eval()


def load_model(build: Callable[[dict], nn.Module], folder: str, device="cpu", dtype=torch.float32,
               variant: Optional[str] = None,
               rename: Optional[Callable[[Dict[str, torch.Tensor]], Dict[str, torch.Tensor]]] = None) -> nn.Module:
    """`assign_model` of the folder's config.json and its weights (after `rename`)."""
    config = read_config(folder)
    state = load_weights(folder, variant)
    return assign_model(build, config, rename(state) if rename is not None else state, device, dtype)


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


# Single-file checkpoints in the original LDM layout (`v1-5-pruned-emaonly.safetensors`, `v2-1_768-ema-pruned.ckpt`,
# lllyasviel's `control_sd15_canny.pth`): one state dict whose prefixes name the models.
UNET_PREFIX = "model.diffusion_model."
VAE_PREFIX = "first_stage_model."
TEXT_PREFIX = "cond_stage_model."
CONTROLNET_PREFIX = "control_model."


def load_single_file(path: str) -> Dict[str, torch.Tensor]:
    """The tensors of a single-file checkpoint: a `.safetensors` file, or a `.ckpt` / `.pth` pickle read with
    `torch.load(weights_only=True)`, its top-level "state_dict" unwrapped.  A pickle `weights_only` refuses (one that
    holds objects other than tensors and plain containers) raises ValueError: it is never unpickled in full."""
    if path.endswith(".safetensors"):
        from safetensors.torch import load_file
        return load_file(path)
    try:
        obj = torch.load(path, map_location="cpu", weights_only=True)
    except pickle.UnpicklingError as e:
        reason = str(e).strip().splitlines()[0]
        raise ValueError(f"{path} cannot be read with torch.load(weights_only=True) ({reason}); "
                         f"convert it to .safetensors") from e
    if isinstance(obj, dict) and isinstance(obj.get("state_dict"), dict):
        obj = obj["state_dict"]
    return obj


def _section(ckpt: Dict[str, torch.Tensor], prefix: str) -> Dict[str, torch.Tensor]:
    out = {k[len(prefix):]: v for k, v in ckpt.items() if k.startswith(prefix)}
    if not out:
        raise ValueError(f"the checkpoint has no tensors under {prefix!r}")
    return out


def _renamed(key: str, table: Dict[str, str]) -> str:
    """`key` with its first matching module path of `table` replaced; unchanged when none matches."""
    for old, new in table.items():
        if key == old or key.startswith(old + "."):
            return new + key[len(old):]
    return key


_LDM_RESNET = {"in_layers.0": "norm1", "in_layers.2": "conv1", "emb_layers.1": "time_emb_proj",
               "out_layers.0": "norm2", "out_layers.3": "conv2", "skip_connection": "conv_shortcut"}
_LDM_UNET_TOP = {"time_embed.0": "time_embedding.linear_1", "time_embed.2": "time_embedding.linear_2",
                 "out.0": "conv_norm_out", "out.2": "conv_out"}


def _unet_key(key: str, layers: int) -> str:
    """diffusers' name of one key of LDM's UNetModel (its input blocks are also the ControlNet's encoder); a key
    outside LDM's grammar is returned unchanged, so the strict load names it.  `layers` is `layers_per_block`: each
    level has that many input blocks and one more output block, and the input blocks after each level but the last
    hold only the downsampler."""
    m = re.fullmatch(r"input_blocks\.(\d+)\.(\d+)\.(.+)", key)
    if m:
        b, sub, rest = int(m[1]), int(m[2]), m[3]
        if b == 0:
            return f"conv_in.{rest}" if sub == 0 else key
        i, j = divmod(b - 1, layers + 1)
        if j == layers:
            return f"down_blocks.{i}.downsamplers.0.conv.{rest[3:]}" if sub == 0 and rest.startswith("op.") else key
        if sub == 0:
            return f"down_blocks.{i}.resnets.{j}.{_renamed(rest, _LDM_RESNET)}"
        return f"down_blocks.{i}.attentions.{j}.{rest}" if sub == 1 else key
    m = re.fullmatch(r"output_blocks\.(\d+)\.(\d+)\.(.+)", key)
    if m:
        (i, j), sub, rest = divmod(int(m[1]), layers + 1), int(m[2]), m[3]
        if sub == 0:
            return f"up_blocks.{i}.resnets.{j}.{_renamed(rest, _LDM_RESNET)}"
        if rest.startswith("conv."):              # the upsampler: item 1 of a level without attention, else item 2
            return f"up_blocks.{i}.upsamplers.0.{rest}"
        return f"up_blocks.{i}.attentions.{j}.{rest}" if sub == 1 else key
    m = re.fullmatch(r"middle_block\.([012])\.(.+)", key)
    if m:
        sub, rest = int(m[1]), m[2]
        return (f"mid_block.attentions.0.{rest}" if sub == 1 else
                f"mid_block.resnets.{sub // 2}.{_renamed(rest, _LDM_RESNET)}")
    return _renamed(key, _LDM_UNET_TOP)


def unet_state(ckpt: Dict[str, torch.Tensor], layers_per_block: int = 2) -> Dict[str, torch.Tensor]:
    """The UNet of an LDM checkpoint (`model.diffusion_model.*`) under diffusers' names.  The EMA copy
    (`model_ema.*`) is not read: the non-EMA weights are the ones diffusers loads."""
    return {_unet_key(k, layers_per_block): v for k, v in _section(ckpt, UNET_PREFIX).items()}


def controlnet_state(ckpt: Dict[str, torch.Tensor], layers_per_block: int = 2) -> Dict[str, torch.Tensor]:
    """The ControlNet of a cldm checkpoint (`control_model.*`) under diffusers' names: the encoder as in `unet_state`,
    `input_hint_block` (convolutions at the even indices, SiLU between them) as the conditioning embedding's conv_in,
    blocks and conv_out, `zero_convs.i.0` as `controlnet_down_blocks.i` and `middle_block_out.0` as
    `controlnet_mid_block`.  Other prefixes of the file (lllyasviel's `.pth` files also hold a whole SD model) are not
    read."""
    state = _section(ckpt, CONTROLNET_PREFIX)
    hint = [int(m[1]) for k in state if (m := re.match(r"input_hint_block\.(\d+)\.", k))]
    last = max(hint, default=0)
    out = {}
    for key, value in state.items():
        if m := re.fullmatch(r"input_hint_block\.(\d+)\.(.+)", key):
            k, rest = int(m[1]), m[2]
            name = "conv_in" if k == 0 else "conv_out" if k == last else f"blocks.{k // 2 - 1}"
            key = f"controlnet_cond_embedding.{name}.{rest}" if k % 2 == 0 else key
        elif m := re.fullmatch(r"zero_convs\.(\d+)\.0\.(.+)", key):
            key = f"controlnet_down_blocks.{m[1]}.{m[2]}"
        elif key.startswith("middle_block_out.0."):
            key = "controlnet_mid_block." + key[len("middle_block_out.0."):]
        else:
            key = _unet_key(key, layers_per_block)
        out[key] = value
    return out


_LDM_VAE_RESNET = {"nin_shortcut": "conv_shortcut"}
_LDM_VAE_ATTENTION = {"norm": "group_norm", "q": "to_q", "k": "to_k", "v": "to_v", "proj_out": "to_out.0"}


def vae_state(ckpt: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """The VAE of an LDM checkpoint (`first_stage_model.*`) under diffusers' names.  LDM numbers the decoder's levels
    from the highest resolution, diffusers in the order they run, so `decoder.up.k` is `up_blocks.(n-1-k)`; the
    mid-block attention's 1x1 convolution weights [C, C, 1, 1] become linear weights [C, C]."""
    state = _section(ckpt, VAE_PREFIX)
    n = 1 + max((int(m[1]) for k in state if (m := re.match(r"decoder\.up\.(\d+)\.", k))), default=-1)
    out = {}
    for key, value in state.items():
        if m := re.fullmatch(r"encoder\.down\.(\d+)\.block\.(\d+)\.(.+)", key):
            key = f"encoder.down_blocks.{m[1]}.resnets.{m[2]}.{_renamed(m[3], _LDM_VAE_RESNET)}"
        elif m := re.fullmatch(r"encoder\.down\.(\d+)\.downsample\.(.+)", key):
            key = f"encoder.down_blocks.{m[1]}.downsamplers.0.{m[2]}"
        elif m := re.fullmatch(r"decoder\.up\.(\d+)\.block\.(\d+)\.(.+)", key):
            key = f"decoder.up_blocks.{n - 1 - int(m[1])}.resnets.{m[2]}.{_renamed(m[3], _LDM_VAE_RESNET)}"
        elif m := re.fullmatch(r"decoder\.up\.(\d+)\.upsample\.(.+)", key):
            key = f"decoder.up_blocks.{n - 1 - int(m[1])}.upsamplers.0.{m[2]}"
        elif m := re.fullmatch(r"(encoder|decoder)\.mid\.block_([12])\.(.+)", key):
            key = f"{m[1]}.mid_block.resnets.{int(m[2]) - 1}.{_renamed(m[3], _LDM_VAE_RESNET)}"
        elif m := re.fullmatch(r"(encoder|decoder)\.mid\.attn_1\.(norm|q|k|v|proj_out)\.(.+)", key):
            key = f"{m[1]}.mid_block.attentions.0.{_LDM_VAE_ATTENTION[m[2]]}.{m[3]}"
            if m[2] != "norm" and value.dim() == 4:
                value = value.flatten(1)
        elif m := re.fullmatch(r"(encoder|decoder)\.norm_out\.(.+)", key):
            key = f"{m[1]}.conv_norm_out.{m[2]}"
        out[key] = value
    return out


_OPENCLIP_TOP = {"token_embedding": "text_model.embeddings.token_embedding",
                 "positional_embedding": "text_model.embeddings.position_embedding.weight",
                 "ln_final": "text_model.final_layer_norm"}
_OPENCLIP_BLOCK = {"ln_1": "layer_norm1", "ln_2": "layer_norm2", "mlp.c_fc": "mlp.fc1", "mlp.c_proj": "mlp.fc2",
                   "attn.out_proj": "self_attn.out_proj"}


def text_state(ckpt: Dict[str, torch.Tensor], num_hidden_layers: int) -> Dict[str, torch.Tensor]:
    """The text encoder of an LDM checkpoint under the names of transformers' CLIPTextModel.

    SD 1.x (`cond_stage_model.transformer.*`) already has CLIPTextModel's names, with or without the `text_model.`
    level of newer transformers; a stored `position_ids` buffer is dropped.  SD 2.x (`cond_stage_model.model.*`) is
    OpenCLIP's layout: each resblock's packed `attn.in_proj_{weight,bias}` is split in three along dim 0 into q, k
    and v.  SD 2.x reads the penultimate layer, so its text_encoder/config.json has one layer fewer than the file has
    resblocks: the resblocks from `num_hidden_layers` on are dropped, as are `text_projection` and `logit_scale`.  A
    file with fewer resblocks is refused."""
    state = _section(ckpt, TEXT_PREFIX)
    clip = {k[len("transformer."):]: v for k, v in state.items() if k.startswith("transformer.")}
    if clip:
        clip = {(k if k.startswith("text_model.") else "text_model." + k): v for k, v in clip.items()}
        clip.pop("text_model.embeddings.position_ids", None)
        return clip
    openclip = {k[len("model."):]: v for k, v in state.items() if k.startswith("model.")}
    if not openclip:
        raise ValueError(f"the checkpoint has no tensors under {TEXT_PREFIX + 'transformer.'!r} (SD 1.x) or "
                         f"{TEXT_PREFIX + 'model.'!r} (SD 2.x)")
    out, blocks = {}, set()
    for key, value in openclip.items():
        if m := re.fullmatch(r"transformer\.resblocks\.(\d+)\.(.+)", key):
            i, rest = int(m[1]), m[2]
            blocks.add(i)
            if i >= num_hidden_layers:
                continue
            layer = f"text_model.encoder.layers.{i}."
            if m := re.fullmatch(r"attn\.in_proj_(weight|bias)", rest):
                for name, part in zip(("q_proj", "k_proj", "v_proj"), value.chunk(3, dim=0)):
                    out[f"{layer}self_attn.{name}.{m[1]}"] = part
            else:
                out[layer + _renamed(rest, _OPENCLIP_BLOCK)] = value
        elif key not in ("text_projection", "logit_scale"):
            out[_renamed(key, _OPENCLIP_TOP)] = value
    if len(blocks) < num_hidden_layers:
        raise ValueError(f"the checkpoint's text encoder has {len(blocks)} resblocks under "
                         f"{TEXT_PREFIX + 'model.transformer.resblocks'!r}; the base folder's text_encoder/config.json "
                         f"needs num_hidden_layers={num_hidden_layers}")
    return out


def _clip_text_model(config) -> nn.Module:
    """transformers' CLIPTextModel of `config`.  It is built on the meta device, so its `position_ids` buffer, which
    no checkpoint needs to store, is made again on the CPU."""
    from transformers import CLIPTextModel
    encoder = CLIPTextModel(config)
    encoder.text_model.embeddings.register_buffer(
        "position_ids", torch.arange(config.max_position_embeddings, device="cpu").expand((1, -1)), persistent=False)
    return encoder


def load_single_file_models(path: str, model_dir: str, device="cpu", dtype=torch.float32):
    """(unet, vae, tokenizer, text encoder) of a single-file SD checkpoint in the LDM layout.  The file gives only the
    weights; every model is built from `model_dir`, a diffusers folder of the same family (unet/, vae/,
    text_encoder/config.json; the tokenizer, whose vocabulary a single file does not hold, from tokenizer/), and
    assigned with strict=True, so a file of another family is refused naming the key.  The models are cast, moved
    and made channels_last as `load_model` makes them."""
    from transformers import CLIPTextConfig, CLIPTokenizer
    from .sd_unet import UNet2DConditionModel
    from .vae import AutoencoderKL
    ckpt = load_single_file(path)
    unet_config = read_config(os.path.join(model_dir, "unet"))
    unet = assign_model(UNet2DConditionModel.from_config, unet_config,
                        unet_state(ckpt, unet_config.get("layers_per_block", 2)), device, dtype)
    vae = assign_model(AutoencoderKL.from_config, read_config(os.path.join(model_dir, "vae")), vae_state(ckpt),
                       device, dtype)
    text_config = CLIPTextConfig.from_pretrained(model_dir, subfolder="text_encoder", local_files_only=True)
    encoder = assign_model(_clip_text_model, text_config, text_state(ckpt, text_config.num_hidden_layers), device,
                           dtype)
    tokenizer = CLIPTokenizer.from_pretrained(model_dir, subfolder="tokenizer", local_files_only=True)
    return unet, vae, tokenizer, encoder


def load_controlnet_file(path: str, model_dir: str, device="cpu", dtype=torch.float32):
    """The ControlNet of a single cldm file (`control_model.*`, as lllyasviel's `control_sd15_canny.pth` and
    `control_v11p_sd15_canny.pth` are published).  A file holds no config: the network is the one
    `ControlNetModel.from_config` makes of `model_dir`'s unet/config.json, at the Canny defaults (3 conditioning
    channels, a (16, 32, 96, 256) conditioning embedding)."""
    from .controlnet import ControlNetModel
    unet_config = read_config(os.path.join(model_dir, "unet"))
    state = controlnet_state(load_single_file(path), unet_config.get("layers_per_block", 2))
    return assign_model(ControlNetModel.from_config, unet_config, state, device, dtype)
