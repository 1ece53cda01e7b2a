"""Synthetic diffusers checkpoint folders: the restated modules' random-init state dicts written in diffusers' layout,
for the tests and `tools/pipeline_bench.py` (no real weights are needed to exercise loading, the pipeline or its
timing).

`write_checkpoint` writes config.json files, the weights with safetensors (or torch.save), optionally as the fp16
variant or in shards, the VAE's mid-block attentions optionally under the deprecated names the published SD 1.x / 2.x
VAE files use, a random CLIP text encoder (small, or of CLIP ViT-L/14's size) and a CLIP tokenizer over single letters,
so every word of a prompt is several tokens.

`write_lora` writes random LoRAs for the loaded models in the kohya-ss, diffusers, PEFT and attention-processor layouts
`lora.read` takes.

The SD1.5, SD2.1 (768, v) and sd-controlnet-canny configs are the published config.json values of those checkpoints.
"""
import json
import os
import re

import torch

from . import sd_unet
from .controlnet import build_controlnet
from .vae import build_vae

_DOWN = ["CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"]
_UP = ["UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D"]

SD15_UNET = {
    "_class_name": "UNet2DConditionModel", "_diffusers_version": "0.6.0", "act_fn": "silu", "attention_head_dim": 8,
    "block_out_channels": [320, 640, 1280, 1280], "center_input_sample": False, "cross_attention_dim": 768,
    "down_block_types": _DOWN, "downsample_padding": 1, "flip_sin_to_cos": True, "freq_shift": 0, "in_channels": 4,
    "layers_per_block": 2, "mid_block_scale_factor": 1, "norm_eps": 1e-05, "norm_num_groups": 32, "out_channels": 4,
    "sample_size": 64, "up_block_types": _UP}
SD21_UNET = {
    "_class_name": "UNet2DConditionModel", "_diffusers_version": "0.10.0.dev0", "act_fn": "silu",
    "attention_head_dim": [5, 10, 20, 20], "block_out_channels": [320, 640, 1280, 1280], "center_input_sample": False,
    "cross_attention_dim": 1024, "down_block_types": _DOWN, "downsample_padding": 1, "dual_cross_attention": False,
    "flip_sin_to_cos": True, "freq_shift": 0, "in_channels": 4, "layers_per_block": 2, "mid_block_scale_factor": 1,
    "norm_eps": 1e-05, "norm_num_groups": 32, "num_class_embeds": None, "only_cross_attention": False,
    "out_channels": 4, "sample_size": 96, "up_block_types": _UP, "upcast_attention": True,
    "use_linear_projection": True}
SD_VAE = {
    "_class_name": "AutoencoderKL", "_diffusers_version": "0.6.0", "act_fn": "silu",
    "block_out_channels": [128, 256, 512, 512], "down_block_types": ["DownEncoderBlock2D"] * 4, "in_channels": 3,
    "latent_channels": 4, "layers_per_block": 2, "norm_num_groups": 32, "out_channels": 3, "sample_size": 512,
    "up_block_types": ["UpDecoderBlock2D"] * 4}
SD15_CANNY = {
    "_class_name": "ControlNetModel", "_diffusers_version": "0.16.0.dev0", "act_fn": "silu", "attention_head_dim": 8,
    "block_out_channels": [320, 640, 1280, 1280], "class_embed_type": None,
    "conditioning_embedding_out_channels": [16, 32, 96, 256], "controlnet_conditioning_channel_order": "rgb",
    "cross_attention_dim": 768, "down_block_types": _DOWN, "downsample_padding": 1, "flip_sin_to_cos": True,
    "freq_shift": 0, "in_channels": 4, "layers_per_block": 2, "mid_block_scale_factor": 1, "norm_eps": 1e-05,
    "norm_num_groups": 32, "num_class_embeds": None, "only_cross_attention": False,
    "projection_class_embeddings_input_dim": None, "resnet_time_scale_shift": "default", "upcast_attention": False,
    "use_linear_projection": False}
SD15_SCHEDULER = {
    "_class_name": "PNDMScheduler", "_diffusers_version": "0.6.0", "beta_end": 0.012, "beta_schedule": "scaled_linear",
    "beta_start": 0.00085, "num_train_timesteps": 1000, "set_alpha_to_one": False, "skip_prk_steps": True,
    "steps_offset": 1, "trained_betas": None, "clip_sample": False}
SD21_V_SCHEDULER = {
    "_class_name": "DDIMScheduler", "_diffusers_version": "0.8.0", "beta_end": 0.012, "beta_schedule": "scaled_linear",
    "beta_start": 0.00085, "clip_sample": False, "num_train_timesteps": 1000, "prediction_type": "v_prediction",
    "set_alpha_to_one": False, "skip_prk_steps": True, "steps_offset": 1, "trained_betas": None}

# the `tiny` kinds of build_unet / build_vae / build_controlnet, written as diffusers configs
TINY_UNET = {**SD15_UNET, "block_out_channels": [32, 64, 128, 128], "cross_attention_dim": 32,
             "attention_head_dim": [2, 2, 4, 4], "norm_num_groups": 8, "sample_size": 16}
TINY_VAE = {**SD_VAE, "block_out_channels": [32, 64, 64, 64], "layers_per_block": 1, "norm_num_groups": 8}
TINY_CANNY = {**SD15_CANNY, "block_out_channels": [32, 64, 128, 128], "cross_attention_dim": 32,
              "attention_head_dim": [2, 2, 4, 4], "norm_num_groups": 8,
              "conditioning_embedding_out_channels": [8, 8, 16, 16]}

UNET_CONFIGS = {"tiny": TINY_UNET, "sd15": SD15_UNET, "sd21": SD21_UNET}
CONTEXT = {"tiny": 32, "sd15": 768, "sd21": 1024}


# CLIP ViT-L/14's text tower (SD 1.x's text encoder), for timing text encoding at its real size
CLIP_L = {"vocab_size": 49408, "hidden_size": 768, "intermediate_size": 3072, "num_hidden_layers": 12,
          "num_attention_heads": 12}
_DEPRECATED_ATTENTION = {"to_q": "query", "to_k": "key", "to_v": "value", "to_out.0": "proj_attn"}


def deprecated_vae_names(state):
    """The VAE state dict with its mid-block attentions under diffusers' pre-0.14 AttentionBlock names (query, key,
    value, proj_attn), as the SD 1.x / 2.x VAE files on the hub were saved."""
    out = {}
    for key, value in state.items():
        head, sep, tail = key.partition(".attentions.0.")
        if sep and "mid_block" in head:
            for new, old in _DEPRECATED_ATTENTION.items():
                if tail.startswith(new + "."):
                    tail = old + tail[len(new):]
        out[head + sep + tail] = value
    return out


def write_model(folder, net, config, variant=None, dtype=None, fmt="safetensors", shards=1, rename=None):
    """`net`'s state dict (after `rename`) in diffusers' layout: config.json and diffusion_pytorch_model[.variant].<fmt>,
    or `shards` files with a .index[.variant].json weight map."""
    from safetensors.torch import save_file
    os.makedirs(folder, exist_ok=True)
    with open(os.path.join(folder, "config.json"), "w") as f:
        json.dump(config, f)
    state = {k: (v.to(dtype) if dtype is not None else v).contiguous().cpu() for k, v in net.state_dict().items()}
    if rename is not None:
        state = rename(state)
    ext = "safetensors" if fmt == "safetensors" else "bin"
    save = (lambda d, p: save_file(d, p)) if ext == "safetensors" else (lambda d, p: torch.save(d, p))
    name = "diffusion_pytorch_model" + (f".{variant}" if variant else "")
    if shards == 1:
        save(state, os.path.join(folder, f"{name}.{ext}"))
        return
    keys = sorted(state)
    weight_map = {}
    for i in range(shards):
        part = keys[i::shards]
        file = f"{name}-{i + 1:05d}-of-{shards:05d}.{ext}"
        save({k: state[k] for k in part}, os.path.join(folder, file))
        weight_map.update({k: file for k in part})
    index = f"diffusion_pytorch_model.{ext}.index" + (f".{variant}" if variant else "") + ".json"
    with open(os.path.join(folder, index), "w") as f:
        json.dump({"metadata": {}, "weight_map": weight_map}, f)


def write_text_side(model_dir, hidden, layers=1, heads=2, seed=0, text_config=None):
    """tokenizer/ (a CLIPTokenizer over single letters, so every word of a prompt is several tokens) and text_encoder/
    (a random CLIPTextModel of width `hidden`, or of the CLIPTextConfig fields `text_config` gives)."""
    from transformers import CLIPTextConfig, CLIPTextModel, CLIPTokenizer
    vocab = {"<|startoftext|>": 0, "<|endoftext|>": 1}
    for c in "abcdefghijklmnopqrstuvwxyz":
        vocab[c] = len(vocab)
        vocab[c + "</w>"] = len(vocab)
    raw = os.path.join(model_dir, "tokenizer_src")
    os.makedirs(raw, exist_ok=True)
    with open(os.path.join(raw, "vocab.json"), "w") as f:
        json.dump(vocab, f)
    with open(os.path.join(raw, "merges.txt"), "w") as f:
        f.write("#version: 0.2\n")
    tok = CLIPTokenizer(os.path.join(raw, "vocab.json"), os.path.join(raw, "merges.txt"), model_max_length=77)
    tok.save_pretrained(os.path.join(model_dir, "tokenizer"))
    fields = dict(vocab_size=len(vocab), hidden_size=hidden, intermediate_size=2 * hidden, num_hidden_layers=layers,
                  num_attention_heads=heads)
    cfg = CLIPTextConfig(**{**fields, **(text_config or {})}, max_position_embeddings=77, bos_token_id=0,
                         eos_token_id=1, pad_token_id=1)
    state = torch.random.get_rng_state()
    torch.manual_seed(seed)
    try:
        enc = CLIPTextModel(cfg)
    finally:
        torch.random.set_rng_state(state)
    enc.save_pretrained(os.path.join(model_dir, "text_encoder"))


def write_checkpoint(root, kind="tiny", scheduler=SD15_SCHEDULER, controlnet=False, variant=None, dtype=None,
                     fmt="safetensors", shards=1, init_device="cpu", deprecated_vae=False, text_config=None):
    """A diffusers checkpoint directory of the `kind` modules (random init, seeds 1 / 1 / 3) under `root`; with
    `controlnet`, a ControlNet folder beside it; with `deprecated_vae`, the VAE's attention under its published names.
    Returns (model_dir, controlnet_dir or None)."""
    model_dir = os.path.join(root, f"sd-{kind}")
    on_dev = torch.device(init_device).type == "cuda"
    unet = sd_unet.build_unet(kind, seed=1, device=init_device, init_on_device=on_dev)
    write_model(os.path.join(model_dir, "unet"), unet, UNET_CONFIGS[kind], variant, dtype, fmt, shards)
    del unet
    vae_kind = "tiny" if kind == "tiny" else "sd"
    vae = build_vae(vae_kind, seed=1, device=init_device, init_on_device=on_dev)
    write_model(os.path.join(model_dir, "vae"), vae, TINY_VAE if kind == "tiny" else SD_VAE, variant, dtype, fmt,
                shards, rename=deprecated_vae_names if deprecated_vae else None)
    del vae
    os.makedirs(os.path.join(model_dir, "scheduler"), exist_ok=True)
    with open(os.path.join(model_dir, "scheduler", "scheduler_config.json"), "w") as f:
        json.dump(scheduler, f)
    write_text_side(model_dir, CONTEXT[kind], layers=1, heads=2 if kind == "tiny" else 8, text_config=text_config)
    cn_dir = None
    if controlnet:
        cn_dir = os.path.join(root, f"controlnet-{kind}")
        cn = build_controlnet(kind, seed=3)
        write_model(cn_dir, cn, TINY_CANNY if kind == "tiny" else SD15_CANNY, variant, dtype, fmt, shards)
    return model_dir, cn_dir


# kohya-ss's target classes: its default LoRA (Transformer2DModel; CLIPAttention and CLIPMLP of the text encoder) and
# LoCon's convolution blocks
_TARGET_CLASSES = {"transformer": ("Transformer2DModel",), "conv": ("ResnetBlock2D", "Downsample2D", "Upsample2D"),
                   "text_encoder": ("CLIPAttention", "CLIPMLP")}


def lora_targets(unet, text_encoder, targets):
    """[(model, module path)] of the `targets`, in `named_modules` order: "attention" (the UNet attentions' to_q,
    to_k, to_v and to_out.0), and kohya's sets "transformer" (every Linear and Conv2d inside a Transformer2DModel: 192
    on SD), "conv" (inside ResnetBlock2D, Downsample2D and Upsample2D: LoCon) and "text_encoder" (inside CLIPAttention
    and CLIPMLP)."""
    out = []
    for model, net in (("unet", unet), ("text_encoder", text_encoder)):
        classes = sum((_TARGET_CLASSES[t] for t in targets if t != "attention"), ())
        inside = [n for n, m in net.named_modules() if type(m).__name__ in classes]
        for name, m in net.named_modules():
            if not isinstance(m, (torch.nn.Linear, torch.nn.Conv2d)):
                continue
            attention = (model == "unet" and "attention" in targets
                         and re.search(r"\.attn[12]\.(to_q|to_k|to_v|to_out\.0)$", name) is not None)
            if attention or any(name.startswith(p + ".") for p in inside):
                out.append((model, name))
    return out


def _lora_stem(layout, model, name):
    if layout == "kohya":
        return {"unet": "lora_unet_", "text_encoder": "lora_te_"}[model] + name.replace(".", "_")
    if layout in ("diffusers", "peft"):
        return f"{model}.{name}"
    head, _, proj = name.rpartition(".attn")
    attn, _, proj = proj.partition(".")
    if model != "unet" or proj not in ("to_q", "to_k", "to_v", "to_out.0"):
        raise ValueError(f"the attention-processor layout has no key for {model} module {name!r}")
    return f"unet.{head}.attn{attn}.processor.{proj.split('.')[0]}_lora"


_LORA_SUFFIX = {"kohya": (".lora_down.weight", ".lora_up.weight"),
                "diffusers": (".lora.down.weight", ".lora.up.weight"),
                "peft": (".lora_A.weight", ".lora_B.weight"), "processor": (".down.weight", ".up.weight")}


def write_lora(path, unet, text_encoder, layout="kohya", rank=4, targets=("attention",), alpha=None, seed=0):
    """A random LoRA of rank `rank` for the `lora_targets` of `targets` in `layout` ("kohya", "diffusers", "peft" or
    "processor"), written with safetensors (a `.bin` / `.pt` path with torch.save) in fp16, as LoRAs are published.
    The values depend only on the targets' shapes, `rank` and `seed`, never on the layout: down ~ N(0, 1/fan_in) [rank, in, (kh, kw)], up ~ N(0, 1/rank)
    [out, rank, (1, 1)], so a merged update is about as large as the default init's weights.  `alpha` (a number) is
    written as each module's `.alpha`; None writes none.  Returns the targets."""
    from safetensors.torch import save_file
    g = torch.Generator().manual_seed(seed)
    found = lora_targets(unet, text_encoder, targets)
    nets = {"unet": unet, "text_encoder": text_encoder}
    down_sfx, up_sfx = _LORA_SUFFIX[layout]
    state = {}
    for model, name in found:
        shape = nets[model].get_submodule(name).weight.shape
        fan_in = shape[1:].numel()
        down = torch.randn((rank, *shape[1:]), generator=g) / fan_in ** 0.5
        up = torch.randn((shape[0], rank, *([1, 1] if len(shape) == 4 else [])), generator=g) / rank ** 0.5
        stem = _lora_stem(layout, model, name)
        state[stem + down_sfx], state[stem + up_sfx] = down.half(), up.half()
        if alpha is not None:
            state[stem + ".alpha"] = torch.tensor(float(alpha), dtype=torch.float16)
    if str(path).endswith(".safetensors"):
        save_file(state, str(path))
    else:
        torch.save(state, str(path))
    return found
