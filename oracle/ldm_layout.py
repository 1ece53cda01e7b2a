"""Stable Diffusion models written in the original LDM single-file layout, for the tests of `checkpoint.py`'s
single-file converters.

The names follow the way LDM's own modules are built, not a table of renames: CompVis' `openaimodel.UNetModel`
(`time_embed`, then `input_blocks` appended one TimestepEmbedSequential at a time, `middle_block`, `output_blocks`
appended level by level from the lowest resolution, `out`), lllyasviel's `cldm.ControlNet` (the same encoder plus
`input_hint_block`, a Sequential of convolutions with a SiLU after each but the last, one `zero_convs` entry per input
block and `middle_block_out`), `diffusionmodules.model.Encoder` / `Decoder` (`down[i].block[j]`, `mid.block_1`,
`mid.attn_1` on 1x1 convolutions, and the decoder's levels inserted at the front of `up` as they are built), the
`ResBlock`'s Sequentials (`in_layers` = GroupNorm, SiLU, conv; `emb_layers` = SiLU, linear; `out_layers` = GroupNorm,
SiLU, dropout, conv), transformers' CLIPTextModel for SD 1.x, and open_clip's text transformer (`resblocks` with q, k
and v packed into `in_proj`) for SD 2.x.  A Sequential's index counts its parameterless layers, as in LDM.

The tensors are taken from this package's modules by walking their attributes in the order LDM builds its own.
Nothing here is shared with the converters, so a wrong rename there is not cancelled by the same mistake here.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

Tensors = Dict[str, torch.Tensor]


def _put(out: Tensors, name: str, module) -> None:
    for key, value in module.state_dict().items():
        out[f"{name}.{key}"] = value


def _resblock(out: Tensors, name: str, r) -> None:
    """openaimodel.ResBlock: in_layers = (GroupNorm, SiLU, conv), emb_layers = (SiLU, linear),
    out_layers = (GroupNorm, SiLU, Dropout, conv), skip_connection when the width changes."""
    _put(out, f"{name}.in_layers.0", r.norm1)
    _put(out, f"{name}.in_layers.2", r.conv1)
    _put(out, f"{name}.emb_layers.1", r.time_emb_proj)
    _put(out, f"{name}.out_layers.0", r.norm2)
    _put(out, f"{name}.out_layers.3", r.conv2)
    if r.conv_shortcut is not None:
        _put(out, f"{name}.skip_connection", r.conv_shortcut)


def _unet_encoder(out: Tensors, net) -> int:
    """time_embed, input_blocks and middle_block of UNetModel (also cldm.ControlNet's); returns the number of input
    blocks."""
    _put(out, "time_embed.0", net.time_embedding.linear_1)       # Sequential(linear, SiLU, linear)
    _put(out, "time_embed.2", net.time_embedding.linear_2)
    input_blocks = [[("conv", net.conv_in)]]
    for level in net.down_blocks:
        attentions = getattr(level, "attentions", None)
        for j, r in enumerate(level.resnets):
            layers = [("res", r)]
            if attentions is not None:
                layers.append(("module", attentions[j]))
            input_blocks.append(layers)
        if level.downsamplers is not None:
            input_blocks.append([("down", level.downsamplers[0])])
    for b, layers in enumerate(input_blocks):
        for sub, (kind, module) in enumerate(layers):
            name = f"input_blocks.{b}.{sub}"
            if kind == "res":
                _resblock(out, name, module)
            elif kind == "down":
                _put(out, f"{name}.op", module.conv)                 # Downsample.op
            else:
                _put(out, name, module)
    mid = net.mid_block
    _resblock(out, "middle_block.0", mid.resnets[0])
    _put(out, "middle_block.1", mid.attentions[0])
    _resblock(out, "middle_block.2", mid.resnets[1])
    return len(input_blocks)


def ldm_unet(unet, prefix: str = "model.diffusion_model.") -> Tensors:
    """`sd_unet.UNet2DConditionModel`'s tensors under openaimodel.UNetModel's names."""
    out: Tensors = {}
    _unet_encoder(out, unet)
    b = 0
    for level in unet.up_blocks:
        attentions = getattr(level, "attentions", None)
        for j, r in enumerate(level.resnets):
            sub = 0
            _resblock(out, f"output_blocks.{b}.{sub}", r)
            if attentions is not None:
                sub += 1
                _put(out, f"output_blocks.{b}.{sub}", attentions[j])
            if j == len(level.resnets) - 1 and level.upsamplers is not None:
                sub += 1
                _put(out, f"output_blocks.{b}.{sub}.conv", level.upsamplers[0].conv)     # Upsample.conv
            b += 1
    _put(out, "out.0", unet.conv_norm_out)                       # Sequential(GroupNorm, SiLU, conv)
    _put(out, "out.2", unet.conv_out)
    return {prefix + k: v for k, v in out.items()}


def ldm_controlnet(controlnet, prefix: str = "control_model.") -> Tensors:
    """`controlnet.ControlNetModel`'s tensors under cldm.ControlNet's names."""
    out: Tensors = {}
    n_input = _unet_encoder(out, controlnet)
    emb = controlnet.controlnet_cond_embedding
    hint = [emb.conv_in, *emb.blocks, emb.conv_out]              # a SiLU after each convolution but the last
    for k, conv in enumerate(hint):
        _put(out, f"input_hint_block.{2 * k}", conv)
    assert len(controlnet.controlnet_down_blocks) == n_input    # one zero conv per input block
    for i, conv in enumerate(controlnet.controlnet_down_blocks):
        _put(out, f"zero_convs.{i}.0", conv)
    _put(out, "middle_block_out.0", controlnet.controlnet_mid_block)
    return {prefix + k: v for k, v in out.items()}


def _vae_resnet(out: Tensors, name: str, r) -> None:
    for attr in ("norm1", "conv1", "norm2", "conv2"):
        _put(out, f"{name}.{attr}", getattr(r, attr))
    if r.conv_shortcut is not None:
        _put(out, f"{name}.nin_shortcut", r.conv_shortcut)


def _vae_mid(out: Tensors, name: str, mid) -> None:
    _vae_resnet(out, f"{name}.block_1", mid.resnets[0])
    attn = mid.attentions[0]
    _put(out, f"{name}.attn_1.norm", attn.group_norm)
    for conv, linear in (("q", attn.to_q), ("k", attn.to_k), ("v", attn.to_v), ("proj_out", attn.to_out[0])):
        out[f"{name}.attn_1.{conv}.weight"] = linear.weight.detach()[:, :, None, None]     # a 1x1 Conv2d in LDM
        out[f"{name}.attn_1.{conv}.bias"] = linear.bias.detach()
    _vae_resnet(out, f"{name}.block_2", mid.resnets[1])


def ldm_vae(vae, prefix: str = "first_stage_model.") -> Tensors:
    """`vae.AutoencoderKL`'s tensors under LDM's AutoencoderKL names."""
    out: Tensors = {}
    enc, dec = vae.encoder, vae.decoder
    _put(out, "encoder.conv_in", enc.conv_in)
    for i, level in enumerate(enc.down_blocks):
        for j, r in enumerate(level.resnets):
            _vae_resnet(out, f"encoder.down.{i}.block.{j}", r)
        if level.downsamplers is not None:
            _put(out, f"encoder.down.{i}.downsample.conv", level.downsamplers[0].conv)
    _vae_mid(out, "encoder.mid", enc.mid_block)
    _put(out, "encoder.norm_out", enc.conv_norm_out)
    _put(out, "encoder.conv_out", enc.conv_out)
    _put(out, "decoder.conv_in", dec.conv_in)
    _vae_mid(out, "decoder.mid", dec.mid_block)
    up = []
    for level in dec.up_blocks:                                   # built from the lowest resolution: up.insert(0, .)
        up.insert(0, level)
    for i, level in enumerate(up):
        for j, r in enumerate(level.resnets):
            _vae_resnet(out, f"decoder.up.{i}.block.{j}", r)
        if level.upsamplers is not None:
            _put(out, f"decoder.up.{i}.upsample.conv", level.upsamplers[0].conv)
    _put(out, "decoder.norm_out", dec.conv_norm_out)
    _put(out, "decoder.conv_out", dec.conv_out)
    _put(out, "quant_conv", vae.quant_conv)
    _put(out, "post_quant_conv", vae.post_quant_conv)
    return {prefix + k: v for k, v in out.items()}


def ldm_clip(encoder, text_model_level: bool = True, position_ids: bool = False,
             prefix: str = "cond_stage_model.transformer.") -> Tensors:
    """SD 1.x's FrozenCLIPEmbedder: transformers' CLIPTextModel state dict under `cond_stage_model.transformer.`, with
    the `text_model.` level of newer transformers or without it, and with the `position_ids` buffer older
    transformers saved."""
    state = {k: v for k, v in encoder.state_dict().items()}
    if position_ids:
        n = encoder.config.max_position_embeddings
        state["text_model.embeddings.position_ids"] = torch.arange(n)[None]
    if not text_model_level:
        state = {k[len("text_model."):]: v for k, v in state.items()}
    return {prefix + k: v for k, v in state.items()}


def ldm_openclip(encoder, extra_blocks: int = 1, seed: int = 0, prefix: str = "cond_stage_model.model.") -> Tensors:
    """SD 2.x's FrozenOpenCLIPEmbedder: open_clip's text transformer holding the CLIPTextModel's weights, plus
    `extra_blocks` random resblocks after its layers (SD 2.x files hold one more block than the penultimate layer
    the model reads; a negative count drops layers instead), `text_projection` and `logit_scale`."""
    tm = encoder.text_model
    out: Tensors = {"token_embedding.weight": tm.embeddings.token_embedding.weight.detach(),
                    "positional_embedding": tm.embeddings.position_embedding.weight.detach()}
    blocks = []
    for layer in tm.encoder.layers:
        att = layer.self_attn
        block: Tensors = {}
        _put(block, "ln_1", layer.layer_norm1)
        block["attn.in_proj_weight"] = torch.cat([att.q_proj.weight, att.k_proj.weight, att.v_proj.weight]).detach()
        block["attn.in_proj_bias"] = torch.cat([att.q_proj.bias, att.k_proj.bias, att.v_proj.bias]).detach()
        _put(block, "attn.out_proj", att.out_proj)
        _put(block, "ln_2", layer.layer_norm2)
        _put(block, "mlp.c_fc", layer.mlp.fc1)
        _put(block, "mlp.c_proj", layer.mlp.fc2)
        blocks.append(block)
    g = torch.Generator().manual_seed(seed)
    for _ in range(max(extra_blocks, 0)):
        blocks.append({k: torch.randn(v.shape, generator=g).to(v.dtype) for k, v in blocks[0].items()})
    for i, block in enumerate(blocks[:len(blocks) + min(extra_blocks, 0)]):
        out.update({f"transformer.resblocks.{i}.{k}": v for k, v in block.items()})
    _put(out, "ln_final", tm.final_layer_norm)
    width = tm.final_layer_norm.weight.shape[0]
    out["text_projection"] = torch.randn(width, width, generator=g)
    out["logit_scale"] = torch.tensor(math.log(1 / 0.07))
    return {prefix + k: v for k, v in out.items()}


def ema_copy(state: Tensors, prefix: str = "model.diffusion_model.") -> Tensors:
    """LDM's LitEma buffers of the UNet: `model_ema.<name without dots>` for every `model.diffusion_model.<name>`,
    here with other values (the negated weights), plus `decay` and `num_updates`."""
    out = {"model_ema." + k[len("model."):].replace(".", ""): -v for k, v in state.items() if k.startswith(prefix)}
    out["model_ema.decay"] = torch.tensor(0.9999)
    out["model_ema.num_updates"] = torch.tensor(1000, dtype=torch.int32)
    return out


def save(path: str, state: Tensors, dtype: Optional[torch.dtype] = None) -> None:
    """`state` as `.safetensors`, or with torch.save: a `.ckpt` as Lightning saves one, {"state_dict": ...,
    "global_step": 1}, anything else (`.pth`) as the bare dict.  `dtype` casts the floating-point tensors."""
    state = {k: (v.to(dtype) if dtype is not None and v.is_floating_point() else v).detach().contiguous().cpu()
             for k, v in state.items()}
    if path.endswith(".safetensors"):
        from safetensors.torch import save_file
        save_file(state, path)
    elif path.endswith(".ckpt"):
        torch.save({"state_dict": state, "global_step": 1}, path)
    else:
        torch.save(state, path)
