"""diffusers' `ControlNetModel` at the lllyasviel/sd-controlnet-canny configuration, on this package's UNet blocks.

The reference's ControlNet path (preprocess.py:129-149 `controlnet_pred`) runs every UNet call as
`down, mid = controlnet(x, t, ctx, controlnet_cond=canny, conditioning_scale=1)` followed by
`unet(x, t, ctx, down_block_additional_residuals=down, mid_block_additional_residual=mid)`.  The network is a copy of
the UNet's encoder (`conv_in`, `time_embedding`, `down_blocks`, `mid_block`, the same names and shapes, so
`from_unet` can copy them), plus
  * `controlnet_cond_embedding`: conv 3 -> 16, then (16, 32, 96, 256) with a stride-2 convolution at every second
    block, SiLU between the convolutions, and a zero-initialised conv_out to the UNet's first width (320);
  * `controlnet_down_blocks.0-11`: zero-initialised 1x1 convolutions, one per UNet skip;
  * `controlnet_mid_block`: a zero-initialised 1x1 convolution on the mid-block output.
The state-dict names and shapes are diffusers', so real weights load with `strict=True`.  Every lllyasviel ControlNet
of the v1.1 family (depth, softedge, lineart, tile, ip2p, ...) has this architecture; `MultiControlNetModel` runs
several of them on one UNet call, as diffusers' does.

The blocks are `sd_unet`'s, so a CUDA fp16 channels_last ControlNet runs its GroupNorm and GEGLU sites on the
library's kernels like the UNet body does.  Its attention stays plain: the TokenFlow hooks patch the UNet they are
given and nothing else (the reference never patches its ControlNet).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from .sd_unet import (CrossAttnDownBlock2D, DownBlock2D, TimestepEmbedding, UNet2DConditionModel, UNetConfig,
                      UNetMidBlock2DCrossAttn, sd15_config, sinusoidal_timestep_embedding, tiny_config)


@dataclass
class ControlNetConfig:
    unet: UNetConfig
    conditioning_channels: int = 3
    conditioning_embedding_out_channels: Tuple[int, ...] = (16, 32, 96, 256)


def sd15_canny_config() -> ControlNetConfig:
    return ControlNetConfig(sd15_config())


def tiny_canny_config() -> ControlNetConfig:
    """The tiny UNet's encoder with a narrower conditioning embedding (still three stride-2 stages: the cond is 8x the
    latent size)."""
    return ControlNetConfig(tiny_config(), conditioning_embedding_out_channels=(8, 8, 16, 16))


class ControlNetConditioningEmbedding(nn.Module):
    """diffusers' ControlNetConditioningEmbedding: the 3-channel edge image at pixel resolution -> the UNet's first
    width at latent resolution."""

    def __init__(self, embedding_channels: int, conditioning_channels: int, block_out_channels: Tuple[int, ...]):
        super().__init__()
        self.conv_in = nn.Conv2d(conditioning_channels, block_out_channels[0], 3, padding=1)
        blocks = []
        for cin, cout in zip(block_out_channels[:-1], block_out_channels[1:]):
            blocks.append(nn.Conv2d(cin, cin, 3, padding=1))
            blocks.append(nn.Conv2d(cin, cout, 3, padding=1, stride=2))
        self.blocks = nn.ModuleList(blocks)
        self.conv_out = nn.Conv2d(block_out_channels[-1], embedding_channels, 3, padding=1)

    def forward(self, cond):
        x = F.silu(self.conv_in(cond))
        for blk in self.blocks:
            x = F.silu(blk(x))
        return self.conv_out(x)


def _zero(module: nn.Module) -> nn.Module:
    for p in module.parameters():
        nn.init.zeros_(p)
    return module


class ControlNetModel(nn.Module):
    def __init__(self, cfg: Optional[ControlNetConfig] = None):
        super().__init__()
        cfg = cfg or sd15_canny_config()
        self.config = cfg
        u = cfg.unet
        ch = u.block_out_channels
        temb = ch[0] * 4
        g, lp, ctx, L = u.norm_num_groups, u.use_linear_projection, u.cross_attention_dim, u.layers_per_block
        self.conv_in = nn.Conv2d(u.in_channels, ch[0], 3, padding=1)
        self.time_embedding = TimestepEmbedding(ch[0], temb)
        self.controlnet_cond_embedding = ControlNetConditioningEmbedding(
            ch[0], cfg.conditioning_channels, cfg.conditioning_embedding_out_channels)
        down, zero_convs = [], [nn.Conv2d(ch[0], ch[0], 1)]
        cout = ch[0]
        for i in range(len(ch)):
            cin, cout = cout, ch[i]
            last = i == len(ch) - 1
            if not last:
                down.append(CrossAttnDownBlock2D(cin, cout, temb, L, u.num_heads[i], ctx, g, lp, True))
            else:
                down.append(DownBlock2D(cin, cout, temb, L, g, False))
            zero_convs += [nn.Conv2d(cout, cout, 1) for _ in range(L + (0 if last else 1))]
        self.down_blocks = nn.ModuleList(down)
        self.controlnet_down_blocks = nn.ModuleList(zero_convs)
        self.mid_block = UNetMidBlock2DCrossAttn(ch[-1], temb, u.num_heads[-1], ctx, g, lp)
        self.controlnet_mid_block = nn.Conv2d(ch[-1], ch[-1], 1)

    def zero_init(self) -> "ControlNetModel":
        """Zero the zero convolutions (the conditioning embedding's conv_out, the 12 down-block and the mid-block 1x1
        convolutions), as diffusers' constructor does: the residuals are then exactly zero."""
        _zero(self.controlnet_cond_embedding.conv_out)
        _zero(self.controlnet_down_blocks)
        _zero(self.controlnet_mid_block)
        return self

    @classmethod
    def from_config(cls, config: dict) -> "ControlNetModel":
        """The ControlNet a diffusers ControlNet `config.json` describes (its dict).  The UNet-encoder keys are read and
        refused as `sd_unet.encoder_fields` does; conditioning_channels and conditioning_embedding_out_channels are
        read; a channel order other than rgb and global pooling of the conditions are refused (ValueError naming the
        key and the value).  A missing key takes diffusers' default."""
        from .sd_unet import check_fixed, encoder_fields
        check_fixed("controlnet", config, {"controlnet_conditioning_channel_order": "rgb",
                                           "global_pool_conditions": False})
        unet = UNetConfig(**encoder_fields(config, "controlnet"))
        emb = tuple(int(c) for c in config.get("conditioning_embedding_out_channels", (16, 32, 96, 256)))
        return cls(ControlNetConfig(unet, conditioning_channels=int(config.get("conditioning_channels", 3)),
                                    conditioning_embedding_out_channels=emb))

    @classmethod
    def from_unet(cls, unet: UNet2DConditionModel, cfg: Optional[ControlNetConfig] = None) -> "ControlNetModel":
        """diffusers' `ControlNetModel.from_unet`: conv_in, time_embedding, down_blocks and mid_block copied from
        `unet`, the zero convolutions zero, the rest of the conditioning embedding freshly initialised."""
        cfg = cfg or ControlNetConfig(unet.config)
        p = next(unet.parameters())
        net = cls(cfg).to(device=p.device, dtype=p.dtype)
        for name in ("conv_in", "time_embedding", "down_blocks", "mid_block"):
            getattr(net, name).load_state_dict(getattr(unet, name).state_dict())
        if unet.conv_in.weight.is_contiguous(memory_format=torch.channels_last):
            net = net.to(memory_format=torch.channels_last)
        return net.zero_init().eval()

    def forward(self, sample, timestep, encoder_hidden_states=None, controlnet_cond=None,
                conditioning_scale: float = 1.0, return_dict: bool = False, **_):
        """(down_block_res_samples, mid_block_res_sample): the 12 residuals of the UNet's skips and the one of its
        mid-block output, times `conditioning_scale` (diffusers' ControlNetModel.forward without guess_mode).
        `controlnet_cond` is [N, 3, 8h, 8w] for latents of [N, 4, h, w]."""
        if controlnet_cond is None:
            raise ValueError("ControlNetModel.forward needs controlnet_cond")
        if not torch.is_tensor(timestep):
            timestep = torch.tensor([timestep], device=sample.device)
        timestep = timestep.reshape(-1).expand(sample.shape[0]).to(sample.device)
        t_emb = sinusoidal_timestep_embedding(timestep, self.config.unet.block_out_channels[0])
        emb = self.time_embedding(t_emb.to(self.conv_in.weight.dtype))
        x = self.conv_in(sample)
        x = x + self.controlnet_cond_embedding(controlnet_cond.to(x.dtype))
        skips = [x]
        for blk in self.down_blocks:
            x, outs = blk(x, emb, encoder_hidden_states)
            skips.extend(outs)
        x = self.mid_block(x, emb, encoder_hidden_states)
        down = [zc(s) for s, zc in zip(skips, self.controlnet_down_blocks)]
        mid = self.controlnet_mid_block(x)
        if conditioning_scale != 1.0:
            down = [d * conditioning_scale for d in down]
            mid = mid * conditioning_scale
        return tuple(down), mid


class MultiControlNetModel(nn.Module):
    """diffusers' `MultiControlNetModel`: several ControlNets on one UNet call, with `ControlNetModel`'s call signature.

    `controlnet_cond` is one tensor [N, Σ c_k, H, W], the nets' conditionings concatenated along channels in net order;
    it is split by each net's `conditioning_channels`, so every caller that gathers or slices the conditioning by frame
    handles one tensor whatever the number of nets.  Each net's residuals are scaled by its own scale, then added in net
    order in the residuals' dtype (one rounding per add in fp16), as diffusers sums them; the UNet adds the sum to its
    skips as it adds one net's residuals."""

    def __init__(self, nets):
        super().__init__()
        self.nets = nn.ModuleList(nets)
        if len(self.nets) == 0:
            raise ValueError("MultiControlNetModel needs at least one ControlNet")

    @property
    def conditioning_channels(self) -> Tuple[int, ...]:
        return tuple(net.config.conditioning_channels for net in self.nets)

    def forward(self, sample, timestep, encoder_hidden_states=None, controlnet_cond=None, conditioning_scale=1.0,
                return_dict: bool = False, **_):
        """(down_block_res_samples, mid_block_res_sample) of the nets' summed residuals.  `conditioning_scale` is a
        float for every net or a list of one per net."""
        scales = conditioning_scale_for(self, conditioning_scale)
        if controlnet_cond is None or controlnet_cond.shape[1] != sum(self.conditioning_channels):
            got = None if controlnet_cond is None else controlnet_cond.shape[1]
            raise ValueError(f"MultiControlNetModel needs controlnet_cond with {sum(self.conditioning_channels)} "
                             f"channels {self.conditioning_channels}, got {got}")
        down, mid = None, None
        for net, cond, scale in zip(self.nets, controlnet_cond.split(self.conditioning_channels, dim=1), scales):
            d, m = net(sample, timestep, encoder_hidden_states, controlnet_cond=cond, conditioning_scale=scale)
            if down is None:
                down, mid = d, m
            else:
                down = tuple(a + b for a, b in zip(down, d))
                mid = mid + m
        return down, mid


def controlnets(controlnet) -> list:
    """The ControlNets `controlnet` runs: [] for None, its nets for a MultiControlNetModel, else [controlnet]."""
    if controlnet is None:
        return []
    return list(controlnet.nets) if isinstance(controlnet, MultiControlNetModel) else [controlnet]


def conditioning_scale_for(controlnet, scale):
    """`scale` (a number, or a list of one per net) as `controlnet` takes it: a float for a ControlNetModel (a list of
    one is unwrapped), a list of floats for a MultiControlNetModel (a number applies to every net).  A list of another
    length raises ValueError naming both lengths.  Without a ControlNet there is no scale: None."""
    if controlnet is None:
        return None
    k = len(controlnets(controlnet))
    if isinstance(scale, (list, tuple)):
        if len(scale) != k:
            raise ValueError(f"{len(scale)} ControlNet conditioning scales for {k} ControlNets")
        scales = [float(s) for s in scale]
    else:
        scales = [float(scale)] * k
    return scales if isinstance(controlnet, MultiControlNetModel) else scales[0]


def build_controlnet(kind: str = "sd15", seed: int = 1, device="cpu", dtype=torch.float32) -> ControlNetModel:
    """Random-init ControlNet (default PyTorch inits for every parameter, the zero convolutions included, so that the
    residuals are not zero, as with trained weights), drawn on the CPU from `seed` and moved."""
    cfg = {"sd15": sd15_canny_config, "tiny": tiny_canny_config}[kind]()
    gen_state = torch.random.get_rng_state()
    torch.manual_seed(seed)
    try:
        net = ControlNetModel(cfg)
    finally:
        torch.random.set_rng_state(gen_state)
    return net.to(device=device, dtype=dtype).eval()


def controlnet_residuals(controlnet, x, t, ctx, cond, scale=1.0):
    """The first half of the reference's `controlnet_pred` (preprocess.py:130-137): the UNet keyword arguments of one
    call, {} when there is no ControlNet.  `scale` is as `conditioning_scale_for` returns it."""
    if controlnet is None:
        return {}
    down, mid = controlnet(x, t, encoder_hidden_states=ctx, controlnet_cond=cond, conditioning_scale=scale,
                           return_dict=False)
    return {"down_block_additional_residuals": down, "mid_block_additional_residual": mid}
