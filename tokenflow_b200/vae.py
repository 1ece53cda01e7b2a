"""Random-init restatement of diffusers' `AutoencoderKL` at Stable Diffusion's VAE configuration: the stage that turns
frames into the latents the inversion and the edit work on, and the edited latents back into frames.

Like `sd_unet`, it keeps diffusers' module names, nesting and parameter shapes, so a real VAE state dict loads with
`strict=True`, and diffusers' call surface: `encode(x).latent_dist.mean / .sample()` and `decode(z).sample`.

    encoder.conv_in, encoder.down_blocks[0..3].resnets[0..1].{norm1, conv1, norm2, conv2, conv_shortcut},
    encoder.down_blocks[0..2].downsamplers[0].conv, encoder.mid_block.{resnets[0..1], attentions[0]},
    encoder.conv_norm_out, encoder.conv_out, quant_conv, post_quant_conv, decoder.conv_in, decoder.mid_block,
    decoder.up_blocks[0..3].resnets[0..2], decoder.up_blocks[0..2].upsamplers[0].conv, decoder.conv_norm_out,
    decoder.conv_out;  mid-block attention: group_norm, to_q, to_k, to_v, to_out.0

SD's VAE: block_out_channels (128, 256, 512, 512), 2 resnets per encoder block (3 per decoder block), 4 latent
channels, 32 groups, eps 1e-6, one single-head attention in each mid block.  `tiny_config()` keeps the topology at toy
width for CPU tests (8 groups, so its first level has 4 channels per group like SD's).

Every GroupNorm(+SiLU) goes through `sd_unet.norm_act`: on CUDA fp16 channels_last tensors every level runs
tf_group_norm_nhwc, the 128-channel levels at 4 channels per group; CPU, NCHW and fp32 runs keep ATen.  Convolutions are cuDNN, and the mid-block attention (head dim 512, S = 4096 at 512^2) is SDPA.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from .sd_unet import norm_act

SCALING_FACTOR = 0.18215           # SD's latent scale (reference run_tokenflow_pnp.py:151, :157)

# diffusers AutoencoderKL config keys that must hold the one value computed here (RGB frames, 4 latent channels, SD's
# latent scale and no shift, both 1x1 quant convolutions, the mid-block attention); each is diffusers' default
_VAE_FIXED = {"in_channels": 3, "out_channels": 3, "latent_channels": 4, "act_fn": "silu",
              "scaling_factor": SCALING_FACTOR, "shift_factor": None, "latents_mean": None, "latents_std": None,
              "use_quant_conv": True, "use_post_quant_conv": True, "mid_block_add_attention": True}


@dataclass
class VAEConfig:
    in_channels: int = 3
    out_channels: int = 3
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: int = 2
    latent_channels: int = 4
    norm_num_groups: int = 32
    eps: float = 1e-6


def sd_config() -> VAEConfig:
    return VAEConfig()


def tiny_config() -> VAEConfig:
    return VAEConfig(block_out_channels=(32, 64, 64, 64), layers_per_block=1, norm_num_groups=8)


class ResnetBlock2D(nn.Module):
    """diffusers `ResnetBlock2D` without a time embedding (temb_channels=None), output_scale_factor 1."""

    def __init__(self, in_channels: int, out_channels: int, groups: int, eps: float):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, in_channels, eps=eps)
        self.conv1 = nn.Conv2d(in_channels, out_channels, 3, padding=1)
        self.norm2 = nn.GroupNorm(groups, out_channels, eps=eps)
        self.dropout = nn.Dropout(0.0)
        self.conv2 = nn.Conv2d(out_channels, out_channels, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(in_channels, out_channels, 1) if in_channels != out_channels else None

    def forward(self, x):
        h = self.conv1(norm_act(self.norm1, x))
        h = self.conv2(self.dropout(norm_act(self.norm2, h)))
        if self.conv_shortcut is not None:
            x = self.conv_shortcut(x)
        return x + h


class Downsample2D(nn.Module):
    """Stride-2 conv after a (0, 1, 0, 1) zero pad (diffusers' encoder downsampler, padding=0)."""

    def __init__(self, channels: int):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, stride=2, padding=0)

    def forward(self, x):
        return self.conv(F.pad(x, (0, 1, 0, 1), mode="constant", value=0))


class Upsample2D(nn.Module):
    def __init__(self, channels: int):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, padding=1)

    def forward(self, x):
        return self.conv(F.interpolate(x, scale_factor=2.0, mode="nearest"))


class Attention(nn.Module):
    """The mid block's single-head spatial self-attention (diffusers `Attention` with a group_norm, residual
    connection, rescale 1), on SDPA."""

    def __init__(self, channels: int, groups: int, eps: float):
        super().__init__()
        self.heads = 1
        self.group_norm = nn.GroupNorm(groups, channels, eps=eps)
        self.to_q = nn.Linear(channels, channels)
        self.to_k = nn.Linear(channels, channels)
        self.to_v = nn.Linear(channels, channels)
        self.to_out = nn.ModuleList([nn.Linear(channels, channels), nn.Dropout(0.0)])

    def forward(self, x):
        b, c, h, w = x.shape
        residual = x
        y = norm_act(self.group_norm, x, silu=False)
        y = y.permute(0, 2, 3, 1).reshape(b, 1, h * w, c)        # a view for channels_last input
        o = F.scaled_dot_product_attention(self.to_q(y), self.to_k(y), self.to_v(y))
        o = self.to_out[1](self.to_out[0](o.reshape(b, h * w, c)))
        return o.reshape(b, h, w, c).permute(0, 3, 1, 2) + residual


class UNetMidBlock2D(nn.Module):
    def __init__(self, channels: int, groups: int, eps: float):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(channels, channels, groups, eps) for _ in range(2)])
        self.attentions = nn.ModuleList([Attention(channels, groups, eps)])

    def forward(self, x):
        return self.resnets[1](self.attentions[0](self.resnets[0](x)))


class DownEncoderBlock2D(nn.Module):
    def __init__(self, cin: int, cout: int, layers: int, groups: int, eps: float, add_downsample: bool):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, groups, eps) for i in range(layers)])
        self.downsamplers = nn.ModuleList([Downsample2D(cout)]) if add_downsample else None

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        return self.downsamplers[0](x) if self.downsamplers is not None else x


class UpDecoderBlock2D(nn.Module):
    def __init__(self, cin: int, cout: int, layers: int, groups: int, eps: float, add_upsample: bool):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, groups, eps) for i in range(layers)])
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_upsample else None

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        return self.upsamplers[0](x) if self.upsamplers is not None else x


class Encoder(nn.Module):
    def __init__(self, cfg: VAEConfig):
        super().__init__()
        ch, g, eps = cfg.block_out_channels, cfg.norm_num_groups, cfg.eps
        self.conv_in = nn.Conv2d(cfg.in_channels, ch[0], 3, padding=1)
        self.down_blocks = nn.ModuleList([
            DownEncoderBlock2D(ch[max(i - 1, 0)], ch[i], cfg.layers_per_block, g, eps, i < len(ch) - 1)
            for i in range(len(ch))])
        self.mid_block = UNetMidBlock2D(ch[-1], g, eps)
        self.conv_norm_out = nn.GroupNorm(g, ch[-1], eps=eps)
        self.conv_out = nn.Conv2d(ch[-1], 2 * cfg.latent_channels, 3, padding=1)

    def forward(self, x):
        x = self.conv_in(x)
        for blk in self.down_blocks:
            x = blk(x)
        return self.conv_out(norm_act(self.conv_norm_out, self.mid_block(x)))


class Decoder(nn.Module):
    def __init__(self, cfg: VAEConfig):
        super().__init__()
        ch, g, eps = tuple(reversed(cfg.block_out_channels)), cfg.norm_num_groups, cfg.eps
        self.conv_in = nn.Conv2d(cfg.latent_channels, ch[0], 3, padding=1)
        self.mid_block = UNetMidBlock2D(ch[0], g, eps)
        self.up_blocks = nn.ModuleList([
            UpDecoderBlock2D(ch[max(i - 1, 0)], ch[i], cfg.layers_per_block + 1, g, eps, i < len(ch) - 1)
            for i in range(len(ch))])
        self.conv_norm_out = nn.GroupNorm(g, ch[-1], eps=eps)
        self.conv_out = nn.Conv2d(ch[-1], cfg.out_channels, 3, padding=1)

    def forward(self, z):
        x = self.mid_block(self.conv_in(z))
        for blk in self.up_blocks:
            x = blk(x)
        return self.conv_out(norm_act(self.conv_norm_out, x))


class DiagonalGaussianDistribution:
    """diffusers' posterior: mean and log-variance halves of the moments, log-variance clamped to [-30, 20]."""

    def __init__(self, parameters: torch.Tensor):
        self.parameters = parameters
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)

    def sample(self, generator: Optional[torch.Generator] = None) -> torch.Tensor:
        noise = torch.randn(self.mean.shape, generator=generator, device=self.mean.device, dtype=self.mean.dtype)
        return self.mean + self.std * noise

    def mode(self) -> torch.Tensor:
        return self.mean


class EncoderOutput:
    def __init__(self, latent_dist: DiagonalGaussianDistribution):
        self.latent_dist = latent_dist


class DecoderOutput:
    def __init__(self, sample: torch.Tensor):
        self.sample = sample


class AutoencoderKL(nn.Module):
    def __init__(self, cfg: Optional[VAEConfig] = None):
        super().__init__()
        self.config = cfg = cfg or sd_config()
        self.encoder = Encoder(cfg)
        self.decoder = Decoder(cfg)
        self.quant_conv = nn.Conv2d(2 * cfg.latent_channels, 2 * cfg.latent_channels, 1)
        self.post_quant_conv = nn.Conv2d(cfg.latent_channels, cfg.latent_channels, 1)

    @classmethod
    def from_config(cls, config: dict) -> "AutoencoderKL":
        """The VAE a diffusers `vae/config.json` describes (its dict).  Reads block_out_channels, layers_per_block and
        norm_num_groups; raises ValueError, naming the key and the value, on anything else this restatement and the
        frame conversions around it do not compute (`_VAE_FIXED`, block types other than DownEncoderBlock2D /
        UpDecoderBlock2D).  A missing key takes diffusers' default; other keys (sample_size, force_upcast, ...) change
        nothing."""
        from .sd_unet import check_block_types, check_fixed
        check_fixed("vae", config, _VAE_FIXED)
        ch = tuple(int(c) for c in config.get("block_out_channels", (64,)))
        check_block_types("vae", config, "down_block_types", ["DownEncoderBlock2D"] * len(ch))
        check_block_types("vae", config, "up_block_types", ["UpDecoderBlock2D"] * len(ch))
        return cls(VAEConfig(block_out_channels=ch, layers_per_block=int(config.get("layers_per_block", 1)),
                             norm_num_groups=int(config.get("norm_num_groups", 32))))

    def encode(self, x: torch.Tensor) -> EncoderOutput:
        """x [N, 3, H, W] in [-1, 1] -> posterior over [N, 4, H/8, W/8] (unscaled)."""
        return EncoderOutput(DiagonalGaussianDistribution(self.quant_conv(self.encoder(x))))

    def decode(self, z: torch.Tensor) -> DecoderOutput:
        """z [N, 4, h, w] (unscaled) -> [N, 3, 8h, 8w] in about [-1, 1]."""
        return DecoderOutput(self.decoder(self.post_quant_conv(z)))


def build_vae(kind: str = "sd", seed: int = 1, device="cpu", dtype=torch.float32,
              init_on_device: bool = False) -> AutoencoderKL:
    """Random-init (default PyTorch inits) VAE, seeded like `sd_unet.build_unet`: drawn on the CPU by default, or
    directly on `device` with `init_on_device=True` (a different random stream)."""
    cfg = {"sd": sd_config, "tiny": tiny_config}[kind]()
    if init_on_device and torch.device(device).type == "cuda":
        cuda_state = torch.cuda.get_rng_state(device)
        torch.cuda.manual_seed(seed)
        try:
            with torch.device(device):
                net = AutoencoderKL(cfg)
        finally:
            torch.cuda.set_rng_state(cuda_state, device)
        return net.to(dtype=dtype).eval()
    gen_state = torch.random.get_rng_state()
    torch.manual_seed(seed)
    try:
        net = AutoencoderKL(cfg)
    finally:
        torch.random.set_rng_state(gen_state)
    return net.to(device=device, dtype=dtype).eval()
