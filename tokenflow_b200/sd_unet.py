"""Random-init Stable-Diffusion-shaped UNet with the diffusers class names / attributes the
TokenFlow hooks patch.

`diffusers` is not installed here and there is no network, so the L1 "third-party model runtime"
(SURVEY.md §1, Appendix B) is restated as a small local module tree.  It is plumbing, not the
product: every conv / linear / cross-attention here is a stock PyTorch (cuDNN / cuBLAS) call.  Two
elementwise stages run on the library's kernels when the body runs fp16 channels_last on an H100
(`norm_act`, `GEGLU`): GroupNorm with the time-embedding add before it and the SiLU after it
(tf_group_norm_nhwc: ATen has no channels_last GroupNorm and would copy to NCHW and back around every
norm), and the GEGLU gate (tf_geglu).  Both keep the eager fp16 rounding sequence; anything else (CPU,
NCHW, fp32, channel counts the kernel does not cover) runs the ATen ops.
The hooks discover modules *by class name* (reference util.py:46-58) and by the hard-coded SD
topology (reference tokenflow_utils.py:20-40, 208-214), so the names and nesting below follow the
mid-2023 diffusers layout:

    unet.down_blocks[0..2].attentions[0..1].transformer_blocks[0].{attn1,attn2}
    unet.mid_block.attentions[0].transformer_blocks[0].{attn1,attn2}
    unet.up_blocks[1..3].attentions[0..2].transformer_blocks[0].{attn1,attn2}
    unet.up_blocks[1].resnets[1]

Shapes: SD1.5 (heads 8 everywhere, ctx 768, conv proj_in) and SD2.1 (head_dim 64, ctx 1024,
linear proj_in).  `tiny=True` keeps the topology but shrinks the channels for CPU tests.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F


@dataclass
class UNetConfig:
    in_channels: int = 4
    out_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    layers_per_block: int = 2
    cross_attention_dim: int = 768
    # heads per resolution level (SD1.5: 8 everywhere; SD2.1: 5/10/20/20 → head_dim 64)
    num_heads: Tuple[int, ...] = (8, 8, 8, 8)
    norm_num_groups: int = 32
    use_linear_projection: bool = False
    sample_size: Optional[int] = 64


# diffusers UNet2DConditionModel / ControlNetModel config keys.  `from_config` reads the keys that set the topology
# (`encoder_fields`); each key below must hold the one value computed here, which is also diffusers' default, so a
# missing key passes.  Every other key (_class_name, _diffusers_version, upcast_attention, ...) changes nothing.
_ENCODER_FIXED = {
    "in_channels": 4, "mid_block_type": "UNetMidBlock2DCrossAttn", "only_cross_attention": False,
    "dual_cross_attention": False, "class_embed_type": None, "num_class_embeds": None, "addition_embed_type": None,
    "addition_time_embed_dim": None, "projection_class_embeddings_input_dim": None, "encoder_hid_dim": None,
    "encoder_hid_dim_type": None, "time_cond_proj_dim": None, "flip_sin_to_cos": True, "freq_shift": 0,
    "act_fn": "silu", "norm_eps": 1e-5, "downsample_padding": 1, "mid_block_scale_factor": 1,
    "resnet_time_scale_shift": "default", "attention_type": "default",
}
_UNET_FIXED = {
    "out_channels": 4, "center_input_sample": False, "resnet_skip_time_act": False, "resnet_out_scale_factor": 1.0,
    "time_embedding_type": "positional", "time_embedding_dim": None, "time_embedding_act_fn": None,
    "timestep_post_act": None, "conv_in_kernel": 3, "conv_out_kernel": 3, "class_embeddings_concat": False,
    "mid_block_only_cross_attention": None, "cross_attention_norm": None, "reverse_transformer_layers_per_block": None,
    "dropout": 0.0,
}


def check_fixed(what: str, config: dict, fixed: dict) -> None:
    """ValueError naming the key and the value for the first key of `config` that does not hold `fixed[key]`."""
    for key, value in fixed.items():
        got = config.get(key, value)
        if got != value:
            raise ValueError(f"{what} config {key}={got!r} is not supported (only {value!r})")


def check_block_types(what: str, config: dict, key: str, want) -> None:
    got = list(config.get(key, want))
    if got != list(want):
        raise ValueError(f"{what} config {key}={got!r} is not supported (only {list(want)!r})")


def encoder_fields(config: dict, what: str) -> dict:
    """The UNetConfig fields of a diffusers UNet or ControlNet config dict, after refusing the settings the blocks
    here do not compute: an input other than 4 latent channels (depth: 5, inpainting: 9), SDXL's extra embeddings and
    several transformer layers per block, class or timestep-condition embeddings, a mid block other than the
    cross-attention one, block types outside SD's arrangement, and the other keys of `_ENCODER_FIXED`.

    diffusers' naming quirk: without `num_attention_heads`, `attention_head_dim` holds the number of heads per level
    (SD1.5: 8, SD2.x: [5, 10, 20, 20]), which is how diffusers itself reads it."""
    check_fixed(what, config, _ENCODER_FIXED)
    layers = config.get("transformer_layers_per_block", 1)
    if any(v != 1 for v in (layers if isinstance(layers, (list, tuple)) else [layers])):
        raise ValueError(f"{what} config transformer_layers_per_block={layers!r} is not supported (only 1)")
    ch = tuple(int(c) for c in config.get("block_out_channels", (320, 640, 1280, 1280)))
    n = len(ch)
    check_block_types(what, config, "down_block_types", ["CrossAttnDownBlock2D"] * (n - 1) + ["DownBlock2D"])
    per_block = config.get("layers_per_block", 2)
    if not isinstance(per_block, int):
        raise ValueError(f"{what} config layers_per_block={per_block!r} is not supported (only one int)")
    ctx = config.get("cross_attention_dim", 1280)
    if isinstance(ctx, (list, tuple)):
        if len(set(ctx)) != 1:
            raise ValueError(f"{what} config cross_attention_dim={ctx!r} is not supported (only one width)")
        ctx = ctx[0]
    heads = config.get("num_attention_heads") or config.get("attention_head_dim", 8)
    heads = tuple(int(h) for h in heads) if isinstance(heads, (list, tuple)) else (int(heads),) * n
    if len(heads) != n:
        raise ValueError(f"{what} config has {len(heads)} head counts for {n} blocks")
    return dict(block_out_channels=ch, layers_per_block=per_block, cross_attention_dim=int(ctx), num_heads=heads,
                norm_num_groups=int(config.get("norm_num_groups", 32)),
                use_linear_projection=bool(config.get("use_linear_projection", False)))


def sd15_config() -> UNetConfig:
    return UNetConfig()


def sd21_config() -> UNetConfig:
    return UNetConfig(cross_attention_dim=1024, num_heads=(5, 10, 20, 20),
                      use_linear_projection=True, sample_size=96)


def tiny_config(ctx: int = 32) -> UNetConfig:
    """SD topology (16 transformer blocks) at toy width for CPU plumbing tests."""
    return UNetConfig(block_out_channels=(32, 64, 128, 128), cross_attention_dim=ctx,
                      num_heads=(2, 2, 4, 4), norm_num_groups=8, sample_size=16)


class GroupNorm(nn.GroupNorm):
    """GroupNorm that stays in fp16 when fed fp16 under autocast (fp32 statistics inside the kernel).
    Autocast's default policy would up-cast the input, write an fp32 output and let the next conv cast
    it back — three extra full-tensor passes per norm that dominated the UNet body's time."""

    def forward(self, x):
        if x.dtype == torch.float16 and x.is_cuda and torch.is_autocast_enabled():
            with torch.autocast("cuda", enabled=False):
                return F.group_norm(x, self.num_groups, self.weight, self.bias, self.eps)
        return super().forward(x)


def norm_act(norm: nn.GroupNorm, x: torch.Tensor, bias: Optional[torch.Tensor] = None,
             silu: bool = True) -> torch.Tensor:
    """[SiLU](norm(x [+ bias[:, :, None, None]])): one tf_group_norm_nhwc call (two launches, three passes over x)
    for the operands `CudaOps.group_norm_nhwc_supported` accepts (CUDA fp16 channels_last, at least 8 channels per
    group, or 4 without a bias: the VAE's 128-channel levels), else the eager ATen sequence (fp16 add, GroupNorm,
    SiLU)."""
    from .ops import CudaOps, body_ops
    if CudaOps.group_norm_nhwc_supported(x, norm, bias):
        ops = body_ops()
        if ops is not None:
            return ops.group_norm_nhwc(x, norm, bias, silu)
    if bias is not None:
        x = x + bias[:, :, None, None]
    x = norm(x)
    return F.silu(x) if silu else x


class BodyLayerNorm(nn.LayerNorm):
    """Same for norm2 / norm3 of the transformer blocks.  (norm1 stays a plain nn.LayerNorm: its fp32
    autocast output is part of the reference's NN-field arithmetic.)"""

    def forward(self, x):
        if x.dtype == torch.float16 and x.is_cuda and torch.is_autocast_enabled():
            with torch.autocast("cuda", enabled=False):
                return F.layer_norm(x, self.normalized_shape, self.weight, self.bias, self.eps)
        return super().forward(x)


class UNetOutput(dict):
    """`unet(...)['sample']` (reference run_tokenflow_pnp.py:210) and `.sample` both work."""

    @property
    def sample(self):
        return self["sample"]


# --------------------------------------------------------------------------------------------
# attention / transformer
# --------------------------------------------------------------------------------------------
class Attention(nn.Module):
    """diffusers `Attention` surface used by the hooks (SURVEY.md Appendix B)."""

    def __init__(self, query_dim: int, cross_attention_dim: Optional[int], heads: int, dim_head: int):
        super().__init__()
        inner = heads * dim_head
        self.heads = heads
        self.scale = dim_head ** -0.5
        ctx = cross_attention_dim if cross_attention_dim is not None else query_dim
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(ctx, inner, bias=False)
        self.to_v = nn.Linear(ctx, inner, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(inner, query_dim), nn.Dropout(0.0)])

    def head_to_batch_dim(self, t: torch.Tensor) -> torch.Tensor:
        b, s, _ = t.shape
        h = self.heads
        return t.reshape(b, s, h, -1).permute(0, 2, 1, 3).reshape(b * h, s, -1)

    def batch_to_head_dim(self, t: torch.Tensor) -> torch.Tensor:
        bh, s, d = t.shape
        h = self.heads
        return t.reshape(bh // h, h, s, d).permute(0, 2, 1, 3).reshape(bh // h, s, d * h)

    def forward(self, hidden_states, encoder_hidden_states=None, attention_mask=None):
        ctx = hidden_states if encoder_hidden_states is None else encoder_hidden_states
        b, s, _ = hidden_states.shape
        h = self.heads
        q = self.to_q(hidden_states).view(b, s, h, -1).transpose(1, 2)
        k = self.to_k(ctx).view(b, ctx.shape[1], h, -1).transpose(1, 2)
        v = self.to_v(ctx).view(b, ctx.shape[1], h, -1).transpose(1, 2)
        o = F.scaled_dot_product_attention(q, k, v, attn_mask=attention_mask, scale=self.scale)
        o = o.transpose(1, 2).reshape(b, s, -1)
        return self.to_out[1](self.to_out[0](o))


class GEGLU(nn.Module):
    def __init__(self, dim_in: int, dim_out: int):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)

    def forward(self, x):
        # two GEMMs on the two halves of the fused weight: both outputs contiguous, so gelu and the
        # product run vectorised (chunking one fused output leaves strided views and the slow path)
        w_x, w_g = self.proj.weight.chunk(2, dim=0)
        b_x, b_g = self.proj.bias.chunk(2, dim=0)
        xh, g = F.linear(x, w_x, b_x), F.linear(x, w_g, b_g)
        if xh.is_cuda and xh.dtype == g.dtype == torch.float16:
            from .ops import body_ops
            ops = body_ops()
            if ops is not None:
                return ops.geglu(xh, g)             # one pass: gelu(g) is never written
        return xh * F.gelu(g)


class FeedForward(nn.Module):
    def __init__(self, dim: int, mult: int = 4):
        super().__init__()
        self.net = nn.ModuleList([GEGLU(dim, dim * mult), nn.Dropout(0.0), nn.Linear(dim * mult, dim)])

    def forward(self, x):
        for m in self.net:
            x = m(x)
        return x


class BasicTransformerBlock(nn.Module):
    """Stock block; `set_tokenflow` swaps its class for the TokenFlow subclass."""

    def __init__(self, dim: int, heads: int, dim_head: int, cross_attention_dim: int):
        super().__init__()
        self.only_cross_attention = False
        self.use_ada_layer_norm = False
        self.use_ada_layer_norm_zero = False
        self.norm1 = nn.LayerNorm(dim)
        self.attn1 = Attention(dim, None, heads, dim_head)
        self.norm2 = BodyLayerNorm(dim)
        self.attn2 = Attention(dim, cross_attention_dim, heads, dim_head)
        self.norm3 = BodyLayerNorm(dim)
        self.ff = FeedForward(dim)

    def forward(self, hidden_states, attention_mask=None, encoder_hidden_states=None,
                encoder_attention_mask=None, timestep=None, cross_attention_kwargs=None,
                class_labels=None):
        hidden_states = self.attn1(self.norm1(hidden_states)) + hidden_states
        hidden_states = self.attn2(self.norm2(hidden_states),
                                   encoder_hidden_states=encoder_hidden_states,
                                   attention_mask=encoder_attention_mask) + hidden_states
        return self.ff(self.norm3(hidden_states)) + hidden_states


class Transformer2DModel(nn.Module):
    def __init__(self, channels: int, heads: int, cross_attention_dim: int, groups: int, linear_proj: bool):
        super().__init__()
        self.use_linear_projection = linear_proj
        self.norm = GroupNorm(groups, channels, eps=1e-6)
        if linear_proj:
            self.proj_in = nn.Linear(channels, channels)
            self.proj_out = nn.Linear(channels, channels)
        else:
            self.proj_in = nn.Conv2d(channels, channels, 1)
            self.proj_out = nn.Conv2d(channels, channels, 1)
        self.transformer_blocks = nn.ModuleList(
            [BasicTransformerBlock(channels, heads, channels // heads, cross_attention_dim)])

    def forward(self, hidden_states, encoder_hidden_states=None):
        b, c, hh, ww = hidden_states.shape
        residual = hidden_states
        x = norm_act(self.norm, hidden_states, silu=False)
        if self.use_linear_projection:
            x = x.permute(0, 2, 3, 1).reshape(b, hh * ww, c)
            x = self.proj_in(x)
        else:
            x = self.proj_in(x)
            x = x.permute(0, 2, 3, 1).reshape(b, hh * ww, c)
        for blk in self.transformer_blocks:
            x = blk(x, attention_mask=None, encoder_hidden_states=encoder_hidden_states,
                    timestep=None, cross_attention_kwargs=None, class_labels=None)
        if self.use_linear_projection:
            x = self.proj_out(x)
            x = x.reshape(b, hh, ww, c).permute(0, 3, 1, 2)
        else:
            x = x.reshape(b, hh, ww, c).permute(0, 3, 1, 2)
            x = self.proj_out(x)
        return x + residual


# --------------------------------------------------------------------------------------------
# resnet / sampling
# --------------------------------------------------------------------------------------------
class ResnetBlock2D(nn.Module):
    """Attribute names follow reference tokenflow_utils.py:54-96 (the conv-injection hook)."""

    def __init__(self, in_channels: int, out_channels: int, temb_channels: int, groups: int):
        super().__init__()
        self.norm1 = GroupNorm(groups, in_channels, eps=1e-5)
        self.conv1 = nn.Conv2d(in_channels, out_channels, 3, padding=1)
        self.time_emb_proj = nn.Linear(temb_channels, out_channels)
        self.norm2 = GroupNorm(groups, out_channels, eps=1e-5)
        self.dropout = nn.Dropout(0.0)
        self.conv2 = nn.Conv2d(out_channels, out_channels, 3, padding=1)
        self.nonlinearity = nn.SiLU()
        self.upsample = None
        self.downsample = None
        self.time_embedding_norm = "default"
        self.output_scale_factor = 1.0
        self.conv_shortcut = nn.Conv2d(in_channels, out_channels, 1) if in_channels != out_channels else None

    def forward(self, input_tensor, temb):
        h = self.conv1(norm_act(self.norm1, input_tensor))
        t = self.time_emb_proj(self.nonlinearity(temb)) if temb is not None else None
        h = self.conv2(self.dropout(norm_act(self.norm2, h, bias=t)))       # temb add + norm2 + SiLU
        if self.conv_shortcut is not None:
            input_tensor = self.conv_shortcut(input_tensor)
        out = input_tensor + h
        return out if self.output_scale_factor == 1.0 else out / self.output_scale_factor


class Downsample2D(nn.Module):
    def __init__(self, channels: int):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, stride=2, padding=1)

    def forward(self, x):
        return self.conv(x)


class Upsample2D(nn.Module):
    def __init__(self, channels: int):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, padding=1)

    def forward(self, x, output_size=None):
        """Nearest-neighbour doubling, or nearest-neighbour to `output_size` (h, w): the size of the skip the next up
        block concatenates, when a latent side is not a multiple of the UNet's overall downsampling (diffusers'
        `upsample_size`)."""
        if output_size is None:
            return self.conv(F.interpolate(x, scale_factor=2.0, mode="nearest"))
        return self.conv(F.interpolate(x, size=output_size, mode="nearest"))


class CrossAttnDownBlock2D(nn.Module):
    def __init__(self, cin, cout, temb, layers, heads, ctx, groups, linear_proj, add_downsample):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, temb, groups) for i in range(layers)])
        self.attentions = nn.ModuleList([Transformer2DModel(cout, heads, ctx, groups, linear_proj) for _ in range(layers)])
        self.downsamplers = nn.ModuleList([Downsample2D(cout)]) if add_downsample else None

    def forward(self, x, temb, ctx):
        outs = []
        for r, a in zip(self.resnets, self.attentions):
            x = a(r(x, temb), encoder_hidden_states=ctx)
            outs.append(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
            outs.append(x)
        return x, outs


class DownBlock2D(nn.Module):
    def __init__(self, cin, cout, temb, layers, groups, add_downsample):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, temb, groups) for i in range(layers)])
        self.downsamplers = nn.ModuleList([Downsample2D(cout)]) if add_downsample else None

    def forward(self, x, temb, ctx=None):
        outs = []
        for r in self.resnets:
            x = r(x, temb)
            outs.append(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
            outs.append(x)
        return x, outs


class UNetMidBlock2DCrossAttn(nn.Module):
    def __init__(self, channels, temb, heads, ctx, groups, linear_proj):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(channels, channels, temb, groups) for _ in range(2)])
        self.attentions = nn.ModuleList([Transformer2DModel(channels, heads, ctx, groups, linear_proj)])

    def forward(self, x, temb, ctx):
        x = self.resnets[0](x, temb)
        x = self.attentions[0](x, encoder_hidden_states=ctx)
        return self.resnets[1](x, temb)


class UpBlock2D(nn.Module):
    def __init__(self, cin, cout, prev, temb, layers, groups, add_upsample):
        super().__init__()
        res = []
        for i in range(layers):
            skip = cin if i == layers - 1 else cout
            rin = prev if i == 0 else cout
            res.append(ResnetBlock2D(rin + skip, cout, temb, groups))
        self.resnets = nn.ModuleList(res)
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_upsample else None

    def forward(self, x, skips, temb, ctx=None, upsample_size=None):
        for r in self.resnets:
            x = r(torch.cat([x, skips.pop()], dim=1), temb)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x, upsample_size)
        return x


class CrossAttnUpBlock2D(nn.Module):
    def __init__(self, cin, cout, prev, temb, layers, heads, ctx, groups, linear_proj, add_upsample):
        super().__init__()
        res = []
        for i in range(layers):
            skip = cin if i == layers - 1 else cout
            rin = prev if i == 0 else cout
            res.append(ResnetBlock2D(rin + skip, cout, temb, groups))
        self.resnets = nn.ModuleList(res)
        self.attentions = nn.ModuleList([Transformer2DModel(cout, heads, ctx, groups, linear_proj) for _ in range(layers)])
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_upsample else None

    def forward(self, x, skips, temb, ctx, upsample_size=None):
        for r, a in zip(self.resnets, self.attentions):
            x = r(torch.cat([x, skips.pop()], dim=1), temb)
            x = a(x, encoder_hidden_states=ctx)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x, upsample_size)
        return x


# --------------------------------------------------------------------------------------------
# UNet
# --------------------------------------------------------------------------------------------
def sinusoidal_timestep_embedding(timesteps: torch.Tensor, dim: int) -> torch.Tensor:
    """flip_sin_to_cos=True, freq_shift=0 (the SD settings)."""
    half = dim // 2
    exponent = -math.log(10000.0) * torch.arange(half, dtype=torch.float32, device=timesteps.device) / half
    emb = timesteps[:, None].float() * torch.exp(exponent)[None, :]
    return torch.cat([torch.cos(emb), torch.sin(emb)], dim=-1)


class TimestepEmbedding(nn.Module):
    def __init__(self, cin: int, cout: int):
        super().__init__()
        self.linear_1 = nn.Linear(cin, cout)
        self.act = nn.SiLU()
        self.linear_2 = nn.Linear(cout, cout)

    def forward(self, x):
        return self.linear_2(self.act(self.linear_1(x)))


class UNet2DConditionModel(nn.Module):
    def __init__(self, cfg: Optional[UNetConfig] = None):
        super().__init__()
        cfg = cfg or sd15_config()
        self.config = cfg
        ch = cfg.block_out_channels
        temb = ch[0] * 4
        g = cfg.norm_num_groups
        lp = cfg.use_linear_projection
        ctx = cfg.cross_attention_dim
        L = cfg.layers_per_block
        self.conv_in = nn.Conv2d(cfg.in_channels, ch[0], 3, padding=1)
        self.time_embedding = TimestepEmbedding(ch[0], temb)

        down = []
        cout = ch[0]
        for i in range(len(ch)):
            cin, cout = cout, ch[i]
            last = i == len(ch) - 1
            if not last:
                down.append(CrossAttnDownBlock2D(cin, cout, temb, L, cfg.num_heads[i], ctx, g, lp, True))
            else:
                down.append(DownBlock2D(cin, cout, temb, L, g, False))
        self.down_blocks = nn.ModuleList(down)
        self.mid_block = UNetMidBlock2DCrossAttn(ch[-1], temb, cfg.num_heads[-1], ctx, g, lp)

        rev = list(reversed(ch))
        rev_heads = list(reversed(cfg.num_heads))
        up = []
        cout = rev[0]
        for i in range(len(rev)):
            prev, cout = cout, rev[i]
            cin = rev[min(i + 1, len(rev) - 1)]
            last = i == len(rev) - 1
            if i == 0:
                up.append(UpBlock2D(cin, cout, prev, temb, L + 1, g, not last))
            else:
                up.append(CrossAttnUpBlock2D(cin, cout, prev, temb, L + 1, rev_heads[i], ctx, g, lp, not last))
        self.up_blocks = nn.ModuleList(up)
        self.conv_norm_out = GroupNorm(g, ch[0], eps=1e-5)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(ch[0], cfg.out_channels, 3, padding=1)

    @classmethod
    def from_config(cls, config: dict) -> "UNet2DConditionModel":
        """The UNet a diffusers `unet/config.json` describes (its dict), built with this module's default init.
        Raises ValueError, naming the key and the value, on any setting it does not compute (`encoder_fields`, the
        up blocks, and the UNet-only keys of `_UNET_FIXED`); a missing key takes diffusers' default.
        `upcast_attention` is accepted and changes nothing (DESIGN.md §1 f-6)."""
        check_fixed("unet", config, _UNET_FIXED)
        fields = encoder_fields(config, "unet")
        n = len(fields["block_out_channels"])
        check_block_types("unet", config, "up_block_types", ["UpBlock2D"] + ["CrossAttnUpBlock2D"] * (n - 1))
        return cls(UNetConfig(**fields, sample_size=config.get("sample_size")))

    def forward(self, sample, timestep, encoder_hidden_states=None, down_block_additional_residuals=None,
                mid_block_additional_residual=None, return_dict: bool = True, **_):
        """diffusers' UNet2DConditionModel.forward.  A ControlNet's outputs (controlnet.py) come in as
        `down_block_additional_residuals`, one per skip, added to the skips before the up blocks read them, and
        `mid_block_additional_residual`, added to the mid-block output.  `return_dict=False` returns `(sample,)`.
        Other keyword arguments are accepted and ignored."""
        if not torch.is_tensor(timestep):
            timestep = torch.tensor([timestep], device=sample.device)
        timestep = timestep.reshape(-1).expand(sample.shape[0]).to(sample.device)
        t_emb = sinusoidal_timestep_embedding(timestep, self.config.block_out_channels[0])
        emb = self.time_embedding(t_emb.to(self.conv_in.weight.dtype))
        x = self.conv_in(sample)
        skips = [x]
        for blk in self.down_blocks:
            x, outs = blk(x, emb, encoder_hidden_states)
            skips.extend(outs)
        if down_block_additional_residuals is not None:
            if len(down_block_additional_residuals) != len(skips):
                raise ValueError(f"{len(down_block_additional_residuals)} down-block residuals for {len(skips)} skips")
            skips = [s + r for s, r in zip(skips, down_block_additional_residuals)]
        x = self.mid_block(x, emb, encoder_hidden_states)
        if mid_block_additional_residual is not None:
            x = x + mid_block_additional_residual
        # diffusers' rule for latents whose sides are not multiples of 2 ** (number of upsamplers): every up block but
        # the last upsamples to the size of the skip it will concatenate next (a plain doubling would give 22 rows
        # where the skip has 21); other latents keep the doubling
        factor = 2 ** sum(b.upsamplers is not None for b in self.up_blocks)
        ragged = any(s % factor for s in sample.shape[-2:])
        for blk in self.up_blocks:
            size = None
            if ragged and blk.upsamplers is not None:
                size = skips[-len(blk.resnets) - 1].shape[-2:]
            x = blk(x, skips, emb, encoder_hidden_states, upsample_size=size)
        x = self.conv_out(norm_act(self.conv_norm_out, x))          # conv_norm_out + conv_act (SiLU)
        return UNetOutput(sample=x) if return_dict else (x,)


def build_unet(kind: str = "sd15", seed: int = 1, device="cpu", dtype=torch.float32,
               init_on_device: bool = False) -> UNet2DConditionModel:
    """Random-init (default PyTorch inits) SD-shape UNet, seeded like the reference default
    (configs/config_pnp.yaml:2).  By default the parameters are drawn on the CPU (device independent, what
    the tests and golden vectors use) and moved; `init_on_device=True` draws them directly on `device`
    (much faster under torchrun's OMP_NUM_THREADS=1; identical on every rank for a given seed and device
    type, but a different random stream than the CPU init)."""
    cfg = {"sd15": sd15_config, "sd21": sd21_config, "tiny": tiny_config}[kind]()
    if init_on_device and torch.device(device).type == "cuda":
        try:
            cuda_state = torch.cuda.get_rng_state(device)
            torch.cuda.manual_seed(seed)
            try:
                with torch.device(device):
                    net = UNet2DConditionModel(cfg)
            finally:
                torch.cuda.set_rng_state(cuda_state, device)
            return net.to(dtype=dtype).eval()
        except Exception:  # noqa: BLE001  — fall back to the CPU init below
            pass
    gen_state = torch.random.get_rng_state()
    torch.manual_seed(seed)
    try:
        net = UNet2DConditionModel(cfg)
    finally:
        torch.random.set_rng_state(gen_state)
    return net.to(device=device, dtype=dtype).eval()
