"""Stable Diffusion's UNet, VAE and ControlNet as plain fp64 functions of a state dict in the original LDM layout.

This is an independent statement of what the models compute, for checking `tokenflow_b200`'s diffusers-shaped
restatements (`sd_unet`, `vae`, `controlnet`) and the converters that load LDM files into them.  It follows the module
structure of CompVis' latent-diffusion code and lllyasviel's ControlNet, not diffusers':

* `openaimodel.UNetModel`: `time_embed` on `timestep_embedding`, `input_blocks` / `middle_block` / `output_blocks`
  built from `model_channels`, `channel_mult`, `num_res_blocks`, `attention_resolutions` and `num_heads` /
  `num_head_channels`, every input block's output pushed on `hs` and popped by the output blocks;
* `ResBlock`: `in_layers` (GroupNorm, SiLU, conv), `emb_layers` (SiLU, linear) added per channel, `out_layers`
  (GroupNorm, SiLU, dropout, conv), and `skip_connection` (a 1x1 conv when the width changes);
* `attention.SpatialTransformer` with its `BasicTransformerBlock` (self-attention, cross-attention, GEGLU
  feed-forward, each after a LayerNorm and added to its input), `proj_in` / `proj_out` as 1x1 convolutions around
  the 'b c h w -> b (h w) c' rearrangement, or as linear layers inside it (`use_linear_in_transformer`, SD 2.x);
* `cldm.ControlNet`: the same encoder, `input_hint_block` (convolutions with a SiLU after each but the last, stride 2
  at every second one) added after the first input block, one `zero_convs` entry per input block and
  `middle_block_out`, all scaled by the conditioning scale as `ControlLDM` does; `ControlledUnetModel` adds the last
  residual to the middle block's output and each other one to the skip it pairs with;
* `diffusionmodules.model.Encoder` / `Decoder` (`down[i].block[j]`, `mid.block_1`, `mid.attn_1` with q, k, v and
  proj_out as 1x1 convolutions, `up` indexed from the highest resolution and run from the lowest, the encoder's
  downsampling convolution after a (0, 1, 0, 1) zero pad) and `DiagonalGaussianDistribution` (mean, log-variance
  clamped to [-30, 20]).

Every operation is `torch.nn.functional` on fp64 tensors, except the sinusoid of `timestep_embedding`, which LDM takes
in fp32 (so does diffusers); it is cast to fp64 before `time_embed`.

Two extensions over LDM's hard-coded constants let the toy configurations of the tests be stated: `norm_groups`
(LDM: 32) and a per-level tuple for `num_heads` (LDM: one number).  One rule is diffusers' and not LDM's: for latents
whose sides are not multiples of 2 ** (number of upsamplers), diffusers upsamples each output level to the size of
the skip the next level concatenates (its `upsample_size`), where LDM only doubles and would fail to concatenate.
`unet` restates diffusers there.

The state dict is the one `oracle/ldm_layout.py` writes (`ldm_unet`, `ldm_vae`, `ldm_controlnet`), or a `.safetensors`
file in that layout, or a `Params` of one.  `unet` and `controlnet` refuse a state dict holding a tensor their
forward does not read; the VAE's encoder and decoder read one dict between them, so a caller passes both the same
`Params` and calls `check_all_read` after.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch
import torch.nn.functional as F

Tensors = Dict[str, torch.Tensor]
SCALE_FACTOR = 0.18215                 # SD's latent scale


class Params:
    """The tensors of one model (the keys under `prefix`) as fp64 on `device`, with a record of the names read."""

    def __init__(self, state: Union[str, Tensors], prefix: str, device):
        if isinstance(state, str):
            from safetensors.torch import load_file
            state = load_file(state)
        self.tensors = {k[len(prefix):]: v for k, v in state.items() if k.startswith(prefix)}
        if not self.tensors:
            raise KeyError(f"no tensors under {prefix!r}")
        self.device, self.read = device, set()

    def __call__(self, name: str) -> torch.Tensor:
        self.read.add(name)
        return self.tensors[name].to(device=self.device, dtype=torch.float64)

    def check_all_read(self) -> None:
        unread = sorted(set(self.tensors) - self.read)
        if unread:
            raise KeyError(f"{len(unread)} tensors not used by the forward, first {unread[:4]}")


def _params(state: Union[str, Tensors, Params], prefix: str, device) -> Params:
    return state if isinstance(state, Params) else Params(state, prefix, device)


def to_fp64(state: Tensors, device) -> Tensors:
    """`state` as fp64 tensors on `device`: convert once when the same weights run several forwards."""
    return {k: v.to(device=device, dtype=torch.float64) for k, v in state.items()}


# ------------------------------------------------------------------------------------------------
# layers
# ------------------------------------------------------------------------------------------------
def conv(p: Params, name: str, x, stride: int = 1, padding: Optional[int] = None):
    w = p(f"{name}.weight")
    return F.conv2d(x, w, p(f"{name}.bias"), stride=stride, padding=w.shape[-1] // 2 if padding is None else padding)


def linear(p: Params, name: str, x, bias: bool = True):
    return F.linear(x, p(f"{name}.weight"), p(f"{name}.bias") if bias else None)


def group_norm(p: Params, name: str, x, groups: int, eps: float):
    return F.group_norm(x, groups, p(f"{name}.weight"), p(f"{name}.bias"), eps)


def layer_norm(p: Params, name: str, x):
    w = p(f"{name}.weight")
    return F.layer_norm(x, w.shape, w, p(f"{name}.bias"), 1e-5)


def timestep_embedding(timesteps: torch.Tensor, dim: int, max_period: int = 10000) -> torch.Tensor:
    """LDM's `diffusionmodules.util.timestep_embedding`: [cos, sin] of t times fp32 frequencies, as fp64."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(start=0, end=half, dtype=torch.float32,
                                                           device=timesteps.device) / half)
    args = timesteps[:, None].float() * freqs[None]
    embedding = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    if dim % 2:
        embedding = torch.cat([embedding, torch.zeros_like(embedding[:, :1])], dim=-1)
    return embedding.double()


# ------------------------------------------------------------------------------------------------
# openaimodel.UNetModel
# ------------------------------------------------------------------------------------------------
def res_block(p: Params, name: str, x, emb, groups: int):
    """openaimodel.ResBlock (use_scale_shift_norm=False): GroupNorm32 has eps 1e-5."""
    h = conv(p, f"{name}.in_layers.2", F.silu(group_norm(p, f"{name}.in_layers.0", x, groups, 1e-5)))
    h = h + linear(p, f"{name}.emb_layers.1", F.silu(emb))[:, :, None, None]
    h = conv(p, f"{name}.out_layers.3", F.silu(group_norm(p, f"{name}.out_layers.0", h, groups, 1e-5)))
    skip = conv(p, f"{name}.skip_connection", x) if x.shape[1] != h.shape[1] else x
    return skip + h


def attention(p: Params, name: str, x, context, heads: int):
    """attention.CrossAttention: q from x, k and v from the context (x for self-attention), no biases, softmax over
    the keys of q k^T * dim_head ** -0.5 per head, then to_out.0."""
    context = x if context is None else context
    q = linear(p, f"{name}.to_q", x, bias=False)
    k = linear(p, f"{name}.to_k", context, bias=False)
    v = linear(p, f"{name}.to_v", context, bias=False)
    b, n, inner = q.shape
    d = inner // heads
    q, k, v = (t.reshape(b, t.shape[1], heads, d).permute(0, 2, 1, 3) for t in (q, k, v))   # b n (h d) -> b h n d
    sim = torch.matmul(q, k.transpose(-1, -2)) * d ** -0.5
    out = torch.matmul(sim.softmax(dim=-1), v)
    return linear(p, f"{name}.to_out.0", out.permute(0, 2, 1, 3).reshape(b, n, inner))


def feed_forward(p: Params, name: str, x):
    """attention.FeedForward(glu=True): GEGLU (value half first, gate half second, exact GELU), dropout, linear."""
    h, gate = linear(p, f"{name}.net.0.proj", x).chunk(2, dim=-1)
    return linear(p, f"{name}.net.2", h * F.gelu(gate))


def transformer_block(p: Params, name: str, x, context, heads: int):
    x = attention(p, f"{name}.attn1", layer_norm(p, f"{name}.norm1", x), None, heads) + x
    x = attention(p, f"{name}.attn2", layer_norm(p, f"{name}.norm2", x), context, heads) + x
    return feed_forward(p, f"{name}.ff", layer_norm(p, f"{name}.norm3", x)) + x


def spatial_transformer(p: Params, name: str, x, context, heads: int, groups: int, use_linear: bool):
    """attention.SpatialTransformer with one BasicTransformerBlock; its GroupNorm (`Normalize`) has eps 1e-6."""
    b, c, h, w = x.shape
    x_in = x
    x = group_norm(p, f"{name}.norm", x, groups, 1e-6)
    if not use_linear:
        x = conv(p, f"{name}.proj_in", x)
    x = x.permute(0, 2, 3, 1).reshape(b, h * w, -1)                      # b c h w -> b (h w) c
    if use_linear:
        x = linear(p, f"{name}.proj_in", x)
    x = transformer_block(p, f"{name}.transformer_blocks.0", x, context, heads)
    if use_linear:
        x = linear(p, f"{name}.proj_out", x)
    x = x.reshape(b, h, w, -1).permute(0, 3, 1, 2)                       # b (h w) c -> b c h w
    if not use_linear:
        x = conv(p, f"{name}.proj_out", x)
    return x + x_in


Layer = Tuple[str, int]              # ("res" | "attn" | "down" | "up" | "conv", number of heads for "attn")


def unet_layout(model_channels: int, channel_mult: Sequence[int], num_res_blocks: int,
                attention_resolutions: Sequence[int], num_heads: Union[int, Sequence[int]] = -1,
                num_head_channels: int = -1) -> Tuple[List[List[Layer]], List[Layer], List[List[Layer]]]:
    """(input_blocks, middle_block, output_blocks) as UNetModel.__init__ appends them: the layers of each
    TimestepEmbedSequential, in order.  `ds` is the downsampling factor; a level gets a SpatialTransformer after each
    ResBlock when `ds` is in `attention_resolutions`.  Heads: `num_heads` (per level when a sequence), or
    width // `num_head_channels` when that is not -1."""
    def heads(level: int) -> int:
        ch = model_channels * channel_mult[level]
        if num_head_channels != -1:
            return ch // num_head_channels
        return num_heads[level] if isinstance(num_heads, (list, tuple)) else num_heads

    levels = len(channel_mult)
    input_blocks: List[List[Layer]] = [[("conv", 0)]]
    ds = 1
    for level in range(levels):
        for _ in range(num_res_blocks):
            layers = [("res", 0)]
            if ds in attention_resolutions:
                layers.append(("attn", heads(level)))
            input_blocks.append(layers)
        if level != levels - 1:
            input_blocks.append([("down", 0)])
            ds *= 2
    middle = [("res", 0), ("attn", heads(levels - 1)), ("res", 0)]
    output_blocks: List[List[Layer]] = []
    for level in reversed(range(levels)):
        for i in range(num_res_blocks + 1):
            layers = [("res", 0)]
            if ds in attention_resolutions:
                layers.append(("attn", heads(level)))
            if level and i == num_res_blocks:
                layers.append(("up", 0))
                ds //= 2
            output_blocks.append(layers)
    return input_blocks, middle, output_blocks


def _sequential(p: Params, name: str, layers: List[Layer], h, emb, context, groups: int, use_linear: bool,
                up_size=None):
    """One TimestepEmbedSequential."""
    for i, (kind, heads) in enumerate(layers):
        sub = f"{name}.{i}"
        if kind == "conv":
            h = conv(p, sub, h)
        elif kind == "res":
            h = res_block(p, sub, h, emb, groups)
        elif kind == "attn":
            h = spatial_transformer(p, sub, h, context, heads, groups, use_linear)
        elif kind == "down":
            h = conv(p, f"{sub}.op", h, stride=2, padding=1)
        else:
            if up_size is None:
                h = F.interpolate(h, scale_factor=2, mode="nearest")
            else:
                h = F.interpolate(h, size=up_size, mode="nearest")
            h = conv(p, f"{sub}.conv", h)
    return h


def _time_embed(p: Params, timesteps, model_channels: int, n: int, device):
    t = torch.as_tensor(timesteps, device=device).reshape(-1).expand(n)
    t_emb = timestep_embedding(t, model_channels)
    return linear(p, "time_embed.2", F.silu(linear(p, "time_embed.0", t_emb)))


def unet(state: Union[str, Tensors, Params], x, timesteps, context, *, model_channels: int, channel_mult: Sequence[int],
         num_res_blocks: int, attention_resolutions: Sequence[int], context_dim: int,
         num_heads: Union[int, Sequence[int]] = -1, num_head_channels: int = -1,
         use_linear_in_transformer: bool = False, norm_groups: int = 32, control: Optional[Sequence] = None,
         prefix: str = "model.diffusion_model.") -> torch.Tensor:
    """openaimodel.UNetModel.forward (ControlledUnetModel's when `control` holds a ControlNet's outputs: one residual
    per input block, then the middle block's) in fp64 on x's device.  `timesteps` is one value or one per sample."""
    p = _params(state, prefix, x.device)
    x, context = x.double(), context.double()
    assert context.shape[-1] == context_dim, (context.shape, context_dim)
    input_blocks, middle, output_blocks = unet_layout(model_channels, channel_mult, num_res_blocks,
                                                      attention_resolutions, num_heads, num_head_channels)
    run = dict(groups=norm_groups, use_linear=use_linear_in_transformer)
    emb = _time_embed(p, timesteps, model_channels, x.shape[0], x.device)
    control = None if control is None else [c.double() for c in control]
    hs = []
    h = x
    for b, layers in enumerate(input_blocks):
        h = _sequential(p, f"input_blocks.{b}", layers, h, emb, context, **run)
        hs.append(h)
    h = _sequential(p, "middle_block", middle, h, emb, context, **run)
    if control is not None:
        assert len(control) == len(input_blocks) + 1
        h = h + control.pop()
    # diffusers' rule, not LDM's: when a latent side is not a multiple of 2 ** (number of upsamplers), upsample to the
    # size of the skip the next output block concatenates (diffusers' `upsample_size`) instead of doubling
    factor = 2 ** sum(kind == "up" for layers in output_blocks for kind, _ in layers)
    ragged = any(s % factor for s in x.shape[-2:])
    for b, layers in enumerate(output_blocks):
        skip = hs.pop()
        if control is not None:
            skip = skip + control.pop()
        h = torch.cat([h, skip], dim=1)
        up_size = hs[-1].shape[-2:] if ragged and layers[-1][0] == "up" else None
        h = _sequential(p, f"output_blocks.{b}", layers, h, emb, context, up_size=up_size, **run)
    out = conv(p, "out.2", F.silu(group_norm(p, "out.0", h, norm_groups, 1e-5)))
    p.check_all_read()
    return out


# ------------------------------------------------------------------------------------------------
# cldm.ControlNet
# ------------------------------------------------------------------------------------------------
def hint_block(p: Params, hint):
    """cldm's input_hint_block: a Sequential of convolutions at the even indices with a SiLU after each but the last.
    cldm writes it out for the widths (16, 32, 96, 256): conv_in, then per width step a 3x3 conv at the width and a
    stride-2 conv to the next one, then the zero conv to model_channels.  The widths are read from the weights here;
    the strides follow that pattern (every conv at an even position of the list but the first and the last)."""
    idx = sorted({int(k.split(".")[1]) for k in p.tensors if k.startswith("input_hint_block.")})
    assert idx == list(range(0, 2 * len(idx), 2)), idx
    h = hint.double()
    for pos, k in enumerate(idx):
        stride = 2 if pos % 2 == 0 and 0 < pos < len(idx) - 1 else 1
        h = conv(p, f"input_hint_block.{k}", h, stride=stride, padding=1)
        if pos < len(idx) - 1:
            h = F.silu(h)
    return h


def controlnet(state: Union[str, Tensors, Params], x, hint, timesteps, context, *, model_channels: int,
               channel_mult: Sequence[int], num_res_blocks: int, attention_resolutions: Sequence[int],
               context_dim: int, num_heads: Union[int, Sequence[int]] = -1, num_head_channels: int = -1,
               use_linear_in_transformer: bool = False, norm_groups: int = 32, scale: float = 1.0,
               prefix: str = "control_model.") -> List[torch.Tensor]:
    """cldm.ControlNet.forward times ControlLDM's control scale: one residual per input block (zero_convs.i), then
    the middle block's (middle_block_out), all multiplied by `scale`.  `hint` is [N, 3, 8h, 8w] for x [N, 4, h, w]."""
    p = _params(state, prefix, x.device)
    x, context = x.double(), context.double()
    assert context.shape[-1] == context_dim, (context.shape, context_dim)
    input_blocks, middle, _ = unet_layout(model_channels, channel_mult, num_res_blocks, attention_resolutions,
                                          num_heads, num_head_channels)
    run = dict(groups=norm_groups, use_linear=use_linear_in_transformer)
    emb = _time_embed(p, timesteps, model_channels, x.shape[0], x.device)
    guided_hint = hint_block(p, hint)
    outs = []
    h = x
    for b, layers in enumerate(input_blocks):
        h = _sequential(p, f"input_blocks.{b}", layers, h, emb, context, **run)
        if guided_hint is not None:
            h = h + guided_hint
            guided_hint = None
        outs.append(conv(p, f"zero_convs.{b}.0", h))
    h = _sequential(p, "middle_block", middle, h, emb, context, **run)
    outs.append(conv(p, "middle_block_out.0", h))
    p.check_all_read()
    return [o * scale for o in outs]


# ------------------------------------------------------------------------------------------------
# diffusionmodules.model.Encoder / Decoder, AutoencoderKL
# ------------------------------------------------------------------------------------------------
def vae_res_block(p: Params, name: str, x, out_channels: int, groups: int):
    """model.ResnetBlock without a time embedding; `Normalize` is GroupNorm with eps 1e-6; nin_shortcut (1x1) when
    the width changes."""
    h = conv(p, f"{name}.conv1", F.silu(group_norm(p, f"{name}.norm1", x, groups, 1e-6)))
    h = conv(p, f"{name}.conv2", F.silu(group_norm(p, f"{name}.norm2", h, groups, 1e-6)))
    if x.shape[1] != out_channels:
        x = conv(p, f"{name}.nin_shortcut", x)
    return x + h


def attn_block(p: Params, name: str, x, groups: int):
    """model.AttnBlock: single-head attention over the pixels, q, k, v and proj_out as 1x1 convolutions."""
    h_ = group_norm(p, f"{name}.norm", x, groups, 1e-6)
    q, k, v = (conv(p, f"{name}.{n}", h_) for n in ("q", "k", "v"))
    b, c, h, w = q.shape
    q = q.reshape(b, c, h * w).permute(0, 2, 1)                           # b, hw, c
    k = k.reshape(b, c, h * w)                                            # b, c, hw
    w_ = torch.softmax(torch.bmm(q, k) * int(c) ** -0.5, dim=2)           # b, hw (queries), hw (keys)
    v = v.reshape(b, c, h * w)
    h_ = torch.bmm(v, w_.permute(0, 2, 1)).reshape(b, c, h, w)
    return x + conv(p, f"{name}.proj_out", h_)


def _vae_mid(p: Params, name: str, h, groups: int):
    c = h.shape[1]
    h = vae_res_block(p, f"{name}.block_1", h, c, groups)
    h = attn_block(p, f"{name}.attn_1", h, groups)
    return vae_res_block(p, f"{name}.block_2", h, c, groups)


def vae_encode(state: Union[str, Tensors, Params], x, *, ch: int, ch_mult: Sequence[int], num_res_blocks: int,
               z_channels: int, norm_groups: int = 32, prefix: str = "first_stage_model.") -> Tuple[torch.Tensor, torch.Tensor]:
    """(mean, logvar) of AutoencoderKL.encode's DiagonalGaussianDistribution for x [N, 3, H, W] in [-1, 1]: Encoder
    (double_z) then quant_conv, log-variance clamped to [-30, 20]."""
    p = _params(state, prefix, x.device)
    hs = [conv(p, "encoder.conv_in", x.double())]
    for level in range(len(ch_mult)):
        for i in range(num_res_blocks):
            hs.append(vae_res_block(p, f"encoder.down.{level}.block.{i}", hs[-1], ch * ch_mult[level], norm_groups))
        if level != len(ch_mult) - 1:
            # model.Downsample(with_conv=True): no asymmetric padding in torch conv, so pad (0, 1, 0, 1) by hand
            hs.append(conv(p, f"encoder.down.{level}.downsample.conv", F.pad(hs[-1], (0, 1, 0, 1), mode="constant",
                                                                             value=0), stride=2, padding=0))
    h = _vae_mid(p, "encoder.mid", hs[-1], norm_groups)
    h = conv(p, "encoder.conv_out", F.silu(group_norm(p, "encoder.norm_out", h, norm_groups, 1e-6)))
    assert h.shape[1] == 2 * z_channels
    moments = conv(p, "quant_conv", h)
    mean, logvar = torch.chunk(moments, 2, dim=1)
    return mean, torch.clamp(logvar, -30.0, 20.0)


def vae_decode(state: Union[str, Tensors, Params], z, *, ch: int, ch_mult: Sequence[int], num_res_blocks: int,
               z_channels: int, norm_groups: int = 32, prefix: str = "first_stage_model.") -> torch.Tensor:
    """AutoencoderKL.decode: post_quant_conv, then the Decoder: conv_in, mid, the levels from the lowest resolution
    (`up[n - 1]`) to the highest (`up[0]`), num_res_blocks + 1 ResnetBlocks each and an Upsample (nearest doubling,
    conv) after every level but `up[0]`, then norm_out, SiLU, conv_out."""
    p = _params(state, prefix, z.device)
    assert z.shape[1] == z_channels
    h = conv(p, "decoder.conv_in", conv(p, "post_quant_conv", z.double()))
    h = _vae_mid(p, "decoder.mid", h, norm_groups)
    for level in reversed(range(len(ch_mult))):
        for i in range(num_res_blocks + 1):
            h = vae_res_block(p, f"decoder.up.{level}.block.{i}", h, ch * ch_mult[level], norm_groups)
        if level != 0:
            h = conv(p, f"decoder.up.{level}.upsample.conv", F.interpolate(h, scale_factor=2.0, mode="nearest"))
    out = conv(p, "decoder.conv_out", F.silu(group_norm(p, "decoder.norm_out", h, norm_groups, 1e-6)))
    return out


# ------------------------------------------------------------------------------------------------
# the reference's pixel and scale chain around the VAE
# ------------------------------------------------------------------------------------------------
def encode_frames(state: Union[str, Tensors], frames_u8: torch.Tensor, **vae_config) -> torch.Tensor:
    """uint8 RGB frames [N, H, W, 3] -> scaled latents, as the reference encodes its frames (preprocess.py:174-182,
    193-195; run_tokenflow_pnp.py:145-153, 176-181): `T.ToTensor()` (channels first, the fp32 quotient x / 255),
    `2 * x - 1`, the posterior mean (deterministic=True) times 0.18215."""
    x = (frames_u8.permute(0, 3, 1, 2).float() / 255).double()
    mean, _ = vae_encode(state, 2 * x - 1, **vae_config)
    return mean * SCALE_FACTOR


def decode_frames(state: Union[str, Tensors], latents: torch.Tensor, **vae_config) -> torch.Tensor:
    """Scaled latents -> uint8 RGB frames [N, 8h, 8w, 3], as the reference decodes and saves them
    (preprocess.py:163-172; run_tokenflow_pnp.py:156-163; util.py:95): latents / 0.18215 decoded,
    `(x / 2 + 0.5).clamp(0, 1)`, times 255, truncated to uint8."""
    return frames_of(vae_decode(state, latents.double() / SCALE_FACTOR, **vae_config))


def frames_of(x: torch.Tensor) -> torch.Tensor:
    """Decoder output [N, 3, H, W] -> uint8 [N, H, W, 3]: `(x / 2 + 0.5).clamp(0, 1)`, times 255, truncated."""
    return ((x / 2 + 0.5).clamp(0, 1) * 255).to(torch.uint8).permute(0, 2, 3, 1)


# ------------------------------------------------------------------------------------------------
# test weights
# ------------------------------------------------------------------------------------------------
@torch.no_grad()
def perturb_constant_parameters(net: torch.nn.Module, seed: int = 0, spread: float = 0.2) -> torch.nn.Module:
    """Give every parameter tensor that holds one value (norm scales of 1, norm and zero-initialised biases, zero
    convolutions) random values around it (+ spread * N(0, 1) * max(|value|, 1)), so that a slip which only matters
    for a non-trivial scale or bias shows.  Randomly initialised tensors are left as they are."""
    g = torch.Generator().manual_seed(seed)
    for param in net.parameters():
        flat = param.detach().reshape(-1)
        if flat.numel() and bool((flat == flat[0]).all()):
            noise = torch.randn(param.shape, generator=g).to(param.device, param.dtype)
            param.add_(noise * spread * max(abs(float(flat[0])), 1.0))
    return net
