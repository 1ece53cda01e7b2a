"""CPU tier: the UNet, VAE and ControlNet against `oracle/ldm_forward.py`, an independent fp64 statement of the same
functions in CompVis LDM's and cldm's formulation, fed the LDM-layout state dict `oracle/ldm_layout.py` writes.

* Every output within max |diff| <= 1e-10 * max(1, |ref|), the models in fp64, loaded two ways: as built, and rebuilt
  from the LDM dict by `checkpoint.unet_state` / `vae_state` / `controlnet_state` + `assign_model` (the converters).
* UNets: the tiny kind and scaled-down SD1.5-like (1x1-conv projections, `attention_head_dim` = 8 heads) and
  SD2.1-like (linear projections, 64-channel heads, given both ways diffusers configs give them) configurations;
  16 x 16 and 13 x 21 latents; t = 1, 500, 999 and a batch of distinct timesteps.  VAEs: the tiny and the SD kinds,
  encoder and decoder with the reference's pixel chain, at 64 x 64 and 104 x 168 pixels.  ControlNets: the tiny and an
  SD1.5-like Canny configuration at conditioning scales 1 and 0.5, their residuals fed through the UNet.
* Every parameter is random and non-zero (norm scales and biases, zero convolutions included).
* Planted slips: each of the mistakes listed in `MUTATIONS`, monkeypatched into the product, is rejected.
* `oracle/ldm_forward.py` imports nothing from `tokenflow_b200`.
"""
import ast
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import ldm_forward as ldm
from oracle import ldm_layout
from tokenflow_b200 import checkpoint, sd_unet
from tokenflow_b200 import controlnet as cn
from tokenflow_b200 import synthetic_checkpoint as fx
from tokenflow_b200 import vae as vae_mod

BOUND = 1e-10                  # max |diff| / max(1, |ref|)
REJECT = 1e-6                  # a planted slip must move some output by more than this

_SD15_LIKE = {**fx.SD15_UNET, "block_out_channels": [64, 128, 128, 128], "cross_attention_dim": 48,
              "attention_head_dim": 8}
_SD21_LIKE = {**fx.SD21_UNET, "block_out_channels": [64, 128, 192, 192], "cross_attention_dim": 64,
              "attention_head_dim": [1, 2, 3, 3]}
_LDM_COMMON = dict(num_res_blocks=2, attention_resolutions=(4, 2, 1))
_SD21_LDM = dict(model_channels=64, channel_mult=(1, 2, 3, 3), num_head_channels=64, context_dim=64,
                 use_linear_in_transformer=True, **_LDM_COMMON)

# kind -> (diffusers config, LDM UNetModel parameters)
UNETS = {
    "tiny": (fx.TINY_UNET, dict(model_channels=32, channel_mult=(1, 2, 4, 4), num_heads=(2, 2, 4, 4), context_dim=32,
                                norm_groups=8, **_LDM_COMMON)),
    "sd15_like": (_SD15_LIKE, dict(model_channels=64, channel_mult=(1, 2, 2, 2), num_heads=8, context_dim=48,
                                   **_LDM_COMMON)),
    # diffusers' naming quirk: without num_attention_heads, attention_head_dim holds the head counts
    "sd21_like_head_counts": (_SD21_LIKE, _SD21_LDM),
    "sd21_like_num_attention_heads": ({**_SD21_LIKE, "num_attention_heads": [1, 2, 3, 3], "attention_head_dim": 64},
                                      _SD21_LDM),
}
CONTROLNETS = {
    "tiny": (fx.TINY_CANNY, "tiny"),
    "sd15_like": ({**fx.SD15_CANNY, **{k: _SD15_LIKE[k] for k in ("block_out_channels", "cross_attention_dim")}},
                  "sd15_like"),
}
_FLAT_VAE = {**fx.TINY_VAE, "block_out_channels": [32, 32, 32, 32]}
# kind -> (diffusers config, LDM AutoencoderKL ddconfig)
VAES = {
    "tiny": (fx.TINY_VAE, dict(ch=32, ch_mult=(1, 2, 2, 2), num_res_blocks=1, z_channels=4, norm_groups=8)),
    "sd": (fx.SD_VAE, dict(ch=128, ch_mult=(1, 2, 4, 4), num_res_blocks=2, z_channels=4)),
    "flat": (_FLAT_VAE, dict(ch=32, ch_mult=(1, 1, 1, 1), num_res_blocks=1, z_channels=4, norm_groups=8)),
}
LATENTS = {"16x16": (16, 16), "13x21": (13, 21)}
TIMESTEPS = {"t1": [1], "t500": [500], "t999": [999], "t_batch": [999, 1, 500]}


def rel_err(got, ref):
    return ((got.double() - ref).abs() / ref.abs().clamp(min=1)).max().item()


def _built(build, seed):
    state = torch.random.get_rng_state()
    torch.manual_seed(seed)
    try:
        net = build()
    finally:
        torch.random.set_rng_state(state)
    return ldm.perturb_constant_parameters(net, seed).double().eval()


def unet_models(kind, load):
    """(product UNet in fp64, its LDM state dict)."""
    config, _ = UNETS[kind]
    net = _built(lambda: sd_unet.build_unet("tiny") if kind == "tiny" else
                 sd_unet.UNet2DConditionModel.from_config(config), seed=1)
    state = ldm_layout.ldm_unet(net)
    if load == "rebuilt":
        net = checkpoint.assign_model(sd_unet.UNet2DConditionModel.from_config, config,
                                      checkpoint.unet_state(state, config["layers_per_block"]), dtype=torch.float64)
    return net, state


def controlnet_models(kind, load):
    """(product ControlNet in fp64, its LDM state dict)."""
    config, _ = CONTROLNETS[kind]
    net = _built(lambda: cn.build_controlnet("tiny") if kind == "tiny" else cn.ControlNetModel.from_config(config),
                 seed=3)
    state = ldm_layout.ldm_controlnet(net)
    if load == "rebuilt":
        net = checkpoint.assign_model(cn.ControlNetModel.from_config, config,
                                      checkpoint.controlnet_state(state, config["layers_per_block"]),
                                      dtype=torch.float64)
    return net, state


def vae_models(kind, load):
    config, _ = VAES[kind]
    net = _built(lambda: vae_mod.AutoencoderKL.from_config(config), seed=2)
    state = ldm_layout.ldm_vae(net)
    if load == "rebuilt":
        net = checkpoint.assign_model(vae_mod.AutoencoderKL.from_config, config, checkpoint.vae_state(state),
                                      dtype=torch.float64)
    return net, state


def _unet_inputs(kind, latent, n, seed=0):
    g = torch.Generator().manual_seed(seed)
    ctx = UNETS[kind][1]["context_dim"]
    return (torch.randn(n, 4, *LATENTS[latent], generator=g, dtype=torch.float64),
            torch.randn(n, 7, ctx, generator=g, dtype=torch.float64))


@torch.no_grad()
def unet_error(kind, load="built", latent="16x16", t=(500,), net=None):
    """Max error of the UNet's output; `net` replaces the product UNet (the LDM dict is still the built one's)."""
    built, state = unet_models(kind, load)
    net = built if net is None else net
    timesteps = torch.tensor(t)
    x, ctx = _unet_inputs(kind, latent, n=max(len(t), 2))
    got = net(x, timesteps, encoder_hidden_states=ctx).sample
    ref = ldm.unet(state, x, timesteps, ctx, **UNETS[kind][1])
    assert got.shape == ref.shape == x.shape
    return rel_err(got, ref)


@torch.no_grad()
def controlnet_errors(kind, load="built", latent="16x16", scale=1.0, net=None):
    """(max error over the 13 residuals, error of the UNet output fed with them); `net` as in `unet_error`."""
    built, state = controlnet_models(kind, load)
    net = built if net is None else net
    unet, unet_state = unet_models(CONTROLNETS[kind][1], load)
    params = UNETS[CONTROLNETS[kind][1]][1]
    x, ctx = _unet_inputs(CONTROLNETS[kind][1], latent, n=2, seed=4)
    h, w = LATENTS[latent]
    cond = torch.rand(2, 3, 8 * h, 8 * w, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    t = torch.tensor([981, 41])
    down, mid = net(x, t, encoder_hidden_states=ctx, controlnet_cond=cond, conditioning_scale=scale)
    ref = ldm.controlnet(state, x, cond, t, ctx, scale=scale, **params)
    got = list(down) + [mid]
    assert len(got) == len(ref) == 13 and all(a.shape == b.shape for a, b in zip(got, ref))
    res_err = max(rel_err(a, b) for a, b in zip(got, ref))
    out = unet(x, t, encoder_hidden_states=ctx, down_block_additional_residuals=down,
               mid_block_additional_residual=mid).sample
    return res_err, rel_err(out, ldm.unet(unet_state, x, t, ctx, control=ref, **params))


def _frames(n, h, w, seed):
    return torch.randint(0, 256, (n, h, w, 3), generator=torch.Generator().manual_seed(seed), dtype=torch.uint8)


@torch.no_grad()
def vae_errors(kind, load="built", size=(64, 64)):
    """(error of the scaled latents from uint8 frames, error of the decoder output) against the reference's chain."""
    from tokenflow_b200.preprocess import encode_imgs
    net, state = vae_models(kind, load)
    cfg = VAES[kind][1]
    frames = _frames(2, *size, seed=6)
    enc = rel_err(encode_imgs(net, frames), ldm.encode_frames(state, frames, **cfg))
    z = torch.randn(2, 4, size[0] // 8, size[1] // 8, generator=torch.Generator().manual_seed(7), dtype=torch.float64)
    dec = rel_err(net.decode(z / vae_mod.SCALING_FACTOR).sample,
                  ldm.vae_decode(state, z / ldm.SCALE_FACTOR, **cfg))
    return enc, dec


# ------------------------------------------------------------------------------------------------
# the product against the restatement
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", sorted(TIMESTEPS))
@pytest.mark.parametrize("latent", sorted(LATENTS))
@pytest.mark.parametrize("load", ["built", "rebuilt"])
@pytest.mark.parametrize("kind", sorted(UNETS))
def test_unet_matches_ldm(kind, load, latent, t):
    err = unet_error(kind, load, latent, TIMESTEPS[t])
    assert err <= BOUND, f"{kind} {load} {latent} {t}: {err:.3g}"


@pytest.mark.parametrize("scale", [1.0, 0.5])
@pytest.mark.parametrize("latent", sorted(LATENTS))
@pytest.mark.parametrize("load", ["built", "rebuilt"])
@pytest.mark.parametrize("kind", sorted(CONTROLNETS))
def test_controlnet_and_unet_with_its_residuals_match_cldm(kind, load, latent, scale):
    res_err, out_err = controlnet_errors(kind, load, latent, scale)
    assert res_err <= BOUND and out_err <= BOUND, (res_err, out_err)


@pytest.mark.parametrize("size", [(64, 64), (104, 168)], ids=["64x64", "104x168"])
@pytest.mark.parametrize("load", ["built", "rebuilt"])
@pytest.mark.parametrize("kind", ["tiny", "sd"])
def test_vae_and_pixel_chain_match_ldm(kind, load, size):
    enc, dec = vae_errors(kind, load, size)
    assert enc <= BOUND and dec <= BOUND, (enc, dec)


@torch.no_grad()
def test_uint8_frames_match_the_reference_chain():
    """`decode_latents` against the restated decode chain, byte for byte (both clamps reached), and every tensor of
    the VAE's LDM dict read by the restated encoder and decoder."""
    from tokenflow_b200.preprocess import decode_latents
    net, state = vae_models("tiny", "rebuilt")
    cfg = VAES["tiny"][1]
    z = torch.randn(2, 4, 8, 8, generator=torch.Generator().manual_seed(8), dtype=torch.float64)
    got, want = decode_latents(net, z), ldm.decode_frames(state, z, **cfg)
    assert got.dtype == want.dtype == torch.uint8 and torch.equal(got, want)
    assert 0 < (want == 0).float().mean() < 0.5 and 0 < (want == 255).float().mean() < 0.5
    p = ldm.Params(state, "first_stage_model.", "cpu")
    ldm.vae_encode(p, torch.zeros(1, 3, 16, 16, dtype=torch.float64), **cfg)
    with pytest.raises(KeyError, match="not used"):
        p.check_all_read()
    ldm.vae_decode(p, torch.zeros(1, 4, 2, 2, dtype=torch.float64), **cfg)
    p.check_all_read()


def test_restatement_reads_a_safetensors_file_and_every_tensor(tmp_path):
    net, state = unet_models("tiny", "built")
    path = str(tmp_path / "unet.safetensors")
    ldm_layout.save(path, state)
    x, ctx = _unet_inputs("tiny", "13x21", n=2)
    with torch.no_grad():
        got = net(x, torch.tensor([7]), encoder_hidden_states=ctx).sample
    assert rel_err(got, ldm.unet(path, x, 7, ctx, **UNETS["tiny"][1])) <= BOUND
    extra = {**state, "model.diffusion_model.input_blocks.1.0.unused.weight": torch.zeros(1)}
    with pytest.raises(KeyError, match="not used"):
        ldm.unet(extra, x, 7, ctx, **UNETS["tiny"][1])


def test_every_parameter_is_random_and_nonzero():
    for net, _ in (unet_models("sd15_like", "built"), controlnet_models("tiny", "built"), vae_models("tiny", "built")):
        for name, p in net.named_parameters():
            flat = p.detach().reshape(-1)
            assert (flat != 0).all() and (flat.numel() == 1 or (flat != flat[0]).any()), name


def test_restatement_imports_nothing_from_the_package():
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "ldm_forward.py")
    with open(path) as f:
        tree = ast.parse(f.read())
    imported = set()
    for node in ast.walk(tree):
        if isinstance(node, ast.Import):
            imported.update(a.name for a in node.names)
        elif isinstance(node, ast.ImportFrom):
            imported.add("." * node.level + (node.module or ""))
    assert imported, "no imports parsed"
    assert not any(m.split(".")[0] in ("tokenflow_b200", "") or "tokenflow" in m for m in imported), imported
    assert imported <= {"__future__", "math", "typing", "torch", "torch.nn.functional", "safetensors.torch"}, imported


# ------------------------------------------------------------------------------------------------
# planted slips
# ------------------------------------------------------------------------------------------------
_SINUSOID = sd_unet.sinusoidal_timestep_embedding


def _sin_cos(timesteps, dim):
    emb = _SINUSOID(timesteps, dim)
    return torch.cat([emb[:, dim // 2:], emb[:, :dim // 2]], dim=-1)


def _skip_first(self, x, skips, temb, ctx=None, upsample_size=None):
    attentions = getattr(self, "attentions", [None] * len(self.resnets))
    for r, a in zip(self.resnets, attentions):
        x = r(torch.cat([skips.pop(), x], dim=1), temb)
        if a is not None:
            x = a(x, encoder_hidden_states=ctx)
    if self.upsamplers is not None:
        x = self.upsamplers[0](x, upsample_size)
    return x


def _bilinear(self, x, output_size=None):
    if output_size is None:
        return self.conv(F.interpolate(x, scale_factor=2.0, mode="bilinear"))
    return self.conv(F.interpolate(x, size=output_size, mode="bilinear"))


def _geglu_swapped(self, x):
    w_g, w_x = self.proj.weight.chunk(2, dim=0)
    b_g, b_x = self.proj.bias.chunk(2, dim=0)
    return F.linear(x, w_x, b_x) * F.gelu(F.linear(x, w_g, b_g))


def _tokens_from_nchw_memory(self, hidden_states, encoder_hidden_states=None):
    """The linear-projection branch flattening [b, c, h, w] straight to [b, h*w, c] (no channel permute), and back."""
    b, c, hh, ww = hidden_states.shape
    x = self.proj_in(sd_unet.norm_act(self.norm, hidden_states, silu=False).reshape(b, hh * ww, c))
    x = self.transformer_blocks[0](x, encoder_hidden_states=encoder_hidden_states)
    return self.proj_out(x).reshape(b, c, hh, ww) + hidden_states


def _no_time_silu(self, x):
    return self.linear_2(self.linear_1(x))


def _symmetric_pad(self, x):
    return self.conv(F.pad(x, (1, 1, 1, 1)))


def _levels_in_ldm_index_order(self, z):
    x = self.mid_block(self.conv_in(z))
    for blk in reversed(self.up_blocks):
        x = blk(x)
    return self.conv_out(sd_unet.norm_act(self.conv_norm_out, x))


def _modules(net, cls):
    return [m for m in net.modules() if isinstance(m, cls)]


def _unet_slip(kind, patch, latent="16x16"):
    def run(monkeypatch):
        net, _ = unet_models(kind, "built")
        patch(monkeypatch, net)
        return unet_error(kind, latent=latent, net=net)
    return run


def _instances(cls, attr, value_of):
    def patch(m, net):
        for mod in _modules(net, cls):
            m.setattr(mod, attr, value_of(mod))
    return patch


def _class(cls, attr, fn):
    return lambda m, net: m.setattr(cls, attr, fn)


def _swap_projections(m, net):
    for mod in _modules(net, sd_unet.Transformer2DModel):
        proj_in, proj_out = mod.proj_in, mod.proj_out
        m.setattr(mod, "proj_in", proj_out)
        m.setattr(mod, "proj_out", proj_in)


def _head_size(m, net):
    """attention_head_dim read as the size of a head: heads = width // attention_head_dim (then rebuilt)."""
    fields = sd_unet.encoder_fields

    def as_head_size(config, what):
        out = fields(config, what)
        out["num_heads"] = tuple(c // h for c, h in zip(out["block_out_channels"], out["num_heads"]))
        return out
    m.setattr(sd_unet, "encoder_fields", as_head_size)


def _vae_slip(kind, patch):
    def run(monkeypatch):
        patch(monkeypatch, None)
        return max(vae_errors(kind))
    return run


def _controlnet_slip(patch, scale=1.0):
    def run(monkeypatch):
        net, _ = controlnet_models("tiny", "built")
        patch(monkeypatch, net)
        return max(controlnet_errors("tiny", scale=scale, net=net))
    return run


def _hint_one_block_late(m, net):
    """The conditioning embedding added to the output of the first ResBlock + SpatialTransformer (cldm's input block
    1) instead of to conv_in's (input block 0)."""
    emb = net.controlnet_cond_embedding
    real = emb.forward
    stash = {}

    def embed(cond):
        stash["hint"] = real(cond)
        return torch.zeros_like(stash["hint"])

    def add_hint(module, args, out):
        return out + stash["hint"]

    m.setattr(emb, "forward", embed)
    net.down_blocks[0].attentions[0].register_forward_hook(add_hint)       # `net` is built for this test alone


def _scale_on_mid_only(m, net):
    forward = cn.ControlNetModel.forward

    def scaled(self, *args, conditioning_scale=1.0, **kw):
        down, mid = forward(self, *args, conditioning_scale=1.0, **kw)
        return down, mid * conditioning_scale
    m.setattr(cn.ControlNetModel, "forward", scaled)


def _rebuilt_slip(kind, patch):
    def run(monkeypatch):
        patch(monkeypatch, None)
        return unet_error(kind, load="rebuilt")
    return run


MUTATIONS = {
    "timestep_embedding_sin_cos_swapped": _unet_slip("sd15_like", _class(sd_unet, "sinusoidal_timestep_embedding",
                                                                         _sin_cos)),
    "skip_concatenated_before_hidden": _unet_slip("tiny", lambda m, net: (
        m.setattr(sd_unet.UpBlock2D, "forward", _skip_first),
        m.setattr(sd_unet.CrossAttnUpBlock2D, "forward", _skip_first))),
    "bilinear_upsampling": _unet_slip("tiny", _class(sd_unet.Upsample2D, "forward", _bilinear)),
    "bilinear_upsampling_to_skip_size": _unet_slip("tiny", _class(sd_unet.Upsample2D, "forward", _bilinear), "13x21"),
    "attention_scale_from_channels": _unet_slip("sd15_like", _instances(
        sd_unet.Attention, "scale", lambda a: a.to_q.weight.shape[0] ** -0.5)),
    "geglu_halves_swapped": _unet_slip("tiny", _class(sd_unet.GEGLU, "forward", _geglu_swapped)),
    "linear_projection_tokens_from_nchw_memory": _unet_slip("sd21_like_head_counts", _class(
        sd_unet.Transformer2DModel, "forward", _tokens_from_nchw_memory)),
    "linear_proj_in_and_proj_out_swapped": _unet_slip("sd21_like_head_counts", _swap_projections),
    "time_embedding_without_silu": _unet_slip("tiny", _class(sd_unet.TimestepEmbedding, "forward", _no_time_silu)),
    "resnet_time_projection_without_silu": _unet_slip("tiny", _instances(
        sd_unet.ResnetBlock2D, "nonlinearity", lambda r: torch.nn.Identity())),
    "attention_head_dim_as_head_size": _rebuilt_slip("sd15_like", _head_size),
    "vae_downsample_padded_symmetrically": _vae_slip("tiny", _class(vae_mod.Downsample2D, "forward", _symmetric_pad)),
    "vae_decoder_levels_not_reversed": _vae_slip("flat", _class(vae_mod.Decoder, "forward",
                                                                _levels_in_ldm_index_order)),
    "controlnet_hint_one_block_late": _controlnet_slip(_hint_one_block_late),
    "conditioning_scale_on_mid_residual_only": _controlnet_slip(_scale_on_mid_only, scale=0.5),
}


@pytest.mark.parametrize("name", sorted(MUTATIONS))
def test_planted_slip_is_rejected(name, monkeypatch):
    err = MUTATIONS[name](monkeypatch)
    assert err > REJECT, f"{name}: max error {err:.3g} is within the comparison's reach"
