"""CPU tier of the VAE stage: the restated AutoencoderKL has diffusers' state-dict surface, the stage functions follow the
reference's batching, scaling and fp16 arithmetic, and the new C-ABI entry points reject bad arguments on the host."""
import ctypes

import pytest
import torch

from tokenflow_b200 import ops as tf_ops
from tokenflow_b200.preprocess import ddim_eps, decode_latents, encode_imgs
from tokenflow_b200.scheduler import DDIMScheduler
from tokenflow_b200.vae import SCALING_FACTOR, AutoencoderKL, build_vae, sd_config, tiny_config


def _resnet_keys(prefix, cin, cout):
    keys = {f"{prefix}.norm1.weight": (cin,), f"{prefix}.norm1.bias": (cin,),
            f"{prefix}.conv1.weight": (cout, cin, 3, 3), f"{prefix}.conv1.bias": (cout,),
            f"{prefix}.norm2.weight": (cout,), f"{prefix}.norm2.bias": (cout,),
            f"{prefix}.conv2.weight": (cout, cout, 3, 3), f"{prefix}.conv2.bias": (cout,)}
    if cin != cout:
        keys.update({f"{prefix}.conv_shortcut.weight": (cout, cin, 1, 1), f"{prefix}.conv_shortcut.bias": (cout,)})
    return keys


def _mid_keys(prefix, c):
    keys = {**_resnet_keys(f"{prefix}.resnets.0", c, c), **_resnet_keys(f"{prefix}.resnets.1", c, c),
            f"{prefix}.attentions.0.group_norm.weight": (c,), f"{prefix}.attentions.0.group_norm.bias": (c,)}
    for name in ("to_q", "to_k", "to_v", "to_out.0"):
        keys.update({f"{prefix}.attentions.0.{name}.weight": (c, c), f"{prefix}.attentions.0.{name}.bias": (c,)})
    return keys


def diffusers_vae_keys(block_out_channels, layers_per_block, latent=4):
    """{name: shape} of diffusers' AutoencoderKL state dict, written out from its module tree."""
    ch = list(block_out_channels)
    keys = {"encoder.conv_in.weight": (ch[0], 3, 3, 3), "encoder.conv_in.bias": (ch[0],)}
    for i, c in enumerate(ch):
        cin = ch[max(i - 1, 0)]
        for j in range(layers_per_block):
            keys.update(_resnet_keys(f"encoder.down_blocks.{i}.resnets.{j}", cin if j == 0 else c, c))
        if i < len(ch) - 1:
            keys.update({f"encoder.down_blocks.{i}.downsamplers.0.conv.weight": (c, c, 3, 3),
                         f"encoder.down_blocks.{i}.downsamplers.0.conv.bias": (c,)})
    keys.update(_mid_keys("encoder.mid_block", ch[-1]))
    keys.update({"encoder.conv_norm_out.weight": (ch[-1],), "encoder.conv_norm_out.bias": (ch[-1],),
                 "encoder.conv_out.weight": (2 * latent, ch[-1], 3, 3), "encoder.conv_out.bias": (2 * latent,),
                 "quant_conv.weight": (2 * latent, 2 * latent, 1, 1), "quant_conv.bias": (2 * latent,),
                 "post_quant_conv.weight": (latent, latent, 1, 1), "post_quant_conv.bias": (latent,)})
    rch = ch[::-1]
    keys.update({"decoder.conv_in.weight": (rch[0], latent, 3, 3), "decoder.conv_in.bias": (rch[0],)})
    keys.update(_mid_keys("decoder.mid_block", rch[0]))
    for i, c in enumerate(rch):
        cin = rch[max(i - 1, 0)]
        for j in range(layers_per_block + 1):
            keys.update(_resnet_keys(f"decoder.up_blocks.{i}.resnets.{j}", cin if j == 0 else c, c))
        if i < len(rch) - 1:
            keys.update({f"decoder.up_blocks.{i}.upsamplers.0.conv.weight": (c, c, 3, 3),
                         f"decoder.up_blocks.{i}.upsamplers.0.conv.bias": (c,)})
    keys.update({"decoder.conv_norm_out.weight": (rch[-1],), "decoder.conv_norm_out.bias": (rch[-1],),
                 "decoder.conv_out.weight": (3, rch[-1], 3, 3), "decoder.conv_out.bias": (3,)})
    return keys


@pytest.mark.parametrize("kind", ["sd", "tiny"])
def test_state_dict_has_diffusers_names_and_shapes(kind):
    cfg = sd_config() if kind == "sd" else tiny_config()
    got = {k: tuple(v.shape) for k, v in AutoencoderKL(cfg).state_dict().items()}
    assert got == diffusers_vae_keys(cfg.block_out_channels, cfg.layers_per_block)
    if kind == "sd":
        assert sum(v.numel() for v in AutoencoderKL(cfg).parameters()) == 83_653_863    # SD's VAE


def test_state_dict_round_trips_strict():
    a, b = build_vae("tiny", seed=1), build_vae("tiny", seed=2)
    x = torch.rand(2, 3, 32, 32) * 2 - 1
    with torch.no_grad():
        assert not torch.equal(a.encode(x).latent_dist.mean, b.encode(x).latent_dist.mean)
        b.load_state_dict(a.state_dict(), strict=True)
        assert torch.equal(a.encode(x).latent_dist.mean, b.encode(x).latent_dist.mean)
        z = torch.randn(2, 4, 4, 4)
        assert torch.equal(a.decode(z).sample, b.decode(z).sample)


class _Spy(torch.nn.Module):
    """Records the batch sizes that reach encode / decode."""

    def __init__(self, vae):
        super().__init__()
        self.vae, self.calls = vae, []

    def encode(self, x):
        self.calls.append(("encode", x.shape[0]))
        return self.vae.encode(x)

    def decode(self, z):
        self.calls.append(("decode", z.shape[0]))
        return self.vae.decode(z)


def _frames(n, h, w, seed=0):
    return torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(seed))


@torch.no_grad()
def test_encode_imgs_follows_the_reference():
    """preprocess.py:174-182 on `torch.stack([T.ToTensor()(f) ...]).to(dtype)`: 2 * imgs - 1, batches, mean * 0.18215."""
    vae = build_vae("tiny", seed=3)
    frames = _frames(7, 32, 40)
    spy = _Spy(vae)
    got = encode_imgs(spy, frames, batch_size=3)
    assert spy.calls == [("encode", 3), ("encode", 3), ("encode", 1)]
    imgs = torch.stack([torch.from_numpy(f.numpy()).permute(2, 0, 1).float().div(255) for f in frames])
    imgs = 2 * imgs - 1
    want = torch.cat([vae.encode(imgs[i:i + 3]).latent_dist.mean * 0.18215 for i in range(0, 7, 3)])
    assert got.shape == (7, 4, 4, 5) and torch.equal(got, want)
    # deterministic=False: the posterior sample, reproducible from the generator
    s1 = encode_imgs(vae, frames, batch_size=3, deterministic=False, generator=torch.Generator().manual_seed(5))
    s2 = encode_imgs(vae, frames, batch_size=3, deterministic=False, generator=torch.Generator().manual_seed(5))
    assert torch.equal(s1, s2) and not torch.equal(s1, got)


@torch.no_grad()
def test_decode_latents_follows_the_reference():
    """preprocess.py:163-172 + util.save_video's uint8 conversion: latents / 0.18215, batches,
    ((img / 2 + 0.5).clamp(0, 1) * 255).to(uint8), as [N, H, W, 3]."""
    vae = build_vae("tiny", seed=4)
    z = torch.randn(5, 4, 4, 6, generator=torch.Generator().manual_seed(1)) * 2
    spy = _Spy(vae)
    got = decode_latents(spy, z, batch_size=2)
    assert spy.calls == [("decode", 2), ("decode", 2), ("decode", 1)]
    imgs = torch.cat([vae.decode(1 / 0.18215 * z[b:b + 2]).sample for b in range(0, 5, 2)])
    want = ((imgs / 2 + 0.5).clamp(0, 1) * 255).to(torch.uint8).permute(0, 2, 3, 1)
    assert got.dtype == torch.uint8 and got.shape == (5, 32, 48, 3) and torch.equal(got, want)
    assert SCALING_FACTOR == 0.18215


def _reference_add_noise(sch, original, noise, timesteps):
    """diffusers DDIMScheduler.add_noise."""
    alphas_cumprod = sch.alphas_cumprod.to(device=original.device, dtype=original.dtype)
    timesteps = timesteps.to(original.device)
    sqrt_alpha_prod = alphas_cumprod[timesteps] ** 0.5
    sqrt_alpha_prod = sqrt_alpha_prod.flatten()
    while len(sqrt_alpha_prod.shape) < len(original.shape):
        sqrt_alpha_prod = sqrt_alpha_prod.unsqueeze(-1)
    sqrt_one_minus_alpha_prod = (1 - alphas_cumprod[timesteps]) ** 0.5
    sqrt_one_minus_alpha_prod = sqrt_one_minus_alpha_prod.flatten()
    while len(sqrt_one_minus_alpha_prod.shape) < len(original.shape):
        sqrt_one_minus_alpha_prod = sqrt_one_minus_alpha_prod.unsqueeze(-1)
    return sqrt_alpha_prod * original + sqrt_one_minus_alpha_prod * noise


def test_ddim_eps_and_add_noise_equal_the_reference_expressions():
    g = torch.Generator().manual_seed(2)
    latents = (torch.randn(6, 4, 8, 8, generator=g) * 1.2).half()
    saved = {t: (torch.randn(6, 4, 8, 8, generator=g) * (1 + t / 1000)).half() for t in (1, 501, 999)}
    sch = DDIMScheduler()
    eps = ddim_eps(latents, saved, sch)
    # run_tokenflow_pnp.py:186-193: the largest saved timestep, 0-dim fp32 alphas
    noisest = 999
    alpha_prod_T = sch.alphas_cumprod[noisest]
    mu_T, sigma_T = alpha_prod_T ** 0.5, (1 - alpha_prod_T) ** 0.5
    want = ((saved[noisest] - mu_T * latents) / sigma_T).to(torch.float16)
    assert eps.dtype == torch.float16 and torch.equal(eps, want)
    sch.set_timesteps(50)
    got = sch.add_noise(latents, eps, sch.timesteps[0])
    assert got.dtype == torch.float16
    assert torch.equal(got, _reference_add_noise(sch, latents, eps, sch.timesteps[0]))


@pytest.fixture(scope="module")
def lib():
    from tokenflow_b200 import _build
    if not tf_ops.library_path().exists():
        _build.build()
    return tf_ops.load_library()


def test_group_norm_and_pixel_entry_points_reject_bad_arguments_without_a_device(lib):
    buf = (ctypes.c_uint8 * 4096)()
    p = (ctypes.addressof(buf) + 15) & ~15
    gn = lambda c, groups, ws=4096, x=p, out=p, n=2, hw=64, bias=None: lib.tf_group_norm_nhwc(
        x, bias, 0, p, p, n, hw, c, groups, 1e-6, 1, p, ws, out, None)
    assert gn(132, 33) == 1 and b"c % 8" in lib.tf_last_error()                  # C % 8 != 0
    assert gn(128, 64) == 3 and b"c / groups" in lib.tf_last_error()              # 2 channels per group
    assert lib.tf_group_norm_nhwc_workspace(2, 64, 128, 64) == -1
    assert gn(8192, 2048) == 3                                                      # C > 4096
    assert gn(128, 32, bias=p) == 3 and b"no bias" in lib.tf_last_error()         # no bias add at 4 per group
    assert lib.tf_group_norm_nhwc_workspace(2, 64, 128, 32) == 2 * 32 * 1 * 16      # 4 channels per group accepted
    need = lib.tf_group_norm_nhwc_workspace(2, 512 * 512, 128, 32)
    assert need == 2 * 32 * 1024 * 16                                               # [N, G, 64 KB chunks] x 16 B
    assert gn(128, 32, ws=need - 16, hw=512 * 512) == 1 and b"workspace" in lib.tf_last_error()
    assert gn(128, 32, x=p + 8) == 1 and b"misaligned" in lib.tf_last_error()
    assert gn(128, 32, out=p + 2) == 1 and b"misaligned" in lib.tf_last_error()
    assert gn(128, 32, n=0) == 0 and gn(128, 32, hw=0) == 0                       # empty: no-op
    for fn in (lib.tf_frames_to_nhwc, lib.tf_nhwc_to_frames):
        assert fn(p, -1, p, None) == 1
        assert fn(p, 0, None, None) == 0
        assert fn(p + 4, 16, p, None) == 1 and b"misaligned" in lib.tf_last_error()
        assert fn(p, 16, p + 8, None) == 1 and b"misaligned" in lib.tf_last_error()
        assert fn(None, 16, p, None) == 1


def test_norm_act_keeps_aten_off_the_native_shapes():
    """CPU, NCHW and fp32 runs of a 4-channel-group GroupNorm take the ATen sequence."""
    from tokenflow_b200.sd_unet import norm_act
    norm = torch.nn.GroupNorm(32, 128, eps=1e-6)
    x = torch.randn(2, 128, 8, 8)
    assert torch.equal(norm_act(norm, x), torch.nn.functional.silu(norm(x)))
    assert torch.equal(norm_act(norm, x, silu=False), norm(x))
    assert not tf_ops.CudaOps.group_norm_nhwc_supported(x, norm)
