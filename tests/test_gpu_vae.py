"""The VAE stage on the H100: the pixel conversions, the restated AutoencoderKL on real activations, and frames ->
edited frames in one process.  (tf_group_norm_nhwc at the VAE's 4-channels-per-group shapes is tested with the other
GroupNorm shapes in tests/test_gpu_body_kernels.py.)

* tf_frames_to_nhwc over all 256 byte values and tf_nhwc_to_frames over all 65 536 fp16 bit patterns, bit-equal to
  the torch expressions they replace; NaN -> 0 is checked on its own.  Sentinel-filled outputs with guard bands.
* The whole VAE (SD configuration, random weights, fp16 channels_last) on 512^2 frames: every 4-channel-group site
  passes `check_group_norm` on its own activations; the native encode and decode are as close to an fp32 run of the
  same weights as the ATen-GroupNorm run (rel-L2 at most 1.05x).
* End to end at 256^2: uint8 frames -> encode -> inversion -> saved_latents -> ddim_eps -> add_noise -> edit ->
  decode equals the same chain through the latents files and torch.load.
"""
import copy
import glob
import os

import pytest
import torch

from oracle.kernel_checks import check_group_norm
from tokenflow_b200 import ops as tf_ops
from tokenflow_b200 import sd_unet
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.editor import TokenFlowEditor
from tokenflow_b200.preprocess import LatentInverter, ddim_eps, decode_latents, encode_imgs
from tokenflow_b200.scheduler import DDIMScheduler
from tokenflow_b200.vae import build_vae

pytestmark = pytest.mark.gpu
GUARD = 256


@pytest.fixture(scope="module")
def ops():
    tfu._install_ops_for_testing(None)
    return tf_ops.CudaOps()


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------
# pixel conversions
# ------------------------------------------------------------------------------------------------
def _every_byte(n, h, w, seed):
    vals = torch.arange(n * h * w * 3) % 256
    perm = torch.randperm(vals.numel(), generator=torch.Generator().manual_seed(seed))
    return vals[perm].to(torch.uint8).view(n, h, w, 3)


def _encoder_input_reference(frames):
    """The reference's host conversion (`T.ToTensor()`, `.to(torch.float16)`) then `2 * imgs - 1` on the device."""
    import torchvision.transforms as T
    imgs = torch.stack([T.ToTensor()(f.numpy()) for f in frames]).to(torch.float16).cuda()
    return 2 * imgs - 1


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 5, 7), (2, 17, 31), (3, 256, 256)])
def test_frames_to_nhwc_every_byte_value(ops, shape):
    frames = _every_byte(*shape, seed=sum(shape))
    assert frames.unique().numel() == min(256, frames.numel())
    want = _encoder_input_reference(frames)
    n, h, w = shape
    numel = n * h * w * 3
    dev = frames.cuda()
    buf = torch.full((numel + 2 * GUARD,), float("nan"), dtype=torch.float16, device="cuda")
    out = buf[GUARD:GUARD + numel]
    assert ops.lib.tf_frames_to_nhwc(dev.data_ptr(), n * h * w, out.data_ptr(), _stream()) == 0
    torch.cuda.synchronize()
    assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + numel:]).all(), "write outside the output"
    assert not torch.isnan(out).any(), "output element left unwritten"
    got = out.view(n, h, w, 3).permute(0, 3, 1, 2)
    assert torch.equal(got.contiguous().view(torch.int16), want.contiguous().view(torch.int16))
    via_ops = ops.frames_to_nhwc(dev)
    assert via_ops.is_contiguous(memory_format=torch.channels_last) and torch.equal(via_ops, got)


def _frames_reference(x):
    return ((x / 2 + 0.5).clamp(0, 1) * 255).to(torch.uint8)


@pytest.mark.parametrize("sentinel", [0xAB, 0x54])
def test_nhwc_to_frames_every_fp16_bit_pattern(ops, sentinel):
    """All 65 536 fp16 values (+-0, subnormals, +-Inf, NaN) and two zeros of padding to a whole pixel: bit-equal to the
    eager fp16 expression; a NaN gives 0.  Two sentinel fills: an element left unwritten cannot match both."""
    bits = torch.cat([torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16), torch.zeros(2, dtype=torch.int16)])
    flat = bits.view(torch.float16).cuda()
    n_px = flat.numel() // 3
    x = flat.view(1, 1, n_px, 3).permute(0, 3, 1, 2)                 # channels_last [1, 3, 1, n_px]
    buf = torch.full((3 * n_px + 2 * GUARD,), sentinel, dtype=torch.uint8, device="cuda")
    out = buf[GUARD:GUARD + 3 * n_px]
    assert ops.lib.tf_nhwc_to_frames(flat.data_ptr(), n_px, out.data_ptr(), _stream()) == 0
    torch.cuda.synchronize()
    assert (buf[:GUARD] == sentinel).all() and (buf[GUARD + 3 * n_px:] == sentinel).all(), "write outside the output"
    want = _frames_reference(x).permute(0, 2, 3, 1).reshape(-1)
    nan = torch.isnan(flat)
    assert int(nan.sum()) == 2046
    assert torch.equal(out[~nan], want[~nan])
    assert (out[nan] == 0).all()
    print(f"torch's uint8 of NaN here: {sorted(set(want[nan].tolist()))}")
    inf = torch.isinf(flat)
    assert sorted(out[inf].tolist()) == [0, 255]
    assert torch.equal(ops.nhwc_to_frames(x), out.view(1, 1, n_px, 3))


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 5, 7), (3, 256, 256)])
def test_nhwc_to_frames_tails_and_layouts(ops, shape):
    n, h, w = shape
    g = torch.Generator(device="cuda").manual_seed(h * w)
    x = (torch.randn(n, 3, h, w, device="cuda", generator=g) * 1.2).half()
    got = ops.nhwc_to_frames(x)                                        # NCHW input: converted to channels_last first
    want = _frames_reference(x).permute(0, 2, 3, 1)
    assert got.shape == (n, h, w, 3) and torch.equal(got, want)
    assert torch.equal(ops.nhwc_to_frames(x.contiguous(memory_format=torch.channels_last)), want)


# ------------------------------------------------------------------------------------------------
# the whole VAE
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def vae():
    return build_vae("sd", seed=1, device="cuda", dtype=torch.float16,
                     init_on_device=True).to(memory_format=torch.channels_last)


class _G4Recorder:
    """Records the `group_norm_nhwc` calls at 4 channels per group."""

    def __init__(self, inner):
        self.inner, self.calls = inner, []

    def __getattr__(self, name):
        return getattr(self.inner, name)

    def group_norm_nhwc(self, x, norm, bias=None, silu=False):
        out = self.inner.group_norm_nhwc(x, norm, bias, silu)
        if x.shape[1] == 4 * norm.num_groups:
            self.calls.append((x, norm, silu, out))
        return out


def _smooth_frames(n, side, seed):
    """Frames with image-like structure: low-frequency colour fields plus a little noise."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(n, 3, side // 64, side // 64, generator=g)
    img = torch.nn.functional.interpolate(low, size=(side, side), mode="bicubic", align_corners=False)
    img = (img + 0.05 * torch.randn(n, 3, side, side, generator=g)).clamp(0, 1)
    return (img * 255).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


@torch.no_grad()
def test_every_g4_site_on_real_activations(ops, vae, monkeypatch):
    rec = _G4Recorder(ops)
    monkeypatch.setattr(tf_ops, "_BODY_OPS", rec)
    lat = encode_imgs(vae, _smooth_frames(2, 512, seed=1), batch_size=2)
    n_enc = len(rec.calls)
    vae.decode(lat / 0.18215)
    assert n_enc == 5 and len(rec.calls) - n_enc == 6, (n_enc, len(rec.calls))
    for i, (x, norm, silu, out) in enumerate(rec.calls):
        stage = "encode" if i < n_enc else "decode"
        check_group_norm(out, x, norm, None, silu, f"{stage} site {i} {tuple(x.shape)} silu={silu}",
                         exempt_aten_misrounded=True)


@torch.no_grad()
def test_native_vae_is_as_close_to_fp32_as_aten(ops, vae, monkeypatch):
    frames = _smooth_frames(4, 512, seed=2)
    x = ops.frames_to_nhwc(frames.cuda())
    z = torch.randn(4, 4, 64, 64, generator=torch.Generator().manual_seed(3)).half().cuda()
    native_enc, native_dec = vae.encode(x).latent_dist.mean, vae.decode(z).sample
    native_frames = decode_latents(vae, z * 0.18215, batch_size=2)
    with monkeypatch.context() as m:
        m.setattr(tf_ops, "_BODY_OPS", None)                         # norm_act takes ATen's GroupNorm
        aten_enc, aten_dec = vae.encode(x).latent_dist.mean, vae.decode(z).sample
        aten_frames = decode_latents(vae, z * 0.18215, batch_size=2)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)      # a true fp32 reference
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    vae32 = copy.deepcopy(vae).float()
    ref_enc, ref_dec = vae32.encode(x.float()).latent_dist.mean, vae32.decode(z.float()).sample
    del vae32
    for name, ours, theirs, ref in (("encode", native_enc, aten_enc, ref_enc), ("decode", native_dec, aten_dec, ref_dec)):
        r_n, r_a = _rel(ours, ref), _rel(theirs, ref)
        print(f"{name}: rel-L2 to fp32 native {r_n:.4g}, ATen GroupNorm {r_a:.4g}")
        assert torch.isfinite(ours).all() and r_n <= 1.05 * r_a, (name, r_n, r_a)
    diff = (native_frames.int() - aten_frames.int()).abs()
    print(f"uint8 frames, native vs ATen GroupNorm: max |diff| {diff.max().item()}, mean {diff.float().mean().item():.4g}")


@torch.no_grad()
def test_frames_to_edited_frames_in_memory_equals_the_disk_chain(ops, vae, tmp_path):
    from tokenflow_b200.util import save_video
    steps, n = 4, 8
    unet_kw = dict(seed=1, device="cuda", dtype=torch.float16)
    unet = sd_unet.build_unet("tiny", **unet_kw).to(memory_format=torch.channels_last)
    ctx = unet.config.cross_attention_dim
    g = torch.Generator().manual_seed(5)
    pnp = torch.randn(1, 7, ctx, generator=g).half().cuda()
    text = torch.randn(2, 7, ctx, generator=g).half().cuda()
    frames = _smooth_frames(n, 256, seed=4)
    lat_dir = str(tmp_path / "latents")
    cfg = {"n_frames": n, "batch_size": 4, "n_timesteps": steps, "guidance_scale": 7.5, "mode": "pnp",
           "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "fused_pass": True, "cuda_graph": True, "keyframe_seed": 1,
           "latents_path": lat_dir}

    def edit(latents, eps_of, source):
        ed = TokenFlowEditor(sd_unet.build_unet("tiny", **unet_kw).to(memory_format=torch.channels_last),
                             DDIMScheduler(), tfu, cfg, text, pnp, source_latents=source)
        eps = eps_of(ed.scheduler)
        x = ed.scheduler.add_noise(latents, eps, ed.scheduler.timesteps[0])
        ed.init_method()
        out = ed.sample_loop(x)
        assert torch.isfinite(out).all()
        return decode_latents(vae, out)

    # in memory
    latents = encode_imgs(vae, frames)
    inv = LatentInverter(unet, DDIMScheduler(), steps)
    inv.ddim_inversion(pnp, latents, str(tmp_path), batch_size=4)
    saved = inv.saved_latents()
    mem = edit(latents, lambda sch: ddim_eps(latents, saved, sch), saved.__getitem__)

    # through the files, as the reference's edit driver reads them (run_tokenflow_pnp.py:166-193)
    torch.save(latents, str(tmp_path / "clean.pt"))
    clean = torch.load(str(tmp_path / "clean.pt")).to(torch.float16).cuda()

    def eps_from_files(sch):
        noisest = max(int(p.split("_")[-1].split(".")[0]) for p in glob.glob(os.path.join(lat_dir, "noisy_latents_*.pt")))
        noisy = torch.load(os.path.join(lat_dir, f"noisy_latents_{noisest}.pt"))[range(n)].cuda()
        alpha_prod_T = sch.alphas_cumprod[noisest]
        mu_T, sigma_T = alpha_prod_T ** 0.5, (1 - alpha_prod_T) ** 0.5
        return ((noisy - mu_T * clean) / sigma_T).to(torch.float16)

    disk = edit(clean, eps_from_files, None)
    assert mem.dtype == torch.uint8 and mem.shape == (n, 256, 256, 3)
    assert torch.equal(mem, disk)
    save_video(mem, str(tmp_path / "edit.mp4"))
    assert os.path.getsize(tmp_path / "edit.mp4") > 0
