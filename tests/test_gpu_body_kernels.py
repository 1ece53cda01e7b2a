"""The UNet body's native kernels: tf_group_norm_nhwc (channels_last GroupNorm + time-embedding add + SiLU) and
tf_geglu, against the eager ATen sequences they replace.

* GroupNorm: every SD1.5 (HW 4096/1024/256/64) and SD2.1 (HW 9216/2304/576/144) level x every body channel count
  (320 ... 2560, 10 to 80 channels per group, so 16-byte vectors straddle two groups at 10/30/60 per group), with and
  without the bias add and the SiLU, eps 1e-5 and 1e-6, N = 2, plus the top-level C2 batch (N = 135).  At least
  99.9 % of the elements are within 1 fp16 ulp of ATen (the bit-equal fraction is printed).  ATen stores the group
  mean and rstd in fp16, so where a statistic rounds to the neighbouring fp16 value the whole group moves: every
  element is within 1 ulp plus what a one-ulp change of the fp16 mean / rstd explains, and the error against an fp64
  evaluation is no worse than ATen's by more than the same amount.  Two launches are bit-identical.  Outputs land in NaN-filled buffers with guard bands: every element is written and
  nothing outside.
* GEGLU: bit-equal to `xh * F.gelu(g)` at the 16 transformer-block shapes of the SD1.5 UNet at C2.
* Argument validation needs no GPU (not marked `gpu`).
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from tokenflow_b200 import ops as tf_ops

SD15_HW = (4096, 1024, 256, 64)
SD21_HW = (9216, 2304, 576, 144)
CHANNELS = (320, 640, 960, 1280, 1920, 2560)
GUARD = 256


@pytest.fixture(scope="module")
def ops():
    return tf_ops.CudaOps()


def _ulp(v: torch.Tensor) -> torch.Tensor:
    """fp16 spacing at |v| (fp32 tensor of magnitudes): 2^(e - 11) for v = m * 2^e, m in [0.5, 1); 2^-24 below."""
    _, e = torch.frexp(v.abs())
    return torch.clamp(torch.ldexp(torch.ones_like(v), e - 11), min=2.0 ** -24)


def _inputs(n, hw, c, bias, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    side = int(round(hw ** 0.5))
    # a per-channel offset larger than the spread, so cancellation in the statistics would show
    x = (torch.randn(n, c, side, side, device="cuda", generator=g) * 1.5
         + 3.0 * torch.randn(1, c, 1, 1, device="cuda", generator=g)).half().contiguous(memory_format=torch.channels_last)
    norm = torch.nn.GroupNorm(32, c).cuda().half()
    with torch.no_grad():
        norm.weight.copy_(1 + 0.3 * torch.randn(c, device="cuda", generator=g))
        norm.bias.copy_(0.3 * torch.randn(c, device="cuda", generator=g))
    b = (torch.randn(n, c, device="cuda", generator=g) * 2).half() if bias else None
    return x, norm, b


def _aten(x, norm, bias, silu):
    if bias is not None:
        x = x + bias[:, :, None, None]
    y = F.group_norm(x, norm.num_groups, norm.weight, norm.bias, norm.eps)
    return F.silu(y) if silu else y


def _fp64(x, norm, bias, silu):
    if bias is not None:
        x = x + bias[:, :, None, None]                      # the fp16 add, as the eager path rounds it
    n, c = x.shape[:2]
    xd = x.double().reshape(n, norm.num_groups, -1)
    mean = xd.mean(-1, keepdim=True)
    var = ((xd - mean) ** 2).mean(-1, keepdim=True)
    y = ((xd - mean) / torch.sqrt(var + norm.eps)).reshape(x.shape)
    y = y * norm.weight.double()[None, :, None, None] + norm.bias.double()[None, :, None, None]
    return y * torch.sigmoid(y) if silu else y


def _guarded_call(ops, x, norm, bias, silu):
    """tf_group_norm_nhwc straight through the C ABI into a NaN-filled buffer with guard bands."""
    n, c, h, w = x.shape
    numel = x.numel()
    buf = torch.full((numel + 2 * GUARD,), float("nan"), dtype=torch.float16, device="cuda")
    out = buf[GUARD:GUARD + numel]
    ws = torch.empty(ops.lib.tf_group_norm_nhwc_workspace(n, h * w, c, norm.num_groups), dtype=torch.uint8,
                     device="cuda")
    st = ops.lib.tf_group_norm_nhwc(x.data_ptr(), bias.data_ptr() if bias is not None else None,
                                    c if bias is not None else 0, norm.weight.data_ptr(), norm.bias.data_ptr(), n, h * w,
                                    c, norm.num_groups, float(norm.eps), int(silu), ws.data_ptr(), ws.numel(),
                                    out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert st == 0, ops.lib.tf_last_error()
    torch.cuda.synchronize()
    assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + numel:]).all(), "write outside the output"
    assert not torch.isnan(out).any(), "output element left unwritten"
    # NHWC buffer -> [n, c, h, w] channels_last view
    return out.view(n, h, w, c).permute(0, 3, 1, 2)


def _stat_flip_bound(x, norm, bias, silu):
    """How far the output moves when ATen's fp16 mean or rstd (RowwiseMomentsCUDAKernel<Half> stores both in the input
    dtype) is one fp16 ulp away: a statistic computed slightly differently can land on the other side of an fp16
    rounding boundary, and then every output element of that group moves by up to
    |rstd * gamma| * ulp(mean) + |x - mean| * |gamma| * ulp(rstd); after SiLU, 1.1 (its largest slope) times that plus
    one ulp of the fp16 pre-activation."""
    if bias is not None:
        x = x + bias[:, :, None, None]
    n, c, h, w = x.shape
    G = norm.num_groups
    _, mean, rstd = torch.ops.aten.native_group_norm(x.contiguous(), norm.weight, norm.bias, n, c, h * w, G, norm.eps)
    mean = mean.float().view(n, G, 1).expand(n, G, c // G).reshape(n, c, 1, 1)
    rstd = rstd.float().view(n, G, 1).expand(n, G, c // G).reshape(n, c, 1, 1)
    gamma = norm.weight.float().abs()[None, :, None, None]
    bound = rstd * gamma * _ulp(mean) + (x.float() - mean).abs() * gamma * _ulp(rstd)
    if not silu:
        return bound
    # SiLU maps a one-ulp difference of its fp16 input y to up to 1.1 ulp(y), more than ulp(silu(y)) for y < 0
    y = F.group_norm(x, G, norm.weight, norm.bias, norm.eps).float()
    return 1.1 * (bound + _ulp(y))


def _check_against_aten(ops, x, norm, bias, silu, tag):
    got = _guarded_call(ops, x, norm, bias, silu)
    want = _aten(x, norm, bias, silu)
    g32, w32 = got.float(), want.float()
    ulp = _ulp(torch.maximum(g32.abs(), w32.abs()))
    diff = (g32 - w32).abs()
    bit_equal = (got == want).float().mean().item()
    within = (diff <= ulp).float().mean().item()
    print(f"{tag}: bit-equal {bit_equal:.5f}, within 1 ulp {within:.5f}, max |diff| / ulp {(diff / ulp).max().item():.2f}")
    assert within >= 0.999, f"{tag}: only {within:.5f} of the elements within 1 ulp of ATen"
    flip = _stat_flip_bound(x, norm, bias, silu)
    assert (diff <= ulp + flip).all(), f"{tag}: {(diff > ulp + flip).sum().item()} elements off by more than 1 ulp " \
                                       "plus a one-ulp change of the fp16 statistics"
    ref = _fp64(x, norm, bias, silu)
    err_got = (g32.double() - ref).abs()
    err_aten = (w32.double() - ref).abs()
    ulp3 = _ulp(torch.maximum(torch.maximum(g32.abs(), w32.abs()), ref.float().abs())).double()
    assert (err_got <= err_aten + ulp3 + flip.double()).all(), f"{tag}: less accurate than ATen"
    again = ops.group_norm_nhwc(x, norm, bias, silu)
    assert torch.equal(again, got), f"{tag}: two launches differ"
    assert again.is_contiguous(memory_format=torch.channels_last)


@pytest.mark.gpu
@pytest.mark.parametrize("eps", [1e-5, 1e-6])
@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("c", CHANNELS)
@pytest.mark.parametrize("hw", SD15_HW + SD21_HW)
def test_group_norm_nhwc_matches_aten(ops, hw, c, bias, silu, eps):
    x, norm, b = _inputs(2, hw, c, bias, seed=hw + c)
    norm.eps = eps
    _check_against_aten(ops, x, norm, b, silu, f"hw={hw} c={c} bias={bias} silu={silu} eps={eps}")


@pytest.mark.gpu
@pytest.mark.parametrize("c,silu", [(320, True), (320, False), (640, True)])
def test_group_norm_nhwc_c2_top_level_batch(ops, c, silu):
    """The fused C2 step's batch: 3 streams x (5 keyframes + 40 frames) = 135 samples at the 64 x 64 latent."""
    x, norm, b = _inputs(135, 4096, c, True, seed=7)
    _check_against_aten(ops, x, norm, b, silu, f"N=135 c={c} silu={silu}")


@pytest.mark.gpu
def test_group_norm_nhwc_broadcast_bias_and_norm_act(ops):
    """A [1, C] bias broadcasts (row stride 0); `sd_unet.norm_act` takes the native path on channels_last fp16 and
    gives the ATen sequence's values."""
    from tokenflow_b200.sd_unet import norm_act
    x, norm, b = _inputs(3, 1024, 640, True, seed=11)
    b1 = b[:1]
    got = ops.group_norm_nhwc(x, norm, b1, True)
    want = _aten(x, norm, b1, True)
    bound = _ulp(torch.maximum(got.float().abs(), want.float().abs())) + _stat_flip_bound(x, norm, b1.expand(3, -1), True)
    assert ((got.float() - want.float()).abs() <= bound).all()
    before = ops.launch_count()
    via_helper = norm_act(norm, x, bias=b1, silu=True)
    assert ops.launch_count() - before == 2
    assert torch.equal(via_helper, got)


def _block_shapes():
    """(rows, inner) of the GEGLU of each of the 16 transformer blocks of the SD1.5 UNet at a 64 x 64 latent."""
    from bench import unet_levels
    out = []
    for S, dim, _, blocks in unet_levels("sd15", 64):
        out += [(S, 4 * dim)] * blocks
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(16))
def test_geglu_bit_equal_to_eager(ops, i):
    S, inner = _block_shapes()[i]
    g = torch.Generator(device="cuda").manual_seed(i)
    xh = (torch.randn(2, S, inner, device="cuda", generator=g) * 2).half()
    gate = (torch.randn(2, S, inner, device="cuda", generator=g) * 3).half()
    got = ops.geglu(xh, gate)
    assert torch.equal(got, xh * F.gelu(gate))


@pytest.mark.gpu
def test_geglu_module_bit_equal_to_eager():
    from tokenflow_b200.sd_unet import GEGLU
    torch.manual_seed(0)
    m = GEGLU(320, 1280).cuda().half()
    x = torch.randn(2, 4096, 320, device="cuda").half()
    w_x, w_g = m.proj.weight.chunk(2, dim=0)
    b_x, b_g = m.proj.bias.chunk(2, dim=0)
    with torch.no_grad():
        assert torch.equal(m(x), F.linear(x, w_x, b_x) * F.gelu(F.linear(x, w_g, b_g)))


def test_group_norm_and_geglu_argument_validation_needs_no_gpu():
    """Bad shapes are rejected on the host before anything touches the device."""
    from tokenflow_b200 import _build
    if not tf_ops.library_path().exists():
        _build.build()
    lib = tf_ops.load_library()
    buf = (ctypes.c_uint8 * 4096)()
    p = (ctypes.addressof(buf) + 15) & ~15
    st = lib.tf_group_norm_nhwc(p, None, 0, p, p, 2, 64, 324, 32, 1e-5, 1, p, 4096, p, None)     # c % 8 != 0
    assert st == 1 and b"c % 8" in lib.tf_last_error()
    st = lib.tf_group_norm_nhwc(p, None, 0, p, p, 2, 64, 328, 32, 1e-5, 1, p, 4096, p, None)     # 32 does not divide 328
    assert st == 1 and b"groups" in lib.tf_last_error()
    assert lib.tf_group_norm_nhwc_workspace(2, 64, 328, 32) == -1
    st = lib.tf_group_norm_nhwc(p, None, 0, p, p, 2, 64, 128, 32, 1e-5, 1, p, 4096, p, None)     # 4 channels / group
    assert st == 3
    st = lib.tf_group_norm_nhwc(p, p, 4, p, p, 2, 64, 320, 32, 1e-5, 1, p, 4096, p, None)       # bias stride 4
    assert st == 1 and b"bias" in lib.tf_last_error()
    need = lib.tf_group_norm_nhwc_workspace(2, 4096, 320, 32)
    assert need > 0
    st = lib.tf_group_norm_nhwc(p, None, 0, p, p, 2, 4096, 320, 32, 1e-5, 1, p, need - 16, p, None)
    assert st == 1 and b"workspace" in lib.tf_last_error()
    assert lib.tf_group_norm_nhwc(p, None, 0, p, p, 0, 4096, 320, 32, 1e-5, 1, None, 0, None, None) == 0   # empty
    assert lib.tf_geglu(None, None, -1, None, None) == 1
    assert lib.tf_geglu(None, None, 0, None, None) == 0
    assert lib.tf_geglu(p + 2, p, 8, p, None) == 1 and b"misaligned" in lib.tf_last_error()
