"""CPU tier of frame resizing and non-square latents.

* The integer algorithm of Pillow's LANCZOS resize (libImaging/Resample.c), restated below in numpy, equals
  `PIL.Image.resize` byte for byte, and the library's host tables (`tf_resize_coeffs`, read through ctypes, no GPU)
  equal this restatement's integer for integer: the kernels apply those tables with the same integer arithmetic.
* The SD-shaped UNet runs at latent sizes whose sides are not multiples of 8 (diffusers' `upsample_size` rule), and
  the TokenFlow hooks on the oracle ops equal the unmodified reference hooks at such a size (a PnP edit, with
  separate and with fused passes).
"""
import ctypes
import math

import numpy as np
import pytest
import torch
from PIL import Image

from tokenflow_b200 import _build, ops
from tokenflow_b200.preprocess import resize_frames

PRECISION_BITS = 22


# ---------------------------------------------------------------------------------------------------------------------
# Pillow's LANCZOS resize in numpy
# ---------------------------------------------------------------------------------------------------------------------
def _lanczos(x: float) -> float:
    def sinc(v):
        if v == 0.0:
            return 1.0
        v = v * math.pi
        return math.sin(v) / v
    return sinc(x) * sinc(x / 3) if -3.0 <= x < 3.0 else 0.0


def lanczos_tables(n_in: int, n_out: int):
    """(bounds [out, 2] int32 (first input pixel, taps used), coeffs [out, taps] int32) of one axis: Resample.c's
    precompute_coeffs + normalize_coeffs_8bpc."""
    scale = float(np.float32(n_in)) / n_out
    fs = max(scale, 1.0)
    support = 3.0 * fs
    ss = 1.0 / fs
    taps = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((n_out, 2), np.int32)
    coeffs = np.zeros((n_out, taps), np.int32)
    for xx in range(n_out):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)          # int() truncates toward zero like the C cast
        xmax = min(int(center + support + 0.5), n_in) - xmin
        w = [_lanczos((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in w:
            ww += v
        for x, v in enumerate(w):
            v = v / ww if ww != 0.0 else v
            coeffs[xx, x] = int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
        bounds[xx] = (xmin, xmax)
    return bounds, coeffs


def _pass(img: np.ndarray, bounds, coeffs, axis: int) -> np.ndarray:
    """One pass along `axis` (1 = horizontal, 0 = vertical) of an [H, W, 3] uint8 image, int32 accumulation."""
    src = np.moveaxis(img.astype(np.int64), axis, 0)
    out = np.empty((len(bounds),) + src.shape[1:], np.uint8)
    for o, (xmin, cnt) in enumerate(bounds):
        acc = (1 << (PRECISION_BITS - 1)) + np.tensordot(coeffs[o, :cnt].astype(np.int64), src[xmin:xmin + cnt], 1)
        out[o] = np.clip(acc >> PRECISION_BITS, 0, 255)
    return np.moveaxis(out, 0, axis)


def resize_reference(img: np.ndarray, h: int, w: int) -> np.ndarray:
    """[H_in, W_in, 3] uint8 -> [h, w, 3]: horizontal pass first into uint8, then vertical; unchanged axes skipped."""
    out = img
    if w != img.shape[1]:
        out = _pass(out, *lanczos_tables(img.shape[1], w), axis=1)
    if h != img.shape[0]:
        out = _pass(out, *lanczos_tables(img.shape[0], h), axis=0)
    return out.copy()


def pil_resize(img: np.ndarray, h: int, w: int) -> np.ndarray:
    return np.asarray(Image.fromarray(img).resize((w, h), Image.LANCZOS))


def content(kind: str, h: int, w: int, seed: int = 0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    if kind == "checker":               # 0 / 255 cells: Lanczos over- and undershoots at every edge
        return np.repeat((((yy // 3 + xx // 2) % 2) * 255).astype(np.uint8)[..., None], 3, axis=2)
    if kind == "edges":                 # hard steps in different directions per channel
        return np.stack([(xx >= w // 3) * 255, (yy >= h // 2) * 255, ((xx + yy) % 7 == 0) * 255], -1).astype(np.uint8)
    raise ValueError(kind)


SIZES = [  # (h_in, w_in) -> (h, w)
    ((45, 80), (24, 42)),          # down both axes
    ((24, 42), (45, 80)),          # up both axes
    ((60, 30), (97, 13)),          # up one axis, down the other
    ((37, 53), (37, 19)),          # horizontal only
    ((41, 29), (11, 29)),          # vertical only
    ((53, 47), (31, 17)),          # primes
    ((19, 23), (1, 1)),            # one-pixel output
    ((7, 5), (3, 200)),            # heavy upscale of a tiny image
    ((31, 33), (31, 33)),          # identity
    ((270, 480), (96, 168)),       # 1920x1080 -> 672x384 at a quarter of the size
]


@pytest.mark.parametrize("kind", ["random", "checker", "edges"])
@pytest.mark.parametrize("src,dst", SIZES, ids=[f"{a[0]}x{a[1]}-{b[0]}x{b[1]}" for a, b in SIZES])
def test_numpy_restatement_equals_pil(src, dst, kind):
    img = content(kind, *src, seed=sum(src) + sum(dst))
    want = pil_resize(img, *dst)
    got = resize_reference(img, *dst)
    assert got.shape == want.shape and np.array_equal(got, want)


def test_clamp_is_exercised():
    """The checkerboard drives the accumulator below 0 and above 255 << 22: both clamps are part of the result."""
    img = content("checker", 53, 47)
    b, k = lanczos_tables(47, 31)
    raw = [(1 << 21) + int(np.dot(k[o, :c].astype(np.int64), img[r, x0:x0 + c, 0].astype(np.int64)))
           for r in range(53) for o, (x0, c) in enumerate(b)]
    assert min(raw) < 0 and max(raw) >> PRECISION_BITS > 255


@pytest.fixture(scope="module")
def lib():
    if _build.needs_build():
        _build.build()
    return ops.load_library()


AXES = [(1920, 672), (1080, 384), (1080, 512), (1280, 384), (720, 672), (320, 672), (240, 384), (1920, 640),
        (1080, 360), (53, 31), (7, 200), (19, 1), (1, 5), (5000, 3), (100, 100)]


@pytest.mark.parametrize("n_in,n_out", AXES)
def test_library_tables_equal_the_restatement(lib, n_in, n_out):
    bounds, coeffs = lanczos_tables(n_in, n_out)
    taps = lib.tf_resize_taps(n_in, n_out)
    assert taps == coeffs.shape[1]
    gb = np.full((n_out, 2), -7, np.int32)
    gk = np.full((n_out, taps), -7, np.int32)
    assert lib.tf_resize_coeffs(n_in, n_out, gb.ctypes.data, gk.ctypes.data) == 0
    assert np.array_equal(gb, bounds) and np.array_equal(gk, coeffs)


def test_resize_arguments_are_checked_on_the_host(lib):
    assert lib.tf_resize_taps(0, 5) == -1 and b"sizes" in lib.tf_last_error()
    assert lib.tf_resize_taps(5, 70000) == -1
    buf = (ctypes.c_int32 * 64)()
    assert lib.tf_resize_coeffs(8, 4, None, buf) == 1
    assert lib.tf_resize_coeffs(-1, 4, buf, buf) == 1
    # a table of the wrong width, a negative frame count, a zero size: rejected before any CUDA call
    taps = lib.tf_resize_taps(64, 32)
    st = lib.tf_resize_u8(None, 1, 64, 64, 32, 32, buf, buf, taps + 1, buf, buf, taps, None, None, None)
    assert st == 1 and b"taps" in lib.tf_last_error()
    assert lib.tf_resize_u8(None, -1, 64, 64, 32, 32, buf, buf, taps, buf, buf, taps, None, None, None) == 1
    assert lib.tf_resize_u8(None, 1, 64, 0, 32, 32, buf, buf, taps, buf, buf, taps, None, None, None) == 1
    st = lib.tf_resize_u8(None, 1, 64, 64, 32, 32, buf, buf, taps, buf, buf, taps, None, None, None)
    assert st == 1 and b"NULL" in lib.tf_last_error()
    assert lib.tf_resize_u8(None, 0, 64, 64, 32, 32, buf, buf, taps, buf, buf, taps, None, None, None) == 0


def test_preprocess_resize_frames_on_the_host_is_pil():
    frames = torch.from_numpy(np.stack([content("random", 45, 80, s) for s in range(3)]))
    got = resize_frames(frames, (24, 42))
    assert got.dtype == torch.uint8 and got.shape == (3, 24, 42, 3)
    for i in range(3):
        assert np.array_equal(got[i].numpy(), pil_resize(frames[i].numpy(), 24, 42))
    same = resize_frames(frames, (45, 80))
    assert torch.equal(same, frames) and same.data_ptr() != frames.data_ptr()
    assert torch.equal(resize_frames(frames, 16), torch.from_numpy(np.stack(
        [pil_resize(f.numpy(), 16, 16) for f in frames])))


# ---------------------------------------------------------------------------------------------------------------------
# latents of any shape
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hw", [(12, 21), (45, 80), (48, 84)])
def test_tiny_unet_runs_at_non_square_latents(hw):
    """Sides that are not multiples of 8 lose a row or column on the way down (21 -> 11 -> 6 -> 3); every up block but
    the last upsamples to its next skip's size instead of doubling."""
    from tokenflow_b200 import sd_unet
    unet = sd_unet.build_unet("tiny")
    x = torch.randn(2, 4, *hw, generator=torch.Generator().manual_seed(0))
    seen = []
    hooks = [b.upsamplers[0].register_forward_hook(lambda m, i, o: seen.append(tuple(o.shape[-2:])))
             for b in unet.up_blocks if b.upsamplers is not None]
    with torch.no_grad():
        out = unet(x, 981, encoder_hidden_states=torch.randn(2, 7, 32)).sample
    for h in hooks:
        h.remove()
    assert out.shape == x.shape and torch.isfinite(out).all()
    sizes = [hw]
    for _ in range(3):
        sizes.append(((sizes[-1][0] + 1) // 2, (sizes[-1][1] + 1) // 2))     # stride-2 conv, padding 1
    assert seen == sizes[2::-1]


def test_unet_keeps_doubling_at_multiples_of_8():
    """Latents whose sides are multiples of 8 take the scale-factor path, the code every existing shape runs."""
    from tokenflow_b200 import sd_unet
    unet = sd_unet.build_unet("tiny")
    calls = []
    for b in unet.up_blocks:
        if b.upsamplers is not None:
            b.upsamplers[0].register_forward_pre_hook(lambda m, args: calls.append(args[1] if len(args) > 1 else None))
    with torch.no_grad():
        unet(torch.randn(1, 4, 16, 24), 1, encoder_hidden_states=torch.randn(1, 7, 32))
    assert calls == [None, None, None]


def test_tiny_vae_at_non_square_frames():
    from tokenflow_b200.preprocess import decode_latents, encode_imgs
    from tokenflow_b200.vae import build_vae
    vae = build_vae("tiny", seed=1)
    frames = torch.from_numpy(np.stack([content("random", 48, 80, s) for s in range(2)]))
    lat = encode_imgs(vae, frames, batch_size=2)
    assert lat.shape == (2, 4, 6, 10)
    out = decode_latents(vae, lat)
    assert out.shape == (2, 48, 80, 3) and out.dtype == torch.uint8


def test_non_square_pnp_edit_matches_reference(golden_dir):
    """The tiny SD-topology UNet at 12 x 21 latents (S = 252, 66, 18 tokens at the attention levels), 4 frames, B = 2,
    a 2-step PnP edit, through this package's hooks on the oracle ops == through the unmodified reference hooks.  The
    golden is `unet_case(ref, "pnp", latent=(12, 21))` of oracle/gen_golden.py."""
    from oracle import golden
    from oracle.oracle_ops import OracleOps
    from tokenflow_b200 import sd_unet
    from tokenflow_b200 import tokenflow_utils as tfu
    from tokenflow_b200.editor import TokenFlowEditor, synthetic_inputs
    from tokenflow_b200.scheduler import DDIMScheduler
    tfu._install_ops_for_testing(OracleOps())
    c = golden.load(golden_dir, "unet_c1_nonsquare.pt")
    assert tuple(c["latent"]) == (12, 21)
    for fused in (False, True):
        cfg = dict(c["config"], fused_pass=fused)
        unet = sd_unet.build_unet("tiny", seed=c["seed"])
        x, text, pnp, src = synthetic_inputs(cfg["n_frames"], c["latent"], unet.config.cross_attention_dim,
                                             cfg["n_timesteps"], seed=c["seed"], ctx_len=c["ctx_len"])
        assert torch.equal(x, c["x0"])
        ed = TokenFlowEditor(unet, DDIMScheduler(), tfu, cfg, text, pnp, source_latents=lambda t: src[t])
        ed.init_method()
        torch.manual_seed(c["seed"])
        steps = []
        out = ed.sample_loop(x, on_step=lambda i, t, z: steps.append(z.clone()))
        assert ed.keyframe_log == c["keyframes"]
        for got, want in zip(steps, c["steps"]):
            assert torch.allclose(got, want, atol=2e-4, rtol=1e-4)
        assert torch.allclose(out, c["out"], atol=2e-4, rtol=1e-4)
