"""CPU tier: the Canny edge maps the ControlNet path conditions on.

* oracle/canny.py (numpy) equals `cv2.Canny` on random, smooth, checkerboard, line, channel-tie and flat frames, from
  1 x 1 up to 384 x 672 and 512 x 512, at several threshold pairs (low > high and non-integer ones included);
* tests/golden/canny.pt (cv2's own outputs, oracle/gen_canny_golden.py) equals the oracle, so the GPU tests that read
  it need no cv2;
* the serpentine probe really needs hysteresis to cross the whole frame;
* the reference's uint8 -> ToTensor -> fp16 -> x255 -> uint8 round trip in front of cv2.Canny returns every byte;
* `preprocess.canny_cond` on CPU frames is the reference's `get_canny_cond` expression;
* bad sizes and NULL buffers are rejected by the C ABI on the host.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import canny as oc
from oracle import gen_canny_golden as gg
from tokenflow_b200 import _build
from tokenflow_b200 import ops as tf_ops
from tokenflow_b200 import preprocess

cv2 = pytest.importorskip("cv2")

SIZES = [(1, 1), (1, 7), (6, 1), (2, 2), (3, 5), (17, 33), (64, 64), (97, 131), (384, 672), (512, 512)]
THRESHOLDS = [(100, 200), (200, 100), (50.7, 120.2), (0, 0), (10, 30), (99.99, 100.01), (300, 900)]


def _frames(kind, h, w, seed):
    return gg.make_frame(kind, h, w, np.random.default_rng(seed))


@pytest.mark.parametrize("kind", ["noise", "smooth", "checker", "lines", "ties", "flat"])
@pytest.mark.parametrize("size", SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_oracle_equals_cv2(kind, size):
    img = _frames(kind, *size, seed=size[0] * 1000 + size[1])
    for low, high in THRESHOLDS:
        assert np.array_equal(oc.canny(img, low, high), cv2.Canny(img, low, high)), (kind, size, low, high)


def test_oracle_equals_cv2_on_single_channel_ties():
    """Three equal channels tie everywhere: the first channel's direction is used, as with one channel."""
    img = _frames("smooth", 64, 96, 5)[:, :, :1]
    rgb = np.repeat(img, 3, axis=2)
    for low, high in THRESHOLDS:
        assert np.array_equal(oc.canny(rgb, low, high), cv2.Canny(rgb, low, high))
        assert np.array_equal(oc.canny(img[:, :, 0], low, high), cv2.Canny(img[:, :, 0], low, high))


def test_golden_matches_oracle():
    gold = torch.load(gg.GOLDEN, weights_only=False)
    for name, (kind, n, h, w, low, high, seed) in gg.CASES.items():
        want = gg.unpack(gold[name]["edges_bits"].numpy(), (n, h, w))
        frames = gg.case_frames(name)
        assert np.array_equal(oc.canny_frames(frames, low, high), want), name
        assert np.array_equal(np.stack([cv2.Canny(f, low, high) for f in frames]), want), name


@pytest.mark.parametrize("size", [(131, 97), (384, 672), (512, 512)])
def test_serpentine_needs_hysteresis_over_the_whole_frame(size):
    h, w = size
    img = gg.serpentine(h, w)
    cls = oc.classes(img, 100, 500)
    assert (cls == 2).sum() < 40 and (cls == 1).sum() > 10 * (cls == 2).sum()
    edges = oc.canny(img, 100, 500)
    assert np.array_equal(edges, cv2.Canny(img, 100, 500))
    start = tuple(np.argwhere(cls == 2)[0])
    (y0, y1), (x0, x1) = oc.chain_span(edges, start)
    assert y0 <= 3 and y1 >= h - 16 and x0 <= 3 and x1 >= w - 4
    assert (edges > 0).sum() == (cls > 0).sum()          # every candidate is reached


def test_reference_byte_round_trip_is_identity():
    """get_canny_cond feeds cv2 `np.uint8(np.array(255 * image))` of the fp16 ToTensor frames (preprocess.py:116-117,
    :193): for every byte that is the byte itself, so the uint8 frames go to Canny unchanged."""
    v = torch.arange(256, dtype=torch.uint8)
    image = (v.float() / 255).to(torch.float16)            # T.ToTensor() then .to(torch.float16)
    back = np.uint8(np.array(255 * image))
    assert np.array_equal(back, np.arange(256, dtype=np.uint8))


def test_canny_cond_cpu_is_the_reference_expression():
    frames = torch.from_numpy(gg.case_frames("smooth_3x97x131_swapped")).contiguous()
    got = preprocess.canny_cond(frames, 100, 200)
    edges = np.stack([cv2.Canny(f, 100, 200) for f in frames.numpy()])
    want = oc.canny_cond(edges)
    assert got.dtype == torch.float16 and got.shape == (3, 3, 97, 131)
    assert torch.equal(got, want)
    assert set(torch.unique(got).tolist()) <= {0.0, 1.0}


@pytest.fixture(scope="module")
def lib():
    if not tf_ops.library_path().exists():
        _build.build()
    return tf_ops.load_library()


def test_host_validation(lib):
    ws = (ctypes.c_uint8 * 4096)()
    p = (ctypes.addressof(ws) + 15) & ~15
    assert lib.tf_canny_workspace(2, 0, 5) == -1 and b"bad size" in lib.tf_last_error()
    assert lib.tf_canny_workspace(-1, 4, 4) == -1
    assert lib.tf_canny_workspace(1, 70000, 1) == -1
    assert lib.tf_canny_workspace(40000, 256, 256) == -1            # n*h*w >= 2^31
    need = lib.tf_canny_workspace(2, 8, 8)
    assert need >= 2 * 8 * 8 * 6
    st = lib.tf_canny_u8(p, 2, 8, 0, 100.0, 200.0, p, need, p, None, None)
    assert st == 1 and b"bad size" in lib.tf_last_error()
    st = lib.tf_canny_u8(p, 2, 8, 8, 100.0, 200.0, p, need - 1, p, None, None)
    assert st == 1 and b"workspace" in lib.tf_last_error()
    st = lib.tf_canny_u8(None, 2, 8, 8, 100.0, 200.0, p, need, p, None, None)
    assert st == 1 and b"NULL" in lib.tf_last_error()
    st = lib.tf_canny_u8(p, 2, 8, 8, 100.0, 200.0, p, need, None, None, None)      # no output at all
    assert st == 1 and b"NULL" in lib.tf_last_error()
    st = lib.tf_canny_u8(p, 2, 8, 8, 100.0, 200.0, p + 1, need, p, None, None)     # misaligned workspace
    assert st == 1
    st = lib.tf_canny_u8(p, 2, 8, 8, float("nan"), 200.0, p, need, p, None, None)
    assert st == 1 and b"NaN" in lib.tf_last_error()
    assert lib.tf_canny_u8(None, 0, 8, 8, 100.0, 200.0, None, 0, None, None, None) == 0    # no frames: no-op
