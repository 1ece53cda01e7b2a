"""CPU tier of the frame-preparation kernels' launch shapes: resizing (`tf_resize_u8`) and Canny (`tf_canny_u8`).

* oracle/frame_prep.py restates how tf_resize_u8 shapes its two launches; the GPU cases of test_gpu_frame_prep.py reach
  every horizontal class (1 to 4 staged rows, default and opt-in shared memory), both sides of every class boundary,
  every vertical class (16- and 4-byte columns, one and several column blocks), and every Canny threshold class.
* The library's host tables equal the numpy restatement of Pillow's (test_frame_sizes_cpu.py) at thousands of taps,
  at exact 3x ratios and at the widest sizes.
* oracle/canny.py equals `cv2.Canny` at 1080p and 4K, on the hysteresis probes, at every threshold class; the
  hysteresis probes are what they claim to be, and tests/golden/canny_probes.pt holds cv2's edges of them.
* A resize whose grid is too large for one launch is refused on the host before either pass is enqueued.
"""
import ctypes

import numpy as np
import pytest
from scipy import ndimage

from oracle import canny as oc
from oracle import frame_prep as fp
from oracle import gen_canny_golden as gg
from test_frame_sizes_cpu import _pass, lanczos_tables, pil_resize, resize_reference
from tokenflow_b200 import _build, ops

# ---------------------------------------------------------------------------------------------------------------------
# the GPU cases reach every dispatch class
# ---------------------------------------------------------------------------------------------------------------------
def test_resize_layout_classes():
    """Spot values of the restatement: the table of rows per width, and the column blocks of the vertical pass."""
    assert [fp.resize_h_rows(w) for w in (1, 4090, 4091, 5456, 5457, 8186, 8187, 16378, 16379, 65536)] == \
        [4, 4, 3, 3, 2, 2, 1, 1, 1, 1]
    lay = fp.resize_layout(2, 3, 16378, 2, 4093)
    assert lay["h"]["smem"] == 3 * 16378 + 16 <= fp.RESIZE_DEFAULT_SMEM and not lay["h"]["opt_in"]
    lay = fp.resize_layout(2, 3, 65536, 2, 16384)
    assert lay["h"]["opt_in"] and lay["h"]["smem"] <= fp.RESIZE_MAX_SMEM and lay["h"]["grid"] == 6
    assert fp.resize_layout(40, 1080, 1920, 768, 768)["v"] == {"vec": 16, "col_blocks": 2, "grid": 40 * 768 * 2}
    assert fp.resize_layout(1, 1080, 1920, 768, 768, tmp_off=1)["v"]["vec"] == 4
    assert fp.resize_layout(1, 1080, 1920, 768, 768, in_off=1)["v"]["vec"] == 16    # the pass reads tmp, not in
    assert fp.resize_layout(1, 1080, 768, 768, 768, in_off=1)["v"]["vec"] == 4      # ... unless it reads in
    assert fp.resize_layout(1, 64, 64, 64, 64) == {"h": None, "v": None, "v_first": False}


def test_gpu_resize_cases_reach_every_class():
    layouts = fp.resize_gpu_layouts()
    h_seen = {fp.resize_h_class(lay) for _, lay in layouts} - {None}
    v_seen = {fp.resize_v_class(lay) for _, lay in layouts} - {None}
    print("horizontal classes (rows, opt-in):", sorted(h_seen))
    print("vertical classes (vec, several column blocks):", sorted(v_seen))
    assert h_seen == set(fp.RESIZE_H_CLASSES)
    assert v_seen == set(fp.RESIZE_V_CLASSES)
    widths = {src[1] for src, _ in fp.RESIZE_ROWS_CASES}
    for a, b in fp.RESIZE_H_BOUNDARIES:
        assert {a, b} <= widths
        assert fp.resize_h_class(fp.resize_layout(1, 3, a, 2, 7)) != fp.resize_h_class(fp.resize_layout(1, 3, b, 2, 7))
    assert 65536 in widths
    # 16-byte columns with 1, 2 and 3 column blocks, from aligned buffers
    blocks = {lay["v"]["col_blocks"] for (_, dst, off), lay in layouts
              if off == 0 and lay["v"] and lay["v"]["vec"] == 16}
    assert {1, 2, 3} <= blocks
    # the offset matrix runs both vertical paths at one size
    both = {fp.resize_v_class(lay)[0] for (src, _, off), lay in layouts if isinstance(off, tuple) and src == (97, 700)}
    assert both == {4, 16}


def test_gpu_canny_thresholds_reach_every_class():
    seen = set().union(*(fp.canny_threshold_classes(lo, hi) for lo, hi in fp.CANNY_THRESHOLDS))
    print("Canny threshold classes:", sorted(seen))
    assert seen == set(fp.CANNY_THRESHOLD_CLASSES)
    assert fp.canny_threshold_classes(200.9, 200.2) == {"swapped", "fractional", "equal", "inside"}
    assert fp.canny_threshold_classes(-300, -20) == {"below"}


# ---------------------------------------------------------------------------------------------------------------------
# host tables on new axes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    if _build.needs_build():
        _build.build()
    return ops.load_library()


AXES = [(65536, 7), (4096, 3), (16384, 1), (3, 9), (9, 3), (27, 9), (768, 1024), (1024, 768), (1, 65536), (65536, 16384),
        (4091, 1021), (7680, 1920)]


@pytest.mark.parametrize("n_in,n_out", AXES)
def test_library_tables_equal_the_restatement(lib, n_in, n_out):
    bounds, coeffs = lanczos_tables(n_in, n_out)
    taps = lib.tf_resize_taps(n_in, n_out)
    assert taps == coeffs.shape[1]
    gb = np.full((n_out, 2), -7, np.int32)
    gk = np.full((n_out, taps), -7, np.int32)
    assert lib.tf_resize_coeffs(n_in, n_out, gb.ctypes.data, gk.ctypes.data) == 0
    assert np.array_equal(gb, bounds) and np.array_equal(gk, coeffs)


def _lanczos_args(n_in, n_out):
    """Every argument Resample.c's precompute_coeffs gives the Lanczos kernel for one axis, as the tables compute it."""
    bounds, _ = lanczos_tables(n_in, n_out)
    scale = float(np.float32(n_in)) / n_out
    ss = 1.0 / max(scale, 1.0)
    return [(x + int(x0) - (o + 0.5) * scale + 0.5) * ss for o, (x0, cnt) in enumerate(bounds) for x in range(cnt)]


def test_exact_ratios_hit_the_lanczos_edges():
    """At 3 -> 9 output centres fall on input pixel centres, so some tap's argument is exactly 0 (sinc's own branch);
    at 27 -> 9 some taps sit exactly on 3, just outside the kernel's [-3, 3) window, and weigh 0."""
    assert 0.0 in _lanczos_args(3, 9)
    assert 3.0 in _lanczos_args(27, 9)
    b, k = lanczos_tables(27, 9)
    assert (b[:, 1] < k.shape[1]).any() or (k == 0).any()


@pytest.mark.parametrize("src,dst", [((4096, 5), (3, 4)), ((501, 5), (100, 4)), ((8192, 2), (8000, 7)),
                                     ((500, 5), (100, 4)), ((4096, 5), (4097, 4)), ((5, 4096), (4, 3))])
def test_pil_resizes_tall_frames_vertically_first(src, dst):
    """Pillow's Image.resize takes a frame more than 100 times taller than wide whose height shrinks through the
    vertical pass first; the two orders round the intermediate differently, so the order is part of the result."""
    img = np.random.default_rng(sum(src)).integers(0, 256, (*src, 3), dtype=np.uint8)
    (h_in, w_in), (h, w) = src, dst
    v_first = _pass(_pass(img, *lanczos_tables(h_in, h), axis=0), *lanczos_tables(w_in, w), axis=1)
    assert fp.resize_v_first(h_in, w_in, h, w) == (h_in > 100 * w_in and h < h_in)
    want = v_first if fp.resize_v_first(h_in, w_in, h, w) else resize_reference(img, h, w)
    assert np.array_equal(pil_resize(img, h, w), want)
    if (src, dst) == ((4096, 5), (3, 4)):
        assert not np.array_equal(resize_reference(img, h, w), want)     # the other order is not PIL's


def test_gpu_resize_cases_take_both_orders():
    cases = [c for c, _ in fp.resize_gpu_layouts()]
    v_first = {fp.resize_v_first(*src, *dst) for src, dst, _ in cases if src[1] != dst[1] and src[0] != dst[0]}
    assert v_first == {False, True}
    assert {((500, 5), (100, 4)), ((501, 5), (100, 4))} <= {(src, dst) for src, dst, _ in cases}


# ---------------------------------------------------------------------------------------------------------------------
# the resize grid limits, on the host
# ---------------------------------------------------------------------------------------------------------------------
def _resize_call(lib, n, h_in, w_in, h, w, ptr=16, tmp=16, out=16):
    buf = (ctypes.c_int32 * 4)()
    ht = lib.tf_resize_taps(w_in, w) if w != w_in else 0
    vt = lib.tf_resize_taps(h_in, h) if h != h_in else 0
    return lib.tf_resize_u8(ptr, n, h_in, w_in, h, w, buf, buf, ht, buf, buf, vt, tmp, out, None)


def test_resize_grid_limits_are_checked_before_any_launch(lib):
    """Pointers that no device could dereference: a refused call must neither launch nor look at them."""
    before = lib.tf_launch_count()
    # horizontal only: 2^31 + 3 rows at 4 per block is one block too many; one frame fewer fits
    n = (2 ** 31 - 1) * 4 // 8 + 1
    assert fp.resize_layout(n, 8, 64, 8, 32)["h"]["grid"] > fp.MAX_GRID
    assert _resize_call(lib, n, 8, 64, 8, 32) == 3 and b"horizontal launch" in lib.tf_last_error()
    assert fp.resize_layout(n - 1, 8, 64, 8, 32)["h"]["grid"] <= fp.MAX_GRID
    # one row per block from w_in = 16379 on
    n = 2 ** 31 // 2
    assert fp.resize_layout(n, 2, 16379, 2, 8)["h"]["grid"] > fp.MAX_GRID
    assert _resize_call(lib, n, 2, 16379, 2, 8) == 3 and b"horizontal launch" in lib.tf_last_error()
    # both passes: the horizontal grid fits, the vertical one does not, and nothing is enqueued for either
    n = 2 ** 26
    lay = fp.resize_layout(n, 2, 8, 64, 16)
    assert lay["h"]["grid"] <= fp.MAX_GRID < lay["v"]["grid"]
    assert _resize_call(lib, n, 2, 8, 64, 16) == 3 and b"vertical launch" in lib.tf_last_error()
    # the vertical pass's column blocks follow the alignment of the buffers it reads and writes
    n = fp.MAX_GRID // (64 * 2) + 1                       # w = 768: 2 blocks of 16-byte columns, 5 of 4-byte ones
    assert fp.resize_layout(n, 32, 768, 64, 768)["v"]["grid"] > fp.MAX_GRID
    assert _resize_call(lib, n, 32, 768, 64, 768) == 3 and b"vertical launch" in lib.tf_last_error()
    n = fp.MAX_GRID // (64 * 5) + 1
    assert fp.resize_layout(n, 32, 768, 64, 768, in_off=1)["v"]["grid"] > fp.MAX_GRID
    assert _resize_call(lib, n, 32, 768, 64, 768, ptr=17) == 3
    # huge frame counts: no product overflows into a small grid
    for n in (2 ** 40, 2 ** 62):
        assert _resize_call(lib, n, 65536, 65536, 1, 1) == 3
        assert _resize_call(lib, n, 1, 1, 65536, 1) == 3
    assert lib.tf_launch_count() == before


# ---------------------------------------------------------------------------------------------------------------------
# the numpy Canny against OpenCV at production sizes and on the hysteresis probes
# ---------------------------------------------------------------------------------------------------------------------
cv2 = pytest.importorskip("cv2")


@pytest.mark.parametrize("kind", ["smooth", "noise"])
@pytest.mark.parametrize("h,w", [(1080, 1920), (2160, 3840)])
def test_oracle_equals_cv2_at_production_sizes(kind, h, w):
    img = gg.make_frame(kind, h, w, np.random.default_rng(h + w))
    assert np.array_equal(oc.canny(img, 100, 200), cv2.Canny(img, 100, 200))


def _probes(h, w):
    rng = np.random.default_rng(h * w)
    return {"dense": (gg.dense(h, w), 100, 500), "comb": (gg.comb(h, w), 100, 500),
            "serpentine": (gg.serpentine(h, w), 100, 500),
            "noise_low": (rng.integers(0, 256, (h, w, 3), dtype=np.uint8), 5, 600)}


@pytest.mark.parametrize("h,w", [(512, 512), (1080, 1920)])
def test_oracle_equals_cv2_on_the_hysteresis_probes(h, w):
    for name, (img, lo, hi) in _probes(h, w).items():
        for f in (img, np.ascontiguousarray(img[::-1, ::-1])):
            assert np.array_equal(oc.canny(f, lo, hi), cv2.Canny(f, lo, hi)), name


def _components(mask):
    return ndimage.label(mask, structure=np.ones((3, 3), dtype=bool))


def test_hysteresis_probes_are_what_they_claim():
    h, w = 512, 512
    p = _probes(h, w)
    # dense: two thirds candidates, one component, strong only in the frame's last 32 x 16 tile, every one an edge
    img, lo, hi = p["dense"]
    cls = oc.classes(img, lo, hi)
    assert (cls > 0).mean() > 0.65 and _components(cls > 0)[1] == 1
    ys, xs = np.nonzero(cls == 2)
    assert ys.min() >= (h - 1) // 16 * 16 and xs.min() >= (w - 1) // 32 * 32
    assert ((oc.canny(img, lo, hi) > 0) == (cls > 0)).all()
    # comb: the teeth are separate above the bar and all reached through it
    img, lo, hi = p["comb"]
    cls = oc.classes(img, lo, hi)
    teeth = len(range(3, w - 4 - 2, 10))
    assert _components(cls[:h - 9] > 0)[1] >= teeth and _components(cls > 0)[1] == 1
    assert ((oc.canny(img, lo, hi) > 0) == (cls > 0)).all()
    # noise at low thresholds: many small components, some without a strong pixel
    img, lo, hi = p["noise_low"]
    cls = oc.classes(img, lo, hi)
    labels, n = _components(cls > 0)
    assert n > 5000 and np.bincount(labels.ravel())[1:].max() < 1000
    assert (oc.canny(img, lo, hi) > 0).sum() < (cls > 0).sum()


@pytest.mark.parametrize("low,high", fp.CANNY_THRESHOLDS)
def test_oracle_equals_cv2_at_every_threshold_class(low, high):
    rng = np.random.default_rng(7)
    for img in (gg.make_frame("smooth", 200, 300, rng), gg.make_frame("noise", 64, 96, rng), gg.dense(64, 96),
                gg.make_frame("checker", 64, 96, rng)):
        assert np.array_equal(oc.canny(img, low, high), cv2.Canny(img, low, high)), (low, high)


def test_probe_golden_matches_oracle_and_cv2():
    """tests/golden/canny_probes.pt (cv2's own edges of the hysteresis probes at 512 x 512 and of a 1080p frame) equals
    the oracle and cv2, so the GPU tier can check the kernel against it without cv2."""
    import torch
    gold = torch.load(gg.PROBE_GOLDEN, weights_only=False)
    assert set(gold) - {"_opencv"} == set(gg.PROBE_CASES) and not set(gg.PROBE_CASES) & set(gg.CASES)
    assert sum(gold[k]["edges_bits"].numel() for k in gg.PROBE_CASES) < 1 << 20
    for name, (kind, n, h, w, low, high, seed) in gg.PROBE_CASES.items():
        want = gg.unpack(gold[name]["edges_bits"].numpy(), (n, h, w))
        frames = gg.case_frames(name)
        assert np.array_equal(oc.canny_frames(frames, low, high), want), name
        assert np.array_equal(np.stack([cv2.Canny(f, low, high) for f in frames]), want), name
    frames = gg.case_frames("hysteresis_8x512x512")
    assert np.array_equal(frames[0], gg.dense(512, 512)) and np.array_equal(frames[4], gg.dense(512, 512)[::-1, ::-1])
