"""GPU tier (-m gpu) of the frame-preparation kernels at every launch shape they take.

* `tf_resize_u8` equals PIL's LANCZOS resize byte for byte in every horizontal class (1 to 4 input rows staged per
  block, default and opt-in shared memory, both sides of each class boundary, up to 65536 wide), with 16-byte
  columns over 1, 2 and 3 column blocks, at thousands of taps and at exact 3x ratios, on frames more than 100 times
  taller than wide (which Pillow resizes vertically first), from 1080p to 768 x 768, and at every (0, 1, 8, 15) byte
  offset of input, intermediate and output; `tmp` and `out` sit between sentinel-filled guard bands and the
  intermediate equals PIL's resize along the first axis.  oracle/frame_prep.py names the class of each case, and
  test_frame_prep_cpu.py checks that the cases reach them all.
* `tf_canny_u8` equals cv2's own edges of tests/golden/canny_probes.pt, and the numpy oracle (itself checked against
  cv2 on the CPU) at production shapes up to 4K, at every threshold class, on the hysteresis probes (a frame-wide
  component lit from its last tile, the serpentine, a comb joined in its last rows, noise at low thresholds), at odd
  buffer offsets, and with pixel labels within one frame of INT32_MAX.
* Captured CUDA graphs of both follow new frame content on replay, and 40 frames at 1080p go through resize and
  Canny on the device to the host chain's conditioning tensor.
"""
import numpy as np
import pytest
import torch
from PIL import Image

from oracle import canny as oc
from oracle import frame_prep as fp
from oracle import gen_canny_golden as gg
from tokenflow_b200 import ops as tf_ops
from tokenflow_b200 import preprocess

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
GUARD = 256                         # a multiple of 16: a view's byte offset past its buffer's start is its alignment


@pytest.fixture(scope="module")
def ops():
    return tf_ops.CudaOps()


def _content(kind, n, h, w, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]             # 0 / 255 cells of a few sizes: Lanczos rings at every edge, both clamps bite
    base = np.stack([((yy // (1 + f) + xx // (2 + f)) % 2) * 255 for f in range(3)], -1).astype(np.uint8)
    frames = np.repeat(base[None], n, axis=0)
    frames[1::2] = 255 - frames[1::2]
    return frames


def _pil(frames, h, w):
    return np.stack([np.asarray(Image.fromarray(f).resize((w, h), Image.LANCZOS)) for f in frames])


def _guarded(numel, off, dtype=torch.uint8, fill=SENTINEL):
    buf = torch.full((GUARD + off + numel + GUARD,), fill, dtype=dtype, device="cuda")
    return buf, buf[GUARD + off:GUARD + off + numel]


def _guards_intact(buf, off, numel, fill=SENTINEL):
    head, tail = buf[:GUARD + off], buf[GUARD + off + numel:]
    if isinstance(fill, float) and fill != fill:
        return bool(head.isnan().all()) and bool(tail.isnan().all())
    return bool((head == fill).all()) and bool((tail == fill).all())


def _resize_check(ops, frames, dst, in_off=0, tmp_off=0, out_off=0):
    """Resize `frames` on the device from buffers at the given byte offsets; everything must equal PIL and nothing
    outside `tmp` and `out` may change.  Returns the layout the call took."""
    n, h_in, w_in, _ = frames.shape
    h, w = dst
    v_first = fp.resize_v_first(h_in, w_in, h, w)
    tmp_hw = (h, w_in) if v_first else (h_in, w)
    ibuf, inp = _guarded(frames.size, in_off)
    inp.copy_(torch.from_numpy(frames.reshape(-1)))
    tbuf, tmp = _guarded(n * tmp_hw[0] * tmp_hw[1] * 3, tmp_off)
    obuf, out = _guarded(n * h * w * 3, out_off)
    lay = fp.resize_layout(n, h_in, w_in, h, w, inp.data_ptr() % 16, tmp.data_ptr() % 16, out.data_ptr() % 16)
    assert lay == fp.resize_layout(n, h_in, w_in, h, w, in_off, tmp_off, out_off)
    got = ops.resize_frames(inp.view(n, h_in, w_in, 3), (h, w), tmp=tmp.view(n, *tmp_hw, 3), out=out.view(n, h, w, 3))
    torch.cuda.synchronize()
    assert got.data_ptr() == out.data_ptr()
    want = _pil(frames, h, w)
    bad = got.cpu().numpy() != want
    assert not bad.any(), f"{lay}: {int(bad.sum())} of {bad.size} bytes differ from PIL"
    assert _guards_intact(obuf, out_off, out.numel())
    assert _guards_intact(ibuf, in_off, inp.numel()) and np.array_equal(inp.cpu().numpy(), frames.reshape(-1))
    if w != w_in and h != h_in:              # both passes: the intermediate is PIL's resize along the first axis
        assert _guards_intact(tbuf, tmp_off, tmp.numel())
        assert np.array_equal(tmp.view(n, *tmp_hw, 3).cpu().numpy(), _pil(frames, *tmp_hw))
    else:                                    # one pass: tmp is not touched
        assert bool((tbuf == SENTINEL).all())
    return lay


def _ids(cases):
    return [f"{s[1]}x{s[0]}-{d[1]}x{d[0]}" for s, d, *_ in cases]


# ---------------------------------------------------------------------------------------------------------------------
# resize
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["random", "checker"])
@pytest.mark.parametrize("src,dst", fp.RESIZE_ROWS_CASES, ids=_ids(fp.RESIZE_ROWS_CASES))
def test_resize_every_horizontal_class(ops, src, dst, kind):
    lay = _resize_check(ops, _content(kind, 2, *src, seed=src[1] + dst[1]), dst)
    assert lay["h"]["rows"] == fp.resize_h_rows(src[1])


@pytest.mark.parametrize("src,dst,off", fp.RESIZE_VEC_CASES, ids=[f"{i}-off{c[2]}" for i, c in
                                                                    zip(_ids(fp.RESIZE_VEC_CASES), fp.RESIZE_VEC_CASES)])
def test_resize_vertical_column_blocks(ops, src, dst, off):
    lay = _resize_check(ops, _content("random", 2, *src, seed=dst[1]), dst, tmp_off=off, out_off=off)
    assert (lay["v"]["vec"] == 16) == (off == 0 and dst[1] % 16 == 0)


@pytest.mark.parametrize("kind", ["random", "checker"])
@pytest.mark.parametrize("src,dst", fp.RESIZE_RATIO_CASES, ids=_ids(fp.RESIZE_RATIO_CASES))
def test_resize_large_taps_and_exact_ratios(ops, src, dst, kind):
    _resize_check(ops, _content(kind, 2, *src, seed=src[0] + dst[0]), dst)


def test_resize_1080p_to_768_square(ops):
    """SD 2.x's 768 x 768 from 8 1080p frames: 16-byte columns in 2 blocks per row, into fresh tensors as well."""
    frames = _content("random", 8, 1080, 1920, seed=768)
    lay = _resize_check(ops, frames, (768, 768))
    assert lay["v"] == {"vec": 16, "col_blocks": 2, "grid": 8 * 768 * 2}
    got = ops.resize_frames(torch.from_numpy(frames).cuda(), (768, 768))
    assert np.array_equal(got.cpu().numpy(), _pil(frames, 768, 768))


@pytest.mark.parametrize("in_off", fp.RESIZE_OFFSETS)
@pytest.mark.parametrize("src,dst", fp.RESIZE_OFFSET_SIZES, ids=_ids(fp.RESIZE_OFFSET_SIZES))
def test_resize_at_every_byte_offset(ops, src, dst, in_off):
    frames = _content("checker", 2, *src, seed=in_off)
    vecs = set()
    for tmp_off in fp.RESIZE_OFFSETS:
        for out_off in fp.RESIZE_OFFSETS:
            vecs.add(_resize_check(ops, frames, dst, in_off, tmp_off, out_off)["v"]["vec"])
    assert vecs == ({4, 16} if dst[1] % 16 == 0 else {4})


# ---------------------------------------------------------------------------------------------------------------------
# Canny
# ---------------------------------------------------------------------------------------------------------------------
def _canny_check(ops, frames, low, high):
    e, c = ops.canny(torch.from_numpy(frames).cuda(), low, high)
    torch.cuda.synchronize()
    got = e.cpu().numpy()
    want = oc.canny_frames(frames, low, high)
    bad = (got != want).reshape(len(frames), -1).sum(1)
    assert not bad.any(), f"({low}, {high}): pixels differing per frame {bad.tolist()}"
    assert torch.equal(c.cpu(), oc.canny_cond(want))
    return want


@pytest.mark.parametrize("name", list(gg.PROBE_CASES))
def test_canny_probe_golden(ops, name):
    """cv2's own edges of the hysteresis probes and of a 1080p frame (tests/golden/canny_probes.pt)."""
    gold = torch.load(gg.PROBE_GOLDEN, weights_only=False)[name]
    kind, n, h, w, low, high, _ = gg.PROBE_CASES[name]
    frames = gg.case_frames(name)
    want = gg.unpack(gold["edges_bits"].numpy(), (n, h, w))
    e, c = ops.canny(torch.from_numpy(frames).cuda(), low, high)
    torch.cuda.synchronize()
    got = e.cpu().numpy()
    bad = (got != want).reshape(n, -1).sum(1)
    assert not bad.any(), f"{name}: pixels differing per frame {bad.tolist()}"
    assert torch.equal(c.cpu(), oc.canny_cond(want))


@pytest.mark.parametrize("n,h,w", [(40, 512, 512), (8, 768, 768), (2, 1080, 1920), (1, 2160, 3840)])
def test_canny_production_shapes(ops, n, h, w):
    rng = np.random.default_rng(n + h + w)
    frames = np.stack([gg.make_frame("smooth" if i % 4 else "noise", h, w, rng) for i in range(n)])
    _canny_check(ops, frames, 100, 200)


@pytest.mark.parametrize("low,high", fp.CANNY_THRESHOLDS)
def test_canny_every_threshold_class(ops, low, high):
    rng = np.random.default_rng(11)
    frames = np.stack([gg.make_frame("smooth", 128, 192, rng), gg.make_frame("noise", 128, 192, rng),
                       gg.dense(128, 192), gg.make_frame("checker", 128, 192, rng)])
    want = _canny_check(ops, frames, low, high)
    classes = fp.canny_threshold_classes(low, high)
    if "above" in classes:                   # no magnitude exceeds 2040: nothing is strong
        assert not want.any()
    if max(low, high) < 0:                   # both clamped to -1: every non-suppressed pixel is an edge
        assert np.array_equal(want > 0, np.stack([oc.classes(f, -1, -1) > 0 for f in frames]))


def _turned(img):
    return np.ascontiguousarray(img[::-1, ::-1])


@pytest.mark.parametrize("h,w", [(512, 512), (1080, 1920), (2160, 3840)])
def test_canny_hysteresis_probes(ops, h, w):
    probes = [gg.serpentine(h, w), gg.dense(h, w)]
    if h < 2160:
        probes += [gg.comb(h, w)]
    frames = np.stack(probes + [_turned(p) for p in probes])
    want = _canny_check(ops, frames, 100, 500)
    # the frame-wide component is lit from the last tile (first tile once turned): every candidate is an edge
    dense_cls = oc.classes(frames[1], 100, 500)
    assert (dense_cls > 0).mean() > 0.65 and np.array_equal(want[1] > 0, dense_cls > 0)
    noise = np.random.default_rng(h).integers(0, 256, (2, h, w, 3), dtype=np.uint8)
    _canny_check(ops, noise, 5, 600)


def test_canny_at_odd_offsets(ops):
    frames_np = gg.case_frames("smooth_3x97x131_swapped")
    n, h, w, _ = frames_np.shape
    want = oc.canny_frames(frames_np, 180.5, 60.25)
    for f_off, e_off, c_off in [(1, 1, 1), (3, 7, 3), (15, 0, 5), (0, 13, 0)]:
        fbuf, frames = _guarded(frames_np.size, f_off)
        frames.copy_(torch.from_numpy(frames_np.reshape(-1)))
        ebuf, edges = _guarded(n * h * w, e_off)
        cbuf, cond = _guarded(3 * n * h * w, c_off, torch.float16, float("nan"))       # element offset: 2 bytes each
        ops.canny(frames.view(n, h, w, 3), 180.5, 60.25, out_edges=edges.view(n, h, w),
                  out_cond=cond.view(n, h, w, 3).permute(0, 3, 1, 2))
        torch.cuda.synchronize()
        assert np.array_equal(edges.view(n, h, w).cpu().numpy(), want), (f_off, e_off, c_off)
        assert torch.equal(cond.view(n, h, w, 3).permute(0, 3, 1, 2).cpu(), oc.canny_cond(want))
        assert _guards_intact(ebuf, e_off, edges.numel()) and _guards_intact(cbuf, c_off, cond.numel(), float("nan"))
        assert np.array_equal(frames.cpu().numpy(), frames_np.reshape(-1))


def test_canny_labels_within_one_frame_of_int32_max(ops):
    """The most 512 x 512 frames one call takes: pixel labels run up to INT32_MAX - 262143.  Frames, workspace and
    edges need about 10 bytes a pixel (21 GB); the GPU is shared, so the test runs only when that much is free."""
    h = w = 512
    n = (2 ** 31 - 2) // (h * w)
    lib = ops.lib
    assert lib.tf_canny_workspace(n, h, w) > 0 and lib.tf_canny_workspace(n + 1, h, w) == -1
    assert n * h * w > 2 ** 31 - 1 - h * w
    need = 10 * n * h * w + (1 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"{need / 2 ** 30:.1f} GiB needed, {free / 2 ** 30:.1f} GiB free")
    frame = gg.dense(h, w)
    want = torch.from_numpy(oc.canny(frame, 100, 500)).cuda()
    try:
        frames = torch.from_numpy(frame).cuda().expand(n, h, w, 3).contiguous()
        edges, _ = ops.canny(frames, 100, 500, cond=False)
        del frames
        bad = (edges != want).flatten(1).sum(1)
        torch.cuda.synchronize()
        wrong = bad.nonzero().flatten()
        assert wrong.numel() == 0, f"{wrong.numel()} of {n} frames differ, first {wrong[:8].tolist()}"
        print(f"{n} frames of {h} x {w}: {n * h * w} labels, INT32_MAX - {2 ** 31 - 1 - n * h * w}")
    finally:
        frames = edges = bad = None
        torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# graphs and the chain
# ---------------------------------------------------------------------------------------------------------------------
GRAPH_RESIZE_CASES = [((5, 4090), (3, 1021)), ((5, 4091), (3, 1021)), ((3, 7680), (2, 1920)),
                      ((3, 16378), (2, 4093)), ((3, 65536), (2, 16384))]


def test_graph_cases_take_every_horizontal_class():
    assert {fp.resize_h_class(fp.resize_layout(2, *s, *d)) for s, d in GRAPH_RESIZE_CASES} == set(fp.RESIZE_H_CLASSES)


@pytest.mark.parametrize("src,dst", GRAPH_RESIZE_CASES, ids=_ids(GRAPH_RESIZE_CASES))
def test_resize_graph_follows_new_content(ops, src, dst):
    (h_in, w_in), (h, w) = src, dst
    first, second = (_content("random", 2, h_in, w_in, seed=s) for s in (1, 2))
    inp = torch.from_numpy(first).cuda()
    tmp = torch.empty((2, h_in, w, 3), dtype=torch.uint8, device="cuda")
    out = torch.empty((2, h, w, 3), dtype=torch.uint8, device="cuda")
    ops.resize_frames(inp, (h, w), tmp=tmp, out=out)                      # warm-up: tables, shared-memory opt-in
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.resize_frames(inp, (h, w), tmp=tmp, out=out)
    for frames in (first, second):
        inp.copy_(torch.from_numpy(frames))
        out.fill_(7)
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), _pil(frames, h, w))


def test_canny_graph_follows_new_content(ops):
    rng = np.random.default_rng(4)
    first = np.stack([gg.make_frame("smooth", 512, 512, rng) for _ in range(2)])
    second = np.stack([gg.dense(512, 512), gg.serpentine(512, 512)])
    frames = torch.from_numpy(first).cuda()
    edges = torch.empty((2, 512, 512), dtype=torch.uint8, device="cuda")
    cond = torch.empty((2, 3, 512, 512), dtype=torch.float16, device="cuda", memory_format=torch.channels_last)
    ops.canny(frames, 100, 500, out_edges=edges, out_cond=cond)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.canny(frames, 100, 500, out_edges=edges, out_cond=cond)
    for content in (first, second):
        frames.copy_(torch.from_numpy(content))
        edges.fill_(7)
        cond.fill_(0.5)
        graph.replay()
        torch.cuda.synchronize()
        want = oc.canny_frames(content, 100, 500)
        assert np.array_equal(edges.cpu().numpy(), want)
        assert torch.equal(cond.cpu(), oc.canny_cond(want))


@pytest.mark.parametrize("size", [(512, 512), (384, 672)])
def test_1080p_frames_to_canny_cond_on_the_device(size):
    """40 frames at 1080p -> preprocess.resize_frames -> preprocess.canny_cond, all on the device, equal to PIL ->
    the Canny oracle -> the reference's conditioning expression on the host."""
    rng = np.random.default_rng(size[1])
    frames = np.stack([gg.make_frame("smooth", 1080, 1920, rng) for _ in range(40)])
    got = preprocess.canny_cond(preprocess.resize_frames(torch.from_numpy(frames).cuda(), size))
    torch.cuda.synchronize()
    want = oc.canny_cond(oc.canny_frames(_pil(frames, *size), 100, 200))
    assert got.is_cuda and got.shape == (40, 3, *size)
    assert torch.equal(got.cpu(), want)
