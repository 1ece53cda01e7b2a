"""GPU tier (-m gpu): `tf_canny_u8` equals OpenCV's Canny byte for byte.

* every case of tests/golden/canny.pt (cv2's own outputs) and the numpy restatement oracle/canny.py, from 1 x 1 to
  384 x 672 and 512 x 512, 1 and 40 frames, sizes that are no multiple of the 32 x 16 tile;
* the serpentine probe: one band winding over the whole frame, weak everywhere but at its start, so hysteresis must
  cross every tile (the oracle's chain is checked to span the frame);
* a workspace filled with garbage and outputs inside sentinel guard bands: nothing outside the outputs is written;
* `cond_f16` equals the reference's get_canny_cond expression on the edges, and `preprocess.canny_cond` returns it;
* a captured CUDA graph of the call replays to the same bytes.
"""
import numpy as np
import pytest
import torch

from oracle import canny as oc
from oracle import gen_canny_golden as gg
from tokenflow_b200 import ops as tf_ops
from tokenflow_b200 import preprocess

pytestmark = pytest.mark.gpu

GUARD = 4096


@pytest.fixture(scope="module")
def ops():
    return tf_ops.CudaOps()


def _canny(ops, frames_np, low, high):
    e, c = ops.canny(torch.from_numpy(frames_np).cuda(), low, high)
    torch.cuda.synchronize()
    return e.cpu().numpy(), c


@pytest.mark.parametrize("name", list(gg.CASES))
def test_golden_cases(ops, name):
    gold = torch.load(gg.GOLDEN, weights_only=False)[name]
    kind, n, h, w, low, high, _ = gg.CASES[name]
    frames = gg.case_frames(name)
    want = gg.unpack(gold["edges_bits"].numpy(), (n, h, w))
    got, cond = _canny(ops, frames, low, high)
    assert np.array_equal(got, want), f"{name}: {(got != want).sum()} of {got.size} pixels differ"
    assert np.array_equal(got, oc.canny_frames(frames, low, high))
    assert torch.equal(cond.cpu(), oc.canny_cond(want))
    assert cond.is_contiguous(memory_format=torch.channels_last)


@pytest.mark.parametrize("n,h,w", [(1, 31, 17), (1, 33, 65), (40, 45, 77), (40, 64, 64), (1, 1, 300), (1, 300, 1)])
@pytest.mark.parametrize("kind", ["noise", "smooth", "lines"])
def test_random_sizes_equal_oracle(ops, n, h, w, kind):
    rng = np.random.default_rng(n * 7919 + h * 31 + w)
    frames = np.stack([gg.make_frame(kind, h, w, rng) for _ in range(n)])
    for low, high in [(100, 200), (220.7, 40.2)]:
        got, _ = _canny(ops, frames, low, high)
        assert np.array_equal(got, oc.canny_frames(frames, low, high)), (low, high)


@pytest.mark.parametrize("h,w", [(131, 97), (384, 672), (512, 512)])
def test_serpentine_crosses_every_tile(ops, h, w):
    img = gg.serpentine(h, w)
    want = oc.canny(img, 100, 500)
    cls = oc.classes(img, 100, 500)
    (y0, y1), (x0, x1) = oc.chain_span(want, tuple(np.argwhere(cls == 2)[0]))
    assert y0 <= 3 and y1 >= h - 16 and x0 <= 3 and x1 >= w - 4          # the oracle's chain spans the frame
    frames = np.stack([img, img[::-1].copy(), img[:, ::-1].copy()])        # the strong start in other corners
    got, _ = _canny(ops, frames, 100, 500)
    assert np.array_equal(got, oc.canny_frames(frames, 100, 500))


def test_garbage_workspace_and_guard_bands(ops):
    lib = ops.lib
    frames_np = gg.case_frames("smooth_3x97x131_swapped")
    n, h, w, _ = frames_np.shape
    frames = torch.from_numpy(frames_np).cuda()
    need = int(lib.tf_canny_workspace(n, h, w))
    g = torch.Generator(device="cuda").manual_seed(3)
    ws = torch.randint(0, 256, (need + 2 * GUARD,), dtype=torch.uint8, device="cuda", generator=g)
    ws_before = ws.clone()
    eb = torch.full((n * h * w + 2 * GUARD,), 0x5A, dtype=torch.uint8, device="cuda")
    cb = torch.full((3 * n * h * w + 2 * GUARD,), float("nan"), dtype=torch.float16, device="cuda")
    st = lib.tf_canny_u8(frames.data_ptr(), n, h, w, 180.5, 60.25, ws[GUARD:].data_ptr(), need,
                         eb[GUARD:].data_ptr(), cb[GUARD:].data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert st == 0, lib.tf_last_error()
    torch.cuda.synchronize()
    edges = eb[GUARD:GUARD + n * h * w].view(n, h, w).cpu().numpy()
    want = oc.canny_frames(frames_np, 180.5, 60.25)
    assert np.array_equal(edges, want)
    cond = cb[GUARD:GUARD + 3 * n * h * w].view(n, h, w, 3).permute(0, 3, 1, 2).cpu()
    assert torch.equal(cond, oc.canny_cond(want))
    assert bool((eb[:GUARD] == 0x5A).all()) and bool((eb[GUARD + n * h * w:] == 0x5A).all())
    assert bool(cb[:GUARD].isnan().all()) and bool(cb[GUARD + 3 * n * h * w:].isnan().all())
    assert torch.equal(ws[:GUARD], ws_before[:GUARD]) and torch.equal(ws[GUARD + need:], ws_before[GUARD + need:])
    # either output alone
    e_only, c_none = ops.canny(frames, 180.5, 60.25, cond=False)
    assert c_none is None and np.array_equal(e_only.cpu().numpy(), want)
    e_none, c_only = ops.canny(frames, 180.5, 60.25, edges=False)
    assert e_none is None and torch.equal(c_only.cpu(), oc.canny_cond(want))


def test_canny_cond_public_function(ops):
    frames_np = gg.case_frames("smooth_40x64x96")
    got = preprocess.canny_cond(torch.from_numpy(frames_np).cuda())
    assert got.shape == (40, 3, 64, 96) and got.dtype == torch.float16 and got.is_cuda
    assert torch.equal(got.cpu(), oc.canny_cond(oc.canny_frames(frames_np, 100, 200)))


def test_graph_replay(ops):
    frames_np = gg.case_frames("smooth_2x384x672")
    frames = torch.from_numpy(frames_np).cuda()
    edges = torch.empty((2, 384, 672), dtype=torch.uint8, device="cuda")
    cond = torch.empty((2, 3, 384, 672), dtype=torch.float16, device="cuda", memory_format=torch.channels_last)
    ops.canny(frames, out_edges=edges, out_cond=cond)                      # warm-up
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.canny(frames, out_edges=edges, out_cond=cond)
    edges.fill_(7)
    cond.fill_(0.5)
    graph.replay()
    torch.cuda.synchronize()
    want = oc.canny_frames(frames_np, 100, 200)
    assert np.array_equal(edges.cpu().numpy(), want)
    assert torch.equal(cond.cpu(), oc.canny_cond(want))
