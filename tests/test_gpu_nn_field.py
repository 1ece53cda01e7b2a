"""GPU tier (-m gpu): tf_nn_field index for index against `oracle.kernel_checks.nn_field_exact`, on operands whose
similarities the tensor core computes exactly in any accumulation order (`exact_similarity_probe`,
`every_fp16_similarity_probe`).  Every index has one right answer: no tie class, no allowance.

Outputs are views into sentinel-filled buffers with guard bands, so an unwritten index or a write outside the output
is seen; the idx_b rows of frames without a second keyframe must stay unwritten.  Every case runs twice and the two
launches must give identical indices.

* Every row width: dim 8 ... 2560 in steps of 8, and 4096.  The kernel keeps the token tile resident in shared memory
  up to dim 640 (its B-stage count falls as the number of 64-channel chunks grows) and streams it with the keyframe
  tiles above; the last chunk is partial unless dim is a multiple of 64.  S = 200 makes both the token tile and the
  key tile partial; F = 6 frames with a mixed keyframe table, K = 3.  A NaN pivot token (a zero token's unit row) in
  the last key tile and a NaN frame token check the NaN rule at every width.
* Token counts 1 ... 1000 at dims 64, 640 and 648, and the UNet levels at their real token counts.
* Every fp16 similarity: 65 536 keyframe tokens carrying every fp16 bit pattern.
* Frame counts around the 64-frame launch chunks, and operands at odd element offsets.
"""
import math

import pytest
import torch

from oracle.kernel_checks import every_fp16_similarity_probe, exact_similarity_probe, nn_field_exact
from tokenflow_b200 import ops as tf_ops

pytestmark = pytest.mark.gpu

INT_SENTINEL = -0x7f7f7f7f
GUARD = 256                     # int32 elements on each side of an output

KF_A, KF_B = [0, 1, 1, 2, 0, 1], [-1, 0, 2, -1, 1, -1]
NAN_PIVOT = (2, 141)            # keyframe 2, token 141: last key tile, thread 2 of the row's merge
NAN_FRAME = (1, 77)


@pytest.fixture(scope="module")
def ops():
    return tf_ops.CudaOps()


class SentinelOutputs:
    """Stands in for the `torch.empty` that tokenflow_b200.ops allocates its outputs with: each int32 output is a view
    into a larger buffer filled with INT_SENTINEL."""

    def __init__(self):
        self.allocs = []

    def empty(self, *size, dtype=None, device=None, **kwargs):
        if len(size) == 1 and isinstance(size[0], (tuple, list, torch.Size)):
            size = tuple(size[0])
        assert dtype == torch.int32, dtype
        n = math.prod(size)
        buf = torch.full((n + 2 * GUARD,), INT_SENTINEL, dtype=dtype, device=device, **kwargs)
        view = buf[GUARD:GUARD + n].view(size)
        self.allocs.append((buf, view))
        return view

    def check(self, out, unwritten=None):
        """`out` is written everywhere except where the bool mask `unwritten` is set, which still holds the
        sentinel, and its guard bands are untouched."""
        torch.cuda.synchronize()
        (buf, view), = [(b, v) for b, v in self.allocs if v.data_ptr() == out.data_ptr()]
        s = (view == INT_SENTINEL).cpu()
        expect = torch.zeros_like(s) if unwritten is None else unwritten.reshape(s.shape)
        assert not (s & ~expect).any(), f"{int((s & ~expect).sum())} indices were not written"
        assert s[expect].all(), f"{int((~s & expect).sum())} indices of frames without a second keyframe were written"
        assert (buf[:GUARD] == INT_SENTINEL).all(), "write before the start of the output"
        assert (buf[GUARD + view.numel():] == INT_SENTINEL).all(), "write past the end of the output"


class _TorchWithSentinelEmpty:
    def __init__(self, sentinel):
        self._sentinel = sentinel

    def __getattr__(self, name):
        return getattr(torch, name)

    def empty(self, *size, **kwargs):
        return self._sentinel.empty(*size, **kwargs)


@pytest.fixture
def sentinel(monkeypatch):
    s = SentinelOutputs()
    monkeypatch.setattr(tf_ops, "torch", _TorchWithSentinelEmpty(s))
    return s


def _assert_indices(got, want, what, cases=None, proto=None, kf_a=None, kf_b=None):
    got = got.cpu()
    bad = got != want
    if not bad.any():
        return
    f, r = (int(v) for v in bad.nonzero()[0])
    where = ""
    if cases is not None:
        kf = (kf_a if "idx_a" in what else kf_b)[f]
        names = [name for k, p, name, _, _ in cases if k == kf and p == int(proto[f, r])]
        where = f" (prototype {int(proto[f, r])}, probe case {names or 'filler'})"
    raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} indices differ from the exact expectation; first "
                         f"at frame {f} token {r}: got {int(got[f, r])}, want {int(want[f, r])}{where}")


def _run(ops, sentinel, x, piv, kf_a, kf_b, what, probe=None):
    """Two launches into sentinel buffers; both equal to nn_field_exact index for index."""
    F, S, _ = x.shape
    want_a, want_b = nn_field_exact(x, piv, kf_a, kf_b)
    xd, pd = x.cuda(), piv.cuda()
    no_b = torch.tensor([b < 0 for b in kf_b]).view(F, 1).expand(F, S)
    first = None
    for launch in range(2):
        idx_a, idx_b = ops.nn_field(xd, pd, kf_a, kf_b)
        sentinel.check(idx_a)
        if want_b is None:
            assert idx_b is None
        else:
            sentinel.check(idx_b, unwritten=no_b)
        extra = {} if probe is None else dict(cases=probe["cases"], proto=probe["proto"], kf_a=kf_a, kf_b=kf_b)
        _assert_indices(idx_a, want_a, f"{what} idx_a", **extra)
        if want_b is not None:
            got_b = torch.where(no_b, torch.full_like(want_b, -1), idx_b.cpu())
            _assert_indices(got_b, want_b, f"{what} idx_b", **extra)
        both = (idx_a.cpu(), None if idx_b is None else idx_b.cpu())
        if first is None:
            first = both
        else:
            assert torch.equal(both[0], first[0]) and (both[1] is None or torch.equal(both[1], first[1])), \
                f"{what}: the second launch gave other indices"
    return first


def _probe(F, K, S, dim, seed, nan_tokens=False):
    pr = exact_similarity_probe(F, K, S, dim, generator=torch.Generator().manual_seed(seed))
    if nan_tokens:
        pr["piv"][NAN_PIVOT] = float("nan")
        pr["x"][NAN_FRAME] = float("nan")
    return pr


@pytest.mark.parametrize("dim", list(range(8, 2561, 8)) + [4096])
def test_nn_field_exact_every_row_width(ops, sentinel, dim):
    pr = _probe(len(KF_A), 3, 200, dim, seed=dim, nan_tokens=True)
    idx_a, idx_b = _run(ops, sentinel, pr["x"], pr["piv"], KF_A, KF_B, f"dim {dim}", pr)
    assert (idx_b[2] == NAN_PIVOT[1]).all() and (idx_a[3] == NAN_PIVOT[1]).all()
    assert idx_a[NAN_FRAME] == 0 and idx_b[NAN_FRAME] == 0


@pytest.mark.parametrize("S", [1, 2, 7, 8, 9, 127, 128, 129, 255, 256, 257, 1000])
@pytest.mark.parametrize("dim", [64, 640, 648])
def test_nn_field_exact_token_counts(ops, sentinel, dim, S):
    pr = _probe(len(KF_A), 3, S, dim, seed=S * 7 + dim)
    _run(ops, sentinel, pr["x"], pr["piv"], KF_A, KF_B, f"S {S} dim {dim}", pr)


# (tokens, dim) of the four UNet levels: SD1.5 at 512 x 512, SD2.1 at 768 x 768, and a 384 x 672 video (48 x 84 latents)
SD_LEVELS = {
    "sd15": [(4096, 320), (1024, 640), (256, 1280), (64, 1280)],
    "sd21": [(9216, 320), (2304, 640), (576, 1280), (144, 1280)],
    "48x84": [(4032, 320), (1008, 640), (252, 1280), (66, 1280)],
}


@pytest.mark.parametrize("S,dim", [pytest.param(S, d, id=f"{name}-{S}x{d}") for name, lv in SD_LEVELS.items()
                                   for S, d in lv])
def test_nn_field_exact_unet_levels(ops, sentinel, S, dim):
    pr = _probe(len(KF_A), 3, S, dim, seed=S + dim)
    _run(ops, sentinel, pr["x"], pr["piv"], KF_A, KF_B, f"S {S} dim {dim}", pr)


def test_nn_field_every_fp16_similarity(ops, sentinel):
    pr = every_fp16_similarity_probe(generator=torch.Generator().manual_seed(0))
    _run(ops, sentinel, pr["x"], pr["piv"], pr["kf_a"], pr["kf_b"], "every fp16 similarity")


@pytest.mark.parametrize("F", [63, 64, 65, 129])
def test_nn_field_frame_counts_across_launch_chunks(ops, sentinel, F):
    """64 frames per launch: every frame has its own keyframes and its own row order, so a frame table or an operand
    offset by a chunk shows."""
    K, S, dim = 3, 136, 72
    kf_a = [f % K for f in range(F)]
    kf_b = [-1 if f % 5 == 2 else (f // 3 + 1) % K for f in range(F)]
    pr = _probe(F, K, S, dim, seed=F)
    _run(ops, sentinel, pr["x"], pr["piv"], kf_a, kf_b, f"F {F}", pr)


def test_nn_field_operands_at_odd_offsets(ops, sentinel):
    """Both operands start at an odd fp16 element offset (CudaOps.nn_field copies them to aligned buffers)."""
    pr = _probe(len(KF_A), 3, 200, 136, seed=5)
    want = nn_field_exact(pr["x"], pr["piv"], KF_A, KF_B)

    def at_odd_offset(t):
        buf = torch.empty(t.numel() + 1, dtype=t.dtype, device="cuda")
        view = buf[1:].view(t.shape)
        view.copy_(t)
        return view

    xd, pd = at_odd_offset(pr["x"]), at_odd_offset(pr["piv"])
    assert xd.data_ptr() % 16 == 2 and pd.data_ptr() % 16 == 2
    idx_a, idx_b = ops.nn_field(xd, pd, KF_A, KF_B)
    sentinel.check(idx_a)
    no_b = torch.tensor([b < 0 for b in KF_B]).view(-1, 1).expand(len(KF_B), 200)
    sentinel.check(idx_b, unwritten=no_b)
    _assert_indices(idx_a, want[0], "odd offsets idx_a")
    _assert_indices(torch.where(no_b, torch.full_like(want[1], -1), idx_b.cpu()), want[1], "odd offsets idx_b")
