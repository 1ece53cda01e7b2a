"""GPU tier (-m gpu): tf_propagate bit for bit against `oracle.kernel_checks.propagate_exact` (numpy float32, equal to
`OracleOps.propagate` by tests/test_propagate_checks_cpu.py), and the NN field's order of NaN similarities.

Outputs are compared bit for bit, NaN with NaN by `isnan` (so +0 and -0 differ), and every output is a view into a
sentinel-filled buffer with guard bands, so an unwritten element or a write outside the output is seen.

* Every row width: dim 8 ... 2560 in steps of 8.  The kernel gives each thread one 16-byte column (dim / 8 of a
  row) and each 320-thread block 320 // (dim / 8) rows, so widths whose vector count does not divide 320 leave
  threads idle; S = 37 rows make the last block ragged.  Widths past 2560 and widths that are not a multiple of 8
  are refused before anything is launched.
* Every fp16 value: all 65 536 bit patterns as stream-a values, against permutations of them as stream-b values
  and residuals, for every weight of blend_weights(B), B in 2 ... 8 and 16, for w = 1 with a second keyframe
  (1 - w = 0, so 0 * inf is NaN) and for a frame without one: inf and NaN propagation, the residual add that
  overflows fp16, and round-to-nearest-even at fp16 midpoints of the fp32 blend.
* Index and frame-table extremes, frame counts around the 64-frame launch chunks, operands at odd offsets, and the
  SD levels at their real token counts.
* NN field: a zero token's unit row is NaN, and the reference's torch.argmax ranks a NaN similarity above every
  number, first NaN first: a zero pivot token wins every row, a zero frame token gets index 0.
"""
import math

import pytest
import torch

from oracle.kernel_checks import (bit_equal, check_nn_field, every_fp16_propagate_inputs, nn_argmax, nn_similarity,
                                  propagate_exact)
from tokenflow_b200 import ops as tf_ops
from tokenflow_b200.ops import blend_weights
from tokenflow_b200.tokenflow_utils import _default_frame_table

pytestmark = pytest.mark.gpu

INT_SENTINEL = -0x7f7f7f7f
GUARD = 256                     # elements on each side; keeps the 16-byte alignment the kernels require
BLEND_SIZES = (2, 3, 4, 5, 6, 7, 8, 16)
DTYPES = [torch.float16, torch.float32]


@pytest.fixture(scope="module")
def ops():
    return tf_ops.CudaOps()


class SentinelOutputs:
    """Stands in for the `torch.empty` that tokenflow_b200.ops allocates its outputs with: each output is a view
    into a larger buffer filled with a sentinel (`fill` for floating point, NaN unless set, INT_SENTINEL for
    int32)."""

    def __init__(self):
        self.allocs = []
        self.fill = float("nan")

    def empty(self, *size, dtype=None, device=None, **kwargs):
        if len(size) == 1 and isinstance(size[0], (tuple, list, torch.Size)):
            size = tuple(size[0])
        n = math.prod(size)
        buf = torch.empty(n + 2 * GUARD, dtype=dtype, device=device, **kwargs)
        fill = INT_SENTINEL if dtype == torch.int32 else self.fill
        buf.fill_(fill)
        view = buf[GUARD:GUARD + n].view(size)
        self.allocs.append((buf, view, fill))
        return view

    @staticmethod
    def is_sentinel(t, fill):
        return torch.isnan(t) if isinstance(fill, float) and math.isnan(fill) else t == fill

    def _find(self, out):
        torch.cuda.synchronize()
        matches = [(buf, view, fill) for buf, view, fill in self.allocs if view.data_ptr() == out.data_ptr()]
        assert len(matches) == 1, "not an output of this op"
        return matches[0]

    def check_guards(self, out):
        """The guard bands of `out`'s buffer still hold the sentinel: nothing was written outside the output."""
        buf, view, fill = self._find(out)
        assert self.is_sentinel(buf[:GUARD], fill).all(), "write before the start of the output"
        assert self.is_sentinel(buf[GUARD + view.numel():], fill).all(), "write past the end of the output"

    def check(self, out, unwritten=None):
        """`out` (the tensor an op allocated, or a view of it) is written everywhere except where the bool mask
        `unwritten` is set, which must still hold the sentinel; its guard bands are untouched."""
        buf, view, fill = self._find(out)
        s = self.is_sentinel(view, fill)
        expect = torch.zeros_like(s) if unwritten is None else unwritten.reshape(s.shape).to(s.device)
        assert not (s & ~expect).any(), f"{int((s & ~expect).sum())} output elements were not written"
        assert s[expect].all(), f"{int((~s & expect).sum())} elements that must stay unwritten were written"
        self.check_guards(out)


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


# ------------------------------------------------------------------------------------------------
# propagation
# ------------------------------------------------------------------------------------------------
def _on_gpu(case):
    return {k: v.cuda() if torch.is_tensor(v) else v for k, v in case.items()}


def _assert_bits(got, want, what=""):
    same = bit_equal(got, want)
    if not same.all():
        i = int((~same).flatten().nonzero()[0])
        g, w = got.detach().cpu().flatten()[i].item(), want.flatten()[i].item()
        raise AssertionError(f"{what}: {int((~same).sum())} of {same.numel()} elements differ from propagate_exact; "
                             f"first at flat index {i} of shape {tuple(want.shape)}: got {g!r}, want {w!r}")


def _check_propagate(ops, sentinel, case, out_dtype, what=""):
    """One call, written exactly over its output and equal to propagate_exact bit for bit (finite inputs)."""
    got = ops.propagate(**_on_gpu(case), out_dtype=out_dtype)
    assert got.dtype == out_dtype
    sentinel.check(got)
    _assert_bits(got, propagate_exact(**case, out_dtype=out_dtype), what)
    return got


def _random_case(kf_a, kf_b, w, S, dim, seed, K=None, idx=None):
    g = torch.Generator().manual_seed(seed)
    F = len(kf_a)
    K = K if K is not None else max(max(kf_a), max(kf_b)) + 1
    A = torch.randn(3, K, S, dim, generator=g).half()
    if idx is None:
        idx_a = torch.randint(0, S, (F, S), generator=g, dtype=torch.int32)
        idx_b = torch.randint(0, S, (F, S), generator=g, dtype=torch.int32)
    else:
        idx_a = torch.full((F, S), idx, dtype=torch.int32)
        idx_b = idx_a.clone()
    if max(kf_b) < 0:
        idx_b = None
    res = torch.randn(3 * F, S, dim, generator=g).half()
    return dict(A=A, idx_a=idx_a, idx_b=idx_b, kf_a=list(kf_a), kf_b=list(kf_b), w=list(w), residual=res)


# one frame without a second keyframe, one blended, one whose second keyframe is its first
MIXED = ([2, 1, 2], [-1, 0, 2], [1.0, blend_weights(3)[0], 0.6])


@pytest.mark.parametrize("dim", range(8, 2561, 8))
def test_propagate_every_row_width(ops, sentinel, dim):
    case = _random_case(*MIXED, S=37, dim=dim, seed=dim)
    for residual in (case["residual"], None):
        for out_dtype in DTYPES:
            _check_propagate(ops, sentinel, dict(case, residual=residual), out_dtype,
                             f"dim {dim} {out_dtype} residual={residual is not None}")


@pytest.mark.parametrize("dim,F,status", [(2568, 3, 3), (2568, 65, 3), (4096, 3, 3), (4, 3, 1), (12, 3, 1),
                                          (2564, 3, 1)])
def test_propagate_refuses_unsupported_row_widths(ops, dim, F, status):
    """Past 2560 a row has more 16-byte vectors than a block has threads (TF_ERR_UNSUPPORTED = 3); a width that is
    not a multiple of 8 has no 16-byte vectors (TF_ERR_INVALID_ARGUMENT = 1).  Nothing is launched."""
    A = torch.zeros(3, 2, 5, dim, dtype=torch.float16, device="cuda")
    idx = torch.zeros(F, 5, dtype=torch.int32, device="cuda")
    before = ops.launch_count()
    with pytest.raises(tf_ops.TokenflowB200Error, match=rf"status {status}\).*dim={dim}"):
        ops.propagate(A, idx, idx, [1] * F, [0] * F, [0.7] * F, None)
    torch.cuda.synchronize()
    assert ops.launch_count() == before


@pytest.fixture(scope="module")
def every_fp16_case():
    weights = [x for B in BLEND_SIZES for x in blend_weights(B)]
    return every_fp16_propagate_inputs(weights, generator=torch.Generator().manual_seed(0))


@pytest.mark.parametrize("with_residual", [True, False])
@pytest.mark.parametrize("out_dtype", DTYPES)
def test_propagate_every_fp16_value(ops, sentinel, every_fp16_case, out_dtype, with_residual):
    """NaN is a legitimate output here, so each call runs twice: into a NaN-filled buffer (an unwritten element
    whose exact value is not NaN differs) and into a 2.5-filled one (an unwritten element whose exact value is NaN
    differs)."""
    case = dict(every_fp16_case, residual=every_fp16_case["residual"] if with_residual else None)
    want = propagate_exact(**case, out_dtype=out_dtype)
    dev = _on_gpu(case)
    for fill in (float("nan"), 2.5):
        sentinel.fill = fill
        got = ops.propagate(**dev, out_dtype=out_dtype)
        sentinel.check_guards(got)
        _assert_bits(got, want, f"sentinel {fill}")
    assert torch.isnan(want).any() and torch.isinf(want).any()


EXTREMES = {
    "every_index_0": dict(kf_a=[2, 1, 2], kf_b=[-1, 0, 2], idx=0),
    "every_index_last": dict(kf_a=[2, 1, 2], kf_b=[-1, 0, 2], idx=-1),
    "one_keyframe": dict(kf_a=[0, 0, 0], kf_b=[-1, 0, -1]),
    "64_keyframes_last": dict(kf_a=[63, 63, 0, 63], kf_b=[-1, 62, 63, 63], K=64),
}


@pytest.mark.parametrize("out_dtype", DTYPES)
@pytest.mark.parametrize("name", sorted(EXTREMES))
def test_propagate_index_and_table_extremes(ops, sentinel, name, out_dtype):
    S, dim = 200, 72                       # 9 vectors per row: 35 rows per block, 5 threads idle
    e = dict(EXTREMES[name])
    idx = e.pop("idx", None)
    F = len(e["kf_a"])
    w = [0.55 + 0.05 * f for f in range(F)]
    case = _random_case(e["kf_a"], e["kf_b"], w, S, dim, seed=len(name), K=e.get("K"),
                        idx=None if idx is None else idx % S)
    _check_propagate(ops, sentinel, case, out_dtype, name)


@pytest.mark.parametrize("F", [63, 64, 65, 128, 129])
def test_propagate_frame_counts_across_launch_chunks(ops, sentinel, F):
    """64 frames per launch: every frame has its own weight and keyframes, so a table offset by a chunk shows."""
    K, S, dim = 5, 24, 40
    kf_a = [f % K for f in range(F)]
    kf_b = [-1 if f % 7 == 3 else (3 * f + 1) % K for f in range(F)]
    w = [0.25 + 0.5 * f / F for f in range(F)]
    assert len(set(w)) == F
    case = _random_case(kf_a, kf_b, w, S, dim, seed=F, K=K)
    for out_dtype in DTYPES:
        _check_propagate(ops, sentinel, case, out_dtype, f"F={F}")


@pytest.mark.parametrize("out_dtype", DTYPES)
def test_propagate_operands_at_odd_offsets(ops, sentinel, out_dtype):
    """The int32 indices are read in place from an odd int32 offset; A and the residual start at an odd fp16
    element offset (the wrapper copies them to aligned buffers)."""
    case = _random_case(*MIXED, S=100, dim=40, seed=11)

    def at_odd_offset(t):
        buf = torch.empty(t.numel() + 1, dtype=t.dtype, device="cuda")
        view = buf[1:].view(t.shape)
        view.copy_(t)
        return view

    dev = {k: at_odd_offset(v) if torch.is_tensor(v) else v for k, v in case.items()}
    assert dev["idx_a"].data_ptr() % 8 == 4 and dev["idx_b"].data_ptr() % 8 == 4
    assert dev["A"].data_ptr() % 16 == 2 and dev["residual"].data_ptr() % 16 == 2
    got = ops.propagate(**dev, out_dtype=out_dtype)
    sentinel.check(got)
    _assert_bits(got, propagate_exact(**case, out_dtype=out_dtype), "odd offsets")


@pytest.mark.parametrize("batch_idx", [0, 2])
@pytest.mark.parametrize("S,dim", [(4096, 320), (1024, 640), (256, 1280), (64, 1280)])
def test_propagate_sd_levels(ops, sentinel, S, dim, batch_idx):
    """The frame pass's call (tokenflow_utils `_tf_frames`): 8 frames of one batch against the keyframes of batches
    0 .. 2, the block's hidden states as the residual, fp16 output."""
    n_frames, K = 8, 3
    kf_a, kf_b, w = _default_frame_table(batch_idx, n_frames)
    g = torch.Generator(device="cuda").manual_seed(S + dim + batch_idx)
    kf = torch.randn(3, K, S, dim, generator=g, device="cuda").half()
    hidden = torch.randn(3 * n_frames, S, dim, generator=g, device="cuda").half()
    idx_a = torch.randint(0, S, (n_frames, S), generator=g, device="cuda", dtype=torch.int32)
    idx_b = torch.randint(0, S, (n_frames, S), generator=g, device="cuda", dtype=torch.int32) if batch_idx else None
    got = ops.propagate(kf, idx_a, idx_b, kf_a, kf_b, w, residual=hidden)
    assert got.dtype == torch.float16
    sentinel.check(got)
    _assert_bits(got, propagate_exact(kf, idx_a, idx_b, kf_a, kf_b, w, hidden, torch.float16), f"S={S} dim={dim}")


# ------------------------------------------------------------------------------------------------
# NN field: NaN similarities
# ------------------------------------------------------------------------------------------------
# zero tokens: (pivot tokens of keyframe 1, pivot tokens of keyframe 0, frame tokens of frame 1)
ZERO_TOKENS = {
    "zero_pivot_token": ([150], [], []),
    "zero_frame_token": ([], [], [77]),
    # tokens 21 and 130 are read by different threads of a row's quad (column % 8 = 5 and 2), 21 and 149 by the same
    "two_zero_pivots_two_threads": ([], [21, 130], []),
    "two_zero_pivots_one_thread": ([], [21, 149], []),
}


@pytest.mark.parametrize("case", sorted(ZERO_TOKENS))
@pytest.mark.parametrize("dim", [64, 640, 1280])
def test_nn_field_nan_similarities(ops, sentinel, dim, case):
    """dim 64 and 640 keep the token tile resident in shared memory, 1280 streams it.  S = 200: two key tiles, the
    second ragged."""
    S = 200
    kf_a, kf_b = [1, 1, 0], [-1, 0, 1]
    piv1, piv0, frame1 = ZERO_TOKENS[case]
    g = torch.Generator().manual_seed(dim)
    piv = torch.nn.functional.layer_norm(torch.randn(2, S, dim, generator=g), (dim,))
    x = piv[kf_a][:, torch.randperm(S, generator=g)] + 0.3 * torch.randn(3, S, dim, generator=g)
    piv[1, piv1] = 0
    piv[0, piv0] = 0
    x[1, frame1] = 0
    sentinel.fill = 2.5                    # the NaN rows below are the unit-row kernel's, not the sentinel's
    xu, pu = ops.unit_rows(x.cuda()), ops.unit_rows(piv.cuda())
    assert torch.equal(torch.isnan(xu).any(dim=-1).cpu(), (x == 0).all(dim=-1))
    assert torch.equal(torch.isnan(pu).any(dim=-1).cpu(), (piv == 0).all(dim=-1))

    idx_a, idx_b = ops.nn_field(xu, pu, kf_a, kf_b)
    sentinel.check(idx_a)
    sentinel.check(idx_b, unwritten=torch.tensor([b < 0 for b in kf_b]).view(3, 1).expand(3, S))
    check_nn_field(idx_a, idx_b, xu, pu, kf_a, kf_b)

    # the same indices stated outright, and the reference's own argmax (torch on CUDA) agreeing
    for f in range(3):
        for kf, idx in ((kf_a[f], idx_a), (kf_b[f], idx_b)):
            if kf < 0:
                continue
            sim = nn_similarity(xu[f], pu[kf])
            want = nn_argmax(sim)
            assert torch.equal(sim.argmax(dim=-1), want)
            zero_cols = piv1 if kf == 1 else piv0
            want_rows = torch.full((S,), min(zero_cols), dtype=torch.long) if zero_cols else want.cpu().clone()
            if f == 1:
                want_rows[frame1] = 0
            assert torch.equal(want.cpu(), want_rows)
            assert torch.equal(idx[f].long().cpu(), want_rows), (f, kf)
