"""GPU tier (-m gpu): every compiled variant of the attention and NN-field kernels at the shapes where tiled
kernels go wrong, against the calibrated checks of oracle/kernel_checks.py.

* Attention: every head-dim bucket of `dispatch()` in tf_ext_attn.cu (d rounded up to 16: 16 ... 128 with
  128-key tiles, 144 ... 192 with 64-key tiles; the paired kernel up to 64) at S below one key tile, a
  tile multiple and a tile multiple + 1, and S = 4, with n = 3 so the extended streams cross ragged slabs.
  The test IDs name the bucket (P<d rounded to 16>) and the kernel (pair / single).
* Logit-shift probe: every real logit near -25, so one leaked zero-filled padding key dominates its row.
* Negative-similarity probe: every real NN similarity below 0, so a padding column (similarity 0) would win.
* Sentinel outputs: the outputs `tokenflow_b200.ops` allocates are views into NaN- / -0x7f7f7f7f-filled
  buffers with guard bands, so an unwritten element, a write past either end, or a write to rows that
  must stay unwritten is seen.
"""
import math

import pytest
import torch

from oracle.kernel_checks import (check_ext_attn, check_nn_field, ext_attn_samples, logit_shift_probe,
                                  negative_similarity_probe, nn_similarity)
from oracle.oracle_ops import OracleOps
from tokenflow_b200 import ops as tf_ops

pytestmark = pytest.mark.gpu

INT_SENTINEL = -0x7f7f7f7f
GUARD = 256                     # elements on each side; keeps the 16-byte alignment the kernels require


@pytest.fixture(scope="module")
def ops():
    return tf_ops.CudaOps()


class SentinelOutputs:
    """Stands in for the `torch.empty` that tokenflow_b200.ops allocates its outputs with: each output is a view
    into a larger buffer filled with a sentinel (NaN for floating point, INT_SENTINEL for int32)."""

    def __init__(self):
        self.allocs = []

    def empty(self, *size, dtype=None, device=None, **kwargs):
        if len(size) == 1 and isinstance(size[0], (tuple, list, torch.Size)):
            size = tuple(size[0])
        n = math.prod(size)
        buf = torch.empty(n + 2 * GUARD, dtype=dtype, device=device, **kwargs)
        buf.fill_(INT_SENTINEL if dtype == torch.int32 else float("nan"))
        view = buf[GUARD:GUARD + n].view(size)
        self.allocs.append((buf, view))
        return view

    @staticmethod
    def is_sentinel(t):
        return t == INT_SENTINEL if t.dtype == torch.int32 else torch.isnan(t)

    def check(self, out, unwritten=None):
        """`out` (the tensor an op allocated, or a view of it) is written everywhere except where the bool mask
        `unwritten` is set, which must still hold the sentinel; its guard bands are untouched."""
        torch.cuda.synchronize()
        matches = [(buf, view) for buf, view in self.allocs if view.data_ptr() == out.data_ptr()]
        assert len(matches) == 1, "not an output of this op"
        buf, view = matches[0]
        s = self.is_sentinel(view)
        expect = torch.zeros_like(s) if unwritten is None else unwritten.reshape(s.shape).to(s.device)
        assert not (s & ~expect).any(), f"{int((s & ~expect).sum())} output elements were not written"
        assert s[expect].all(), f"{int((~s & expect).sum())} elements that must stay unwritten were written"
        assert self.is_sentinel(buf[:GUARD]).all(), "write before the start of the output"
        assert self.is_sentinel(buf[GUARD + view.numel():]).all(), "write past the end of the output"


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
# extended attention: every compiled variant
# ------------------------------------------------------------------------------------------------
SINGLE_D = [8, 24, 40, 56, 72, 96, 104, 112, 128, 136, 144, 160, 176, 192]
PAIRED_D = [16, 24, 40, 64]


def _block_n(d):
    return 128 if d <= 128 else 64


def _attn_cases():
    cases = []
    for d in sorted(set(SINGLE_D) | set(PAIRED_D)):
        N = _block_n(d)
        for S in (4, N - 28, 2 * N, 2 * N + 1):
            for inject in (False, True):
                kernel = "pair" if inject and d <= 64 else "single"
                for probe in (False, True):
                    cid = f"P{-(-d // 16) * 16}-d{d}-S{S}-{kernel}-{'inject' if inject else 'plain'}-" \
                          f"{'probe' if probe else 'random'}"
                    cases.append(pytest.param(d, S, inject, probe, id=cid))
    return cases


@pytest.mark.parametrize("d,S,inject,probe", _attn_cases())
def test_ext_attn_variant(ops, sentinel, d, S, inject, probe):
    n, heads = 3, 2
    dim = heads * d
    g = torch.Generator().manual_seed(1000 * d + S)
    q, k, v = (torch.randn(3 * n, S, dim, generator=g).half() for _ in range(3))
    scale = d ** -0.5
    if probe:
        logit_shift_probe(q, k, heads, scale, generator=g)
    q, k, v = q.cuda(), k.cuda(), v.cuda()
    table = ext_attn_samples(n, inject)
    # over a few keys the probe's softmax is near one-hot and |O| reaches |v| ~ 2.5, where the fp16 output
    # rounding alone is up to 1e-3 (the fp16-P emulation errs by 1.07e-3 at d = 128, S = 4): there the fixed
    # ceiling scales with |O| as in test_ext_attn_peaky_softmax
    rtol = 1.5e-3 if probe else 0.0

    got = ops.ext_attn(q, k, v, heads, scale, inject)
    sentinel.check(got)
    st = check_ext_attn(got, q, k, v, table, heads, scale, rtol=rtol)
    print(f"ext_attn d={d} S={S} inject={inject} probe={probe}: rel {st['rel']:.3g} emulation {st['rel_emu']:.3g} "
          f"ratio {st['ratio']:.3f} error-model use {st['bound_use']:.2f}")

    # a query-row range that runs past S (multi-GPU token split): rows past S stay unwritten
    row0 = 128 if S > 128 else 0
    nrows = S if S > 128 else S + 37
    rows = ops.ext_attn_table(q, k, v, table, heads, scale, row0=row0, nrows=nrows)
    past = torch.zeros(rows.shape, dtype=torch.bool)
    past[:, S - row0:] = True
    sentinel.check(rows, unwritten=past)
    check_ext_attn(rows, q, k, v, table, heads, scale, row0=row0, nrows=nrows, rtol=rtol)


@pytest.mark.parametrize("inject", [False, True])
def test_ext_attn_head_dim_over_192_is_an_error(ops, inject):
    """d = 200 has no compiled variant: the call raises before anything is launched."""
    q = torch.zeros(6, 16, 200, dtype=torch.float16, device="cuda")
    before = ops.launch_count()
    with pytest.raises(tf_ops.TokenflowB200Error, match="head dim 200"):
        ops.ext_attn(q, q, q, 1, 200 ** -0.5, inject)
    assert ops.launch_count() == before


# ------------------------------------------------------------------------------------------------
# NN field: the padding-column guard on both A paths (resident up to dim 640, streamed above)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [64, 100, 144, 576])
@pytest.mark.parametrize("dim", [320, 640, 648, 768, 1280])
def test_nn_field_negative_similarity_probe(ops, sentinel, dim, S):
    F, K = 3, 2
    kf_a, kf_b = [0, 1, 1], [-1, 0, -1]
    x, piv = negative_similarity_probe(F, K, S, dim, kf_a, generator=torch.Generator().manual_seed(dim + S))
    xu, pu = ops.unit_rows(x.cuda()), ops.unit_rows(piv.cuda())
    assert (nn_similarity(xu.view(-1, dim), pu.view(-1, dim)).float() < 0).all()
    idx_a, idx_b = ops.nn_field(xu, pu, kf_a, kf_b)
    sentinel.check(idx_a)
    no_b = torch.tensor([b < 0 for b in kf_b]).view(F, 1).expand(F, S)
    sentinel.check(idx_b, unwritten=no_b)
    check_nn_field(idx_a, idx_b, xu, pu, kf_a, kf_b)


def _video_like(F, K, S, dim, kf, seed, noise=0.3):
    g = torch.Generator().manual_seed(seed)
    piv = torch.nn.functional.layer_norm(torch.randn(K, S, dim, generator=g), (dim,))
    x = torch.stack([piv[kf[f]][torch.randperm(S, generator=g)] for f in range(F)])
    return (x + noise * torch.randn(F, S, dim, generator=g)).cuda(), piv.cuda()


def _frame_table_cases():
    mixed = ([0, 1, 3, 3, 2, 1], [-1, 0, -1, 2, 1, -1])
    # 130 frames (three launches of at most 64): the second launch has no second keyframe at all, the third
    # only some
    kf_a = [(f // 8) % 5 for f in range(130)]
    kf_b = [-1 if 64 <= f < 128 or f % 8 == 0 else max(0, kf_a[f] - 1) for f in range(130)]
    return [pytest.param(*mixed, 200, 320, id="mixed-6"), pytest.param(kf_a, kf_b, 144, 648, id="chunks-130")]


@pytest.mark.parametrize("kf_a,kf_b,S,dim", _frame_table_cases())
def test_nn_field_frame_tables(ops, sentinel, kf_a, kf_b, S, dim):
    F, K = len(kf_a), max(kf_a) + 1
    x, piv = _video_like(F, K, S, dim, kf_a, seed=F)
    xu, pu = ops.unit_rows(x), ops.unit_rows(piv)
    idx_a, idx_b = ops.nn_field(xu, pu, kf_a, kf_b)
    sentinel.check(idx_a)
    sentinel.check(idx_b, unwritten=torch.tensor([b < 0 for b in kf_b]).view(F, 1).expand(F, S))
    check_nn_field(idx_a, idx_b, xu, pu, kf_a, kf_b)


# ------------------------------------------------------------------------------------------------
# sentinel outputs of the remaining ops
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,dim", [(1, 8), (77, 40), (1000, 1280)])
def test_unit_rows_writes_exactly_its_output(ops, sentinel, rows, dim):
    x = torch.randn(rows, dim, device="cuda") * 3 + 0.5
    want = (x / x.norm(dim=-1, keepdim=True)).half()
    for src in (x, x.half()):
        got = ops.unit_rows(src)
        sentinel.check(got)
        assert (got.float() - want.float()).abs().max().item() < 2e-3


@pytest.mark.parametrize("rows,dim", [(3, 8), (100, 40), (512, 1280)])
def test_layernorm_unit_rows_writes_exactly_its_output(ops, sentinel, rows, dim):
    norm = torch.nn.LayerNorm(dim).cuda().half()
    x = (torch.randn(rows, dim, device="cuda") * 2 + 0.3).half()
    got = ops.layernorm_unit_rows(x, norm)
    sentinel.check(got)
    y = torch.nn.functional.layer_norm(x.float(), (dim,), norm.weight.float(), norm.bias.float(), norm.eps)
    assert (got.float() - (y / y.norm(dim=-1, keepdim=True))).abs().max().item() <= 1e-3


@pytest.mark.parametrize("b,S,dim,n_unit", [(3, 64, 40, 1), (4, 100, 640, 4), (2, 33, 1280, 0)])
def test_layernorm_rows_writes_exactly_its_outputs(ops, sentinel, b, S, dim, n_unit):
    norm = torch.nn.LayerNorm(dim).cuda().half()
    x = (torch.randn(b, S, dim, device="cuda") * 2 + 0.3).half()
    y, unit = ops.layernorm_rows(x, norm, n_unit)
    sentinel.check(y)
    y_ref = torch.nn.functional.layer_norm(x.float(), (dim,), norm.weight.float(), norm.bias.float(), norm.eps)
    assert (y.float() - y_ref).abs().max().item() < 4e-3
    if n_unit:
        sentinel.check(unit)
        u_ref = y_ref[:n_unit] / y_ref[:n_unit].norm(dim=-1, keepdim=True)
        assert (unit.float() - u_ref).abs().max().item() <= 1e-3
    else:
        assert unit is None


@pytest.mark.parametrize("out_dtype", [torch.float16, torch.float32])
def test_propagate_writes_exactly_its_output(ops, sentinel, out_dtype):
    F, K, S, dim = 6, 4, 100, 40
    A = torch.randn(3, K, S, dim, device="cuda").half()
    kf_a, kf_b = [0, 1, 3, 3, 2, 1], [-1, 0, -1, 2, 1, -1]
    w = [1.0, 0.3, 1.0, 0.6, 0.45, 1.0]
    idx_a = torch.randint(0, S, (F, S), device="cuda", dtype=torch.int32)
    idx_b = torch.randint(0, S, (F, S), device="cuda", dtype=torch.int32)
    res = torch.randn(3 * F, S, dim, device="cuda").half()
    got = ops.propagate(A, idx_a, idx_b, kf_a, kf_b, w, res, out_dtype=out_dtype)
    sentinel.check(got)
    want = OracleOps().propagate(A, idx_a, idx_b, kf_a, kf_b, w, res)
    assert torch.equal(got, want.to(out_dtype))
