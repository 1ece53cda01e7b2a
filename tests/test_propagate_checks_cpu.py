"""CPU tier: `oracle.kernel_checks.propagate_exact`, the numpy float32 restatement of tf_propagate that
tests/test_gpu_propagate.py compares the kernel with bit for bit, equals `OracleOps.propagate` (torch, written from
the same reference lines) on random rows and on every fp16 bit pattern, so the GPU tests rest on two independent
statements of the reference.  It also differs from the two likeliest wrong arithmetics on the every-pattern inputs,
so a kernel that computed either would fail there."""
import numpy as np
import pytest
import torch

from oracle.kernel_checks import bit_equal, every_fp16_propagate_inputs, propagate_exact
from oracle.oracle_ops import OracleOps
from tokenflow_b200.ops import blend_weights

BLEND_SIZES = (2, 3, 4, 5, 6, 7, 8, 16)


def _every_fp16_case(seed=0):
    weights = [x for B in BLEND_SIZES for x in blend_weights(B)]
    return every_fp16_propagate_inputs(weights, generator=torch.Generator().manual_seed(seed))


def _random_case(kf_a, kf_b, w, with_residual, S=40, dim=24, seed=0):
    g = torch.Generator().manual_seed(seed)
    F, K = len(kf_a), max(max(kf_a), max(kf_b)) + 1
    A = torch.randn(3, K, S, dim, generator=g).half()
    idx_a = torch.randint(0, S, (F, S), generator=g, dtype=torch.int32)
    idx_b = torch.randint(0, S, (F, S), generator=g, dtype=torch.int32) if max(kf_b) >= 0 else None
    res = torch.randn(3 * F, S, dim, generator=g).half() if with_residual else None
    return dict(A=A, idx_a=idx_a, idx_b=idx_b, kf_a=kf_a, kf_b=kf_b, w=w, residual=res)


def _assert_bits(got, want, what):
    same = bit_equal(got, want)
    assert same.all(), f"{what}: {int((~same).sum())} of {same.numel()} elements differ"


def _assert_equals_oracle(case):
    oracle = OracleOps().propagate(**case)
    # fp16 output: the reference expression rounded once, whatever dtype it promoted to
    _assert_bits(propagate_exact(**case, out_dtype=torch.float16), oracle.half(), "fp16 output")
    exact32 = propagate_exact(**case, out_dtype=torch.float32)
    if oracle.dtype == torch.float32 or case["residual"] is None:
        _assert_bits(exact32, oracle.float(), "fp32 output")
    else:
        # no frame blended: the reference stays in fp16 (an fp32 add rounded once); the kernel's fp32 output keeps
        # the sum unrounded, so only its fp16 rounding is the reference's value
        assert oracle.dtype == torch.float16
        _assert_bits(exact32.half(), oracle, "fp32 output rounded to fp16")


TABLES = {
    "unblended": ([0, 2, 1], [-1, -1, -1], [1.0, 1.0, 1.0]),
    "blended": ([2, 2, 2, 2], [1, 1, 1, 1], blend_weights(4)),
    "mixed": ([2, 1, 2], [-1, 0, 2], [1.0, blend_weights(3)[0], 0.6]),
    "w1_second_keyframe": ([1, 1], [0, 0], [1.0, 0.0]),
}


@pytest.mark.parametrize("with_residual", [False, True])
@pytest.mark.parametrize("table", sorted(TABLES))
def test_propagate_exact_equals_oracle_ops_on_random_rows(table, with_residual):
    _assert_equals_oracle(_random_case(*TABLES[table], with_residual, seed=len(table)))


@pytest.mark.parametrize("with_residual", [False, True])
def test_propagate_exact_equals_oracle_ops_on_every_fp16_value(with_residual):
    case = _every_fp16_case()
    if not with_residual:
        case["residual"] = None
    _assert_equals_oracle(case)
    # the unblended frame alone: the reference's fp16 + fp16 residual add
    last = dict(case, idx_a=case["idx_a"][-1:], idx_b=None, kf_a=case["kf_a"][-1:], kf_b=[-1], w=[1.0],
                residual=None if case["residual"] is None else case["residual"].view(3, -1, 256, 256)[:, -1])
    _assert_equals_oracle(last)


def test_every_fp16_inputs_cover_every_pattern_and_the_special_sums():
    case = _every_fp16_case()
    A, res = case["A"], case["residual"]
    F = len(case["kf_a"])
    for s in range(3):
        for slab in (A[s, 0], A[s, 1]):
            assert torch.unique(slab.view(torch.int16)).numel() == 65536
    assert torch.equal(A[0, 1].reshape(-1).view(torch.int16), torch.arange(-32768, 32768, dtype=torch.int16))
    assert res.shape == (3 * F, 256, 256) and case["w"][-2:] == [1.0, 1.0] and case["kf_b"][-2:] == [0, -1]
    out = propagate_exact(**case, out_dtype=torch.float16).float()
    a = A[:, 1].float().unsqueeze(1)                                   # identity indices: out[s, f] sees A[s, 1]
    r = res.view(3, F, 256, 256).float()
    finite_in = torch.isfinite(a) & torch.isfinite(r)
    assert (torch.isinf(out.view(3, F, 256, 256)) & finite_in).any(), "no residual add overflows fp16"
    w1 = out.view(3, F, 256, 256)[:, -2]                               # w = 1 with a second keyframe
    assert (torch.isnan(w1) & torch.isfinite(A[:, 1].float()) & torch.isfinite(r[:, -2])).any(), \
        "no 0 * inf from the second keyframe"


def _wrong_propagate(case, out_dtype, mistake):
    """propagate_exact with one arithmetic mistake: "fma" fuses w * a into the add (one rounding),
    "round_blend" rounds the blend to fp16 before the residual is added."""
    a16 = case["A"].numpy()
    F = len(case["kf_a"])
    ia, ib = case["idx_a"].long().numpy(), case["idx_b"].long().numpy()
    out = np.empty((3, F) + a16.shape[2:], dtype=np.float32)
    with np.errstate(all="ignore"):
        for f in range(F):
            a = a16[:, case["kf_a"][f]][:, ia[f]].astype(np.float32)
            if case["kf_b"][f] >= 0:
                wf = np.float32(case["w"][f])
                b = a16[:, case["kf_b"][f]][:, ib[f]].astype(np.float32)
                if mistake == "fma":
                    a = (np.float64(wf) * a.astype(np.float64) + ((np.float32(1) - wf) * b)).astype(np.float32)
                else:
                    a = wf * a + (np.float32(1) - wf) * b
            if mistake == "round_blend":
                a = a.astype(np.float16).astype(np.float32)
            out[:, f] = a
        out += case["residual"].numpy().reshape(out.shape).astype(np.float32)
        return torch.from_numpy(out.reshape(3 * F, *out.shape[2:]).astype(
            {torch.float16: np.float16, torch.float32: np.float32}[out_dtype]))


@pytest.mark.parametrize("out_dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("mistake", ["fma", "round_blend"])
def test_every_fp16_value_inputs_tell_wrong_arithmetic_apart(mistake, out_dtype):
    case = _every_fp16_case()
    want = propagate_exact(**case, out_dtype=out_dtype)
    same = bit_equal(_wrong_propagate(case, out_dtype, mistake), want)
    assert not same.all()
    print(f"{mistake} {out_dtype}: {int((~same).sum())} of {same.numel()} elements differ")
