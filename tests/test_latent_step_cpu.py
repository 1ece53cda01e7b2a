"""CPU tier: the numpy restatement of the latent updates (oracle/latent_step.py) can tell plausible wrong kernels
apart.

* Planted variants.  A thread-by-thread restatement of tf_cfg_ddim with one deliberate change each (an FMA-contracted
  final sum, a true division by sqrt(alpha_t), the fp32 reciprocal of the fp32 sqrt(alpha_t), an unrounded c - u or
  g * d, guidance written as (1 - g) u + g c, fp64 coefficients, s3 and s4 swapped) must differ from the restatement on the GPU sweep's inputs (every fp16 value of u
  against the structured values of c and x) at a named step of the 50-step schedule.  Unchanged, it must agree.
"""
import functools
import types

import numpy as np
import pytest

from oracle import latent_step as LS
from tokenflow_b200.editor import TokenFlowEditor
from tokenflow_b200.scheduler import DDIMScheduler

STEPS = 50
GUIDANCE = 7.5


def _schedule():
    sch = DDIMScheduler()
    sch.set_timesteps(STEPS)
    return sch


@functools.lru_cache(maxsize=None)
def _coef_rows():
    """The editor's fp32 coefficient table for a 50-step schedule, built by the editor's own method."""
    sch = _schedule()
    stub = types.SimpleNamespace(scheduler=sch, _t_host=[int(t) for t in sch.timesteps], device="cpu")
    return TokenFlowEditor._make_coef_table(stub).numpy()


def _fp64_coefs(row):
    """sqrt(1 - a_t), sqrt(a_t), sqrt(a_prev), sqrt(1 - a_prev) of schedule step `row` in double precision."""
    sch = _schedule()
    t = int(sch.timesteps[row])
    a_t, a_prev = float(sch._alpha(t)), float(sch._alpha(t - 1000 // STEPS))
    return (1 - a_t) ** 0.5, a_t ** 0.5, a_prev ** 0.5, (1 - a_prev) ** 0.5


def _cfg_ddim(u, c, x, row, g, *, fma_sum=False, true_div=False, f32_reciprocal=False, raw_diff=False,
              raw_scaled=False, lerp=False, fp64=False, swap_s3_s4=False):
    """tf_cfg_ddim's arithmetic written out again; each keyword is one plausible kernel or host bug."""
    h = lambda v: v.astype(np.float16).astype(np.float32)
    u, c, x = (v.astype(np.float32) for v in (u, c, x))
    s1, inv_s2, s3, s4 = (np.float32(v) for v in _coef_rows()[row])
    if f32_reciprocal:
        inv_s2 = np.float32(1) / np.float32(_fp64_coefs(row)[1])
    g32 = np.float32(g)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        if lerp:
            e = h(h(np.float32(1 - g32) * u) + h(g32 * c))
        else:
            d = (c - u) if raw_diff else h(c - u)
            m = (g32 * d) if raw_scaled else h(g32 * d)
            e = h(u + m)
        if fp64:
            hd = lambda v: v.astype(np.float16).astype(np.float64)
            S1, S2, S3, S4 = _fp64_coefs(row)
            e64, x64 = e.astype(np.float64), x.astype(np.float64)
            p = hd(hd(x64 - hd(S1 * e64)) * (1.0 / S2))
            return hd(hd(S3 * p) + hd(S4 * e64)).astype(np.float16)
        if swap_s3_s4:
            s3, s4 = s4, s3
        b = h(x - h(s1 * e))
        p = h(b / np.float32(_fp64_coefs(row)[1])) if true_div else h(b * inv_s2)
        c2 = h(s4 * e)
        if fma_sum:     # s3 * p + c2 contracted: one rounding of the exact product-sum
            return (s3.astype(np.float64) * p.astype(np.float64) + c2).astype(np.float32).astype(np.float16)
        return h(h(s3 * p) + c2).astype(np.float16)


def _sweep_chunks(step=1):
    """The GPU sweep's inputs, one x value at a time (every `step`-th structured value): u takes every fp16 value, c
    every structured value."""
    s = LS.structured_fp16()
    u = np.broadcast_to(LS.ALL_FP16[None, :], (len(s), 1 << 16))
    c = np.broadcast_to(s[:, None], u.shape)
    for xv in s[::step]:
        yield u, c, np.full(u.shape, xv, dtype=np.float16)


def _differs(row, g, step=1, **variant):
    """True as soon as one chunk of the sweep tells the variant apart from the restatement."""
    coef = _coef_rows()[row]
    for u, c, x in _sweep_chunks(step):
        if not LS.same_bits(_cfg_ddim(u, c, x, row, g, **variant), LS.cfg_ddim(u, c, x, coef, g)).all():
            return True
    return False


def test_restatement_on_hand_computed_edges():
    f16 = lambda *v: np.array(v, np.float16)
    # d = 18000, g * d = 135000 overflows: e = inf, x - s1 * e = -inf, and -inf + s4 * inf = NaN
    assert np.isnan(LS.cfg_ddim(f16(-9000), f16(9000), f16(1), (0.5, 2.0, 1.0, 0.25), GUIDANCE)[0])
    # e = 1 and x = inf: inf survives every step when s4 * e is finite
    assert np.isposinf(LS.cfg_ddim(f16(1), f16(1), f16(np.inf), (1.0, 1.0, 1.0, 0.0), 1.0)[0])
    # the smallest subnormal passes through unchanged
    assert LS.ddim(f16(0), f16(2 ** -24), (0.0, 1.0, 1.0, 0.0)).view(np.uint16)[0] == 0x0001
    # -2^-24 / 4 rounds to -0 in fp16, and -0 + -0 keeps the sign
    assert LS.ddim(f16(-0.0), f16(-2 ** -24), (1.0, 0.25, 1.0, 1.0)).view(np.uint16)[0] == 0x8000
    # 1 + 2^-11 is a tie between 1 and 1 + 2^-10: the fp16 rounding of e goes to the even 1.0
    assert LS.cfg_ddim(f16(1), f16(1 + 2 ** -10), f16(0), (0.0, 1.0, 0.0, 1.0), 0.5)[0] == 1.0


@pytest.mark.parametrize("row,g", [(0, GUIDANCE), (21, 3.3), (49, 0.0)])
def test_unchanged_restatement_agrees_with_the_oracle(row, g):
    assert not _differs(row, g, step=7)              # x = +-0, the largest subnormal, -inf, -9000 and N(0, 1) values


# variant -> the schedule step at which it must be told apart.  A true division differs from the multiply by the fp32
# reciprocal only where the two fp32 results straddle an fp16 rounding boundary: at 58 fp16 values of b = x - s1 e at
# step 21 and 60 at step 33, and at no fp16 value at the other 48 steps.  The fp32 reciprocal of the fp32 sqrt(a_t)
# (instead of ATen's double reciprocal, rounded) differs in the last bit at 8 steps and changes outputs at steps 25 and
# 46.
VARIANTS = {
    "fma_contracted_final_sum": (dict(fma_sum=True), 0),
    "true_division_by_sqrt_alpha": (dict(true_div=True), 21),
    "fp32_reciprocal_of_sqrt_alpha": (dict(f32_reciprocal=True), 25),
    "unrounded_c_minus_u": (dict(raw_diff=True), 0),
    "unrounded_g_times_d": (dict(raw_scaled=True), 0),
    "guidance_as_lerp": (dict(lerp=True), 0),
    "fp64_coefficients": (dict(fp64=True), 0),
    "s3_s4_swapped": (dict(swap_s3_s4=True), 0),
}


@pytest.mark.parametrize("name", sorted(VARIANTS))
def test_sweep_tells_the_planted_variant_apart(name):
    variant, row = VARIANTS[name]
    assert _differs(row, GUIDANCE, **variant), f"{name} is indistinguishable at step {row}"
