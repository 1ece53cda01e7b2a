"""CPU tier: the norm1 and unit-row checkers (oracle/kernel_checks.py) accept the kernels' arithmetic and reject
plausible mistakes.

`_unit_rows_kernel` and `_layernorm_kernel` restate tokenflow_b200/csrc/tf_unit_rows.cu in plain torch, in the
kernels' order: one warp per row, lane l holding channels 4l + 128i (tf_unit_rows) or the 8-channel vectors
l + 32j (the LayerNorm kernel, slot j), per-lane sums in that order, then the xor butterfly 16 ... 1.  LayerNorm runs
in fp32 (fp32 mean, two-pass variance, fp32 rsqrt, then the affine); the squared norms of the unit rows are fp64 and
the quotient is `div_by`: q = x * fp32(1/nrm), then fma(fma(-nrm, q, x), r, q), with fma emulated exactly.  The
restatements must pass both checkers; each keyword of theirs is one deliberate defect, which must fail the checker
on the probe named beside it.  Nothing here needs a GPU."""
import math

import pytest
import torch

from oracle.kernel_checks import (LN_SLOT_CHANNELS, check_layernorm_rows, check_unit_rows, ln_affine_f32,
                                  norm1_module, norm1_probe)

LANES = 32


def _fma32(a, b, c):
    """fp32 fma(a, b, c), exactly: the product is exact in fp64, the sum's error comes from TwoSum, and rounding the
    sum to odd in fp64 before rounding to fp32 makes the double rounding innocuous (53 >= 24 + 2)."""
    p = a.double() * b.double()
    cd = c.double()
    s = p + cd
    bp = s - p
    e = (p - (s - bp)) + (cd - bp)
    bits = s.view(torch.int64)
    away = (e > 0) == (s > 0)                      # the exact sum is larger in magnitude than s
    odd = torch.where(away, bits + 1, bits - 1)
    bits = torch.where((e != 0) & (bits & 1 == 0), odd, bits)
    return bits.view(torch.float64).float()


def _div_by(x, nrm, *, newton=True, ieee_range=True):
    """tf_unit_rows.cu `div_by` of fp32 x [rows, dim] by the fp32 row norms nrm [rows, 1]."""
    nrm = nrm.expand_as(x)
    r = torch.ones_like(nrm) / nrm                 # __frcp_rn
    q = x * r
    if newton:
        q = _fma32(_fma32(-nrm, q, x), r, q)
    if ieee_range:
        ieee = ~((nrm >= 2.0 ** -64) & (nrm <= 2.0 ** 64))
        q = torch.where(ieee, x / nrm, q)
    return q


def _butterfly(s):
    lane = torch.arange(LANES)
    for o in (16, 8, 4, 2, 1):
        s = s + s[:, lane ^ o]
    return s


def _unit_rows_kernel(x, *, fp32_sumsq=False, rsqrt_mul=False, newton=True, ieee_range=True):
    """tf_unit_rows of x [..., dim] (fp32 or fp16) -> fp16.  Defects: `fp32_sumsq` (the squared norm summed in fp32),
    `rsqrt_mul` (x * rsqrt(Σx²) instead of the division), `newton=False` (div_by without its correction),
    `ieee_range=False` (no IEEE division at extreme norms: the kernel before that branch)."""
    dim = x.shape[-1]
    xf = x.reshape(-1, dim).float()
    rows, it = xf.shape[0], -(-dim // (4 * LANES))
    acc = torch.float32 if fp32_sumsq else torch.float64
    v = torch.zeros(rows, it * 4 * LANES, dtype=acc)
    v[:, :dim] = xf.to(acc)
    sq = (v * v).view(rows, it, LANES, 4)
    t = ((sq[..., 0] + sq[..., 1]) + sq[..., 2]) + sq[..., 3]
    ss = torch.zeros(rows, LANES, dtype=acc)
    for i in range(it):
        ss = ss + t[:, i]
    ss = _butterfly(ss)[:, :1]
    if rsqrt_mul:
        q = xf * torch.rsqrt(ss).float()
    else:
        q = _div_by(xf, torch.sqrt(ss).float(), newton=newton, ieee_range=ieee_range)
    return q.half().view(x.shape)


def _layernorm_kernel(x, norm, n_unit_rows, *, bessel=False, eps_outside=False, eps=None, unit_from_fp16=False,
                      unit_pre_affine=False, drop_last_vec=False, affine_from_next_vec=False, unit_row_off=False):
    """tf_layernorm_rows of fp16 x [rows, dim] -> (fp16 y [rows, dim], fp16 unit rows of the first n_unit_rows).
    Defects: Bessel's variance / (dim - 1); eps outside the square root; another eps; unit rows from the fp16-rounded
    y or from the pre-affine (x - μ) rstd; the row's last 8-channel vector left out of both statistics; γ / β of the
    next vector; unit rows written one row down."""
    rows, dim = x.shape
    g32, b32, eps32 = ln_affine_f32(norm)
    eps32 = eps32 if eps is None else float(torch.tensor(eps, dtype=torch.float32))
    nvec = dim // 8
    slots = -(-dim // LN_SLOT_CHANNELS)
    width = slots * LN_SLOT_CHANNELS
    v = torch.zeros(rows, width)
    v[:, :dim] = x.float()
    v = v.view(rows, slots, LANES, 8)
    vec = torch.arange(slots)[:, None] * LANES + torch.arange(LANES)[None, :]      # vector index of (slot, lane)
    valid = vec < nvec
    stat = valid & ~((vec == nvec - 1) if drop_last_vec else torch.zeros_like(valid))
    s = torch.zeros(rows, LANES)
    for j in range(slots):
        for e in range(4):
            s = torch.where(stat[j], s + (v[:, j, :, 2 * e] + v[:, j, :, 2 * e + 1]), s)
    inv_dim = torch.tensor(1.0) / dim
    mean = _butterfly(s)[:, :1] * inv_dim
    sq = torch.zeros(rows, LANES)
    for j in range(slots):
        for e in range(8):
            d = v[:, j, :, e] - mean
            sq = torch.where(stat[j], sq + d * d, sq)
    var = _butterfly(sq)[:, :1] * ((torch.tensor(1.0) / (dim - 1)) if bessel else inv_dim)
    rstd = torch.tensor(1.0) / (torch.sqrt(var) + eps32) if eps_outside else torch.rsqrt(var + eps32)
    g, b = torch.zeros(width), torch.zeros(width)
    g[:dim], b[:dim] = g32, b32
    if affine_from_next_vec:
        g[:dim], b[:dim] = torch.roll(g32, -8), torch.roll(b32, -8)
    z = (v - mean[:, :, None, None]) * rstd[:, :, None, None]
    yv = z * g.view(slots, LANES, 8) + b.view(slots, LANES, 8)
    y = yv.reshape(rows, width)[:, :dim]
    src = y.half().float() if unit_from_fp16 else (z.reshape(rows, width)[:, :dim] if unit_pre_affine else y)
    srcv = torch.zeros(rows, width, dtype=torch.float64)
    srcv[:, :dim] = src.double()
    srcv = srcv.view(rows, slots, LANES, 8)
    ss = torch.zeros(rows, LANES, dtype=torch.float64)
    for j in range(slots):
        for e in range(8):
            ss = torch.where(valid[j], ss + srcv[:, j, :, e] * srcv[:, j, :, e], ss)
    nrm = torch.sqrt(_butterfly(ss)[:, :1]).float()
    unit = _div_by(src[:n_unit_rows], nrm[:n_unit_rows]).half()
    if unit_row_off:
        unit = torch.roll(unit, 1, 0)
    return y.half(), unit


def _gen(seed):
    return torch.Generator().manual_seed(seed)


SLOT_DIMS = [8, 40, 248, 256, 264, 320, 512, 520, 640, 768, 776, 1016, 1024, 1032, 1272, 1280]


@pytest.mark.parametrize("dim", SLOT_DIMS)
def test_layernorm_restatement_passes_at_every_slot_boundary(dim):
    g = _gen(dim)
    norm = norm1_module(dim, "signed" if dim % 16 else "positive", generator=g)
    x = norm1_probe("randn", 24, dim, generator=g)
    y, unit = _layernorm_kernel(x, norm, 8)
    st = check_layernorm_rows(y, unit.view(8, dim), x, norm, 8, tag=f"dim {dim}")
    assert st["y_use"] < 0.5 and st["u_use"] < 0.5, st


@pytest.mark.parametrize("kind", ["randn", "var_10eps", "var_1eps", "var_0.1eps", "offset_200", "offset_-3000",
                                  "constant", "outlier_1000", "outlier_30000", "near_60000"])
@pytest.mark.parametrize("dim,gamma", [(40, "signed"), (320, "positive"), (1032, "signed"), (1280, "positive")])
def test_layernorm_restatement_passes_the_statistics_probes(kind, dim, gamma):
    g = _gen(dim + len(kind))
    norm = norm1_module(dim, gamma, generator=g)
    x = norm1_probe(kind, 16, dim, generator=g)
    y, unit = _layernorm_kernel(x, norm, 16)
    st = check_layernorm_rows(y, unit, x, norm, 16, tag=f"{kind} dim {dim}")
    if kind == "constant":                            # y = β (up to δ), unit = β / ||β||
        beta = norm.bias.float()
        assert (y.float() - beta.half().float()).abs().max() <= 2.0 ** -10
    print(st)


@pytest.mark.parametrize("dim", [8, 40, 264, 320, 776, 1032, 1280])
def test_unit_rows_restatement_is_exact(dim):
    g = _gen(dim)
    for x in (torch.randn(64, dim, generator=g) * 3 + 0.5, (torch.randn(64, dim, generator=g) * 3).half(),
              _wide_range(64, dim, g)):
        st = check_unit_rows(_unit_rows_kernel(x), x, tag=f"dim {dim} {x.dtype}")
        assert st["exempt"] == 0


def _wide_range(rows, dim, g):
    """fp32 rows whose elements span 2^-12 ... 2^12 (log-uniform): an fp32 sum of squares loses the small ones."""
    return torch.randn(rows, dim, generator=g) * torch.exp2(torch.randint(-12, 13, (rows, dim), generator=g).float())


def _subnormal_norm_rows(g):
    """fp32 rows of 320 elements around 2^-136: the row norm (about 2^-132) is a subnormal fp32 number, so 1 / norm
    overflows, while x / fp32(norm) is finite."""
    return torch.randn(48, 320, generator=g) * 2.0 ** -136


def test_unit_rows_restatement_is_exact_for_subnormal_norms():
    x = _subnormal_norm_rows(_gen(11))
    n = x.double().norm(dim=-1)
    assert (n < 2.0 ** -126).all() and (n > 2.0 ** -149).all()
    check_unit_rows(_unit_rows_kernel(x), x)


def _scale_sweep(x):
    """Powers of two k, every 10 from -100 to 100 plus the two extremes at which every element and the row norm stay
    normal fp32 numbers below 2^128."""
    lo = max(math.ceil(-126 - math.log2(x.abs().min().item())), math.ceil(-126 - math.log2(x.norm(dim=-1).min().item())))
    hi = math.floor(127 - math.log2(x.norm(dim=-1).max().item()))
    return sorted(set(range(-100, 101, 10)) | {lo, hi})


def test_unit_rows_restatement_is_scale_invariant():
    g = _gen(7)
    x = torch.sign(torch.randn(48, 320, generator=g)) * (0.5 + 1.5 * torch.rand(48, 320, generator=g))
    base = _unit_rows_kernel(x)
    check_unit_rows(base, x)
    for k in _scale_sweep(x):
        xs = x * 2.0 ** k
        assert torch.equal(xs * 2.0 ** -k, x)
        got = _unit_rows_kernel(xs)
        check_unit_rows(got, xs, tag=f"2^{k}")
        assert torch.equal(got, base), k


def _layernorm_case(dim, kind, gamma="positive", rows=16, seed=0):
    g = _gen(seed + dim)
    return norm1_probe(kind, rows, dim, generator=g), norm1_module(dim, gamma, generator=g)


LN_DEFECTS = [
    # (defect, keywords, probe, dims)
    ("Bessel variance / (dim - 1)", {"bessel": True}, "randn", [8, 40, 320]),
    ("eps outside the square root", {"eps_outside": True}, "var_0.1eps", [40, 320, 1280]),
    ("eps 1e-6 instead of 1e-5", {"eps": 1e-6}, "var_0.1eps", [40, 320, 1280]),
    ("unit rows from the fp16-rounded y", {"unit_from_fp16": True}, "randn", [40, 320, 1280]),
    ("unit rows of the pre-affine (x - mean) rstd", {"unit_pre_affine": True}, "randn", [40, 320, 1280]),
    ("last vector of a partly filled slot left out of the statistics", {"drop_last_vec": True}, "randn",
     [264, 776, 1032]),
    ("gamma / beta of the neighbouring vector", {"affine_from_next_vec": True}, "randn", [40, 320, 1280]),
    ("unit rows written one row off", {"unit_row_off": True}, "randn", [40, 320, 1280]),
]


@pytest.mark.parametrize("defect,kw,probe,dims", LN_DEFECTS, ids=[d[0] for d in LN_DEFECTS])
def test_check_layernorm_rows_rejects(defect, kw, probe, dims):
    for dim in dims:
        x, norm = _layernorm_case(dim, probe)
        check_layernorm_rows(*_layernorm_kernel(x, norm, 16), x, norm, 16)
        y, unit = _layernorm_kernel(x, norm, 16, **kw)
        with pytest.raises(AssertionError):
            check_layernorm_rows(y, unit, x, norm, 16, tag=f"{defect}, {probe} probe, dim {dim}")


UNIT_DEFECTS = [
    ("fp32 sum of squares", {"fp32_sumsq": True}, "randn fp32 rows"),
    ("x * rsqrt(sum x^2) instead of the division", {"rsqrt_mul": True}, "randn fp32 rows"),
    ("div_by without the Newton step", {"newton": False}, "randn fp32 rows"),
    ("no IEEE division at extreme norms", {"ieee_range": False}, "rows with a subnormal fp32 norm"),
]


@pytest.mark.parametrize("defect,kw,probe", UNIT_DEFECTS, ids=[d[0] for d in UNIT_DEFECTS])
def test_check_unit_rows_rejects(defect, kw, probe):
    g = _gen(3)
    if probe == "randn fp32 rows":
        xs = [torch.randn(1024, 1280, generator=g) * 3 + 0.5]
    else:
        xs = [_subnormal_norm_rows(g)]
    for x in xs:
        check_unit_rows(_unit_rows_kernel(x), x)
    failed = []
    for x in xs:
        try:
            check_unit_rows(_unit_rows_kernel(x, **kw), x, tag=f"{defect}, {probe}")
        except AssertionError as e:
            failed.append(str(e))
    assert failed, f"{defect} passed the {probe} probe"
    print(failed[0])
