"""ORACLE (test infrastructure) — calibrated checks of the CUDA kernels' outputs.

`check_ext_attn` compares an extended-attention output with the same sample table evaluated in fp64 on
the kernel's fp16 inputs.  Its bounds come from the kernel's arithmetic, not from a fixed tolerance:
the only rounding steps of tf_ext_attn are the fp16 probabilities P (2^-11 relative, each key) and the
fp16 output (2^-11 relative), so

    |got - ref| <= 2^-10 * (A|v| + |ref|) + 2^-24        elementwise,

where A|v| is the same attention applied to |v| (the worst case of the P rounding) and the factor 2^-10
is 2^-11 with a 2x margin.  A bound that scales with the output keeps its power at large n*S, where the
softmax averages over many keys and the outputs shrink.  The relative RMS error is further compared with
an emulation of the same rounding (fp32 scores, fp16 P, fp32 normaliser, fp16 output), which is
scale-free.  The fixed north-star bound max|got - ref| < 1e-3 (BASELINE.json) stays as a ceiling.

`check_nn_field` is the one implementation of the NN-field rule: every index equals the argmax of the
kernel's own fp16 operands (dot products accumulated in fp64, rounded to fp16, first index on ties), up to
rows inside a 1-ulp fp16 tie class, whose winner depends on the GEMM's fp32 accumulation order.  Such
rows are bounded and counted.

`check_group_norm` compares a tf_group_norm_nhwc output with the eager ATen sequence it replaces and with
an fp64 evaluation.  ATen stores the group mean and rstd in fp16, so those bounds cannot see a statistics
error below about one fp16 ulp of the mean or rstd.  `check_group_norm_workspace` closes that gap: it reads
the kernel's per-chunk partial sums (the caller's workspace, `[N, G, stats_chunks]` of (Σd, Σd²)) and
compares every entry with an fp64 evaluation to 2^-16 of the chunk's Σ|d| and Σd².  Each fp32 inner sum
of the kernel runs over at most 32 values (about 2^-19 of their Σ|d| in the worst case); a dropped pixel
moves a chunk's sums by about 1 / stats_px >= 2^-12 of them.

`check_unit_rows` pins tf_unit_rows bit for bit.  The kernel's arithmetic is exact enough to state: the squared
norm is summed in fp64 (about 2^-50 relative, far below the fp32 rounding of its square root), so
nrm = fp32(sqrt(Σx²)); the quotient is the IEEE fp32 x / nrm (Markstein's reciprocal-and-one-correction
sequence, `div_by`), and fp64 division of two fp32 numbers rounded to fp32 is that quotient, since
53 >= 2 * 24 + 2 bits make the double rounding innocuous.  The output is fp16 of the quotient.  A mismatch
is exempt only where the kernel's quotient could lawfully be 1 fp32 ulp away and that ulp decides the fp16
rounding: exactly 1 fp16 ulp off, with the exact fp32 quotient within 1 fp32 ulp of an fp16 midpoint.  Such
elements are counted; at most `max_exempt` (default one in 2^20) may occur.

`check_layernorm_rows` checks tf_layernorm_rows / tf_layernorm_unit_rows against LayerNorm and unit rows
evaluated in fp64 (`layernorm_fp64`), with an interval rule: every fp16 output must be the fp16 rounding of
some value within δ of the fp64 result, δ coming from a first-order error analysis of the kernel's fp32
pipeline (`layernorm_deltas`).  A correct kernel uses a small fraction of δ; a wrong variance divisor, eps
or affine parameter, a dropped vector or a row written to the wrong place moves outputs by many δ.
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import torch
import torch.nn.functional as F

ATTN_REL_ULP = 2.0 ** -10       # fp16 rounding (2^-11 relative) of P and of the output, with a 2x margin
ATTN_ABS_FLOOR = 2.0 ** -24
ATTN_EMU_FACTOR = 2.0
ATTN_EMU_FLOOR = 1e-5


def ext_attn_samples(n: int, inject: bool):
    """The sample table of `CudaOps.ext_attn` ([3n, S, dim] q/k/v, frame-major streams; reference
    tokenflow_utils.py:124-179): source samples attend to their own frame, uncond / cond samples to the n
    frames of their stream, with q and k of the source stream under PnP injection."""
    table = []
    for i in range(3 * n):
        s, f = divmod(i, n)
        if s == 0:
            table.append((i, i, i, 1))
        else:
            table.append((f, 0, s * n, n) if inject else (i, s * n, s * n, n))
    return table


def logit_shift_probe(q: torch.Tensor, k: torch.Tensor, heads: int, scale: float, generator=None):
    """In place: in every head, the last channel of q becomes a and that of k becomes -a(1 + 0.1u), u uniform,
    a = sqrt(25 / scale).  Every real logit then sits near -25 (spread about 2.5), far below the logit 0 of a
    zero-filled padding key: one leaked padding key dominates its softmax row.  fp16 stays well in range."""
    dim = q.shape[-1]
    d = dim // heads
    a = math.sqrt(25.0 / scale)
    last = torch.arange(heads, device=q.device) * d + d - 1
    u = torch.rand(k.shape[:-1] + (heads,), generator=generator).to(k.device)
    q[..., last] = a
    k[..., last] = (-a * (1.0 + 0.1 * u)).to(k.dtype)
    return q, k


def negative_similarity_probe(F: int, K: int, S: int, dim: int, kf: Sequence[int], generator=None):
    """Pivots [K, S, dim] around +e0 and frame tokens [F, S, dim] around -e0 (fp32, not normalised): every
    real similarity is below 0, so a zero-filled padding column (similarity 0) would win any row it reaches.
    Frame f's tokens are a permutation of keyframe kf[f]'s off-axis parts plus noise, so the nearest
    neighbours stay distinct."""
    g = torch.randn(K, S, dim, generator=generator)
    g[..., 0] = 0
    g = g / g.norm(dim=-1, keepdim=True)
    e0 = torch.zeros(dim)
    e0[0] = 1
    piv = e0 + 0.5 * g
    x = torch.empty(F, S, dim)
    for f in range(F):
        noise = 0.3 * torch.randn(S, dim, generator=generator) / math.sqrt(dim)
        noise[:, 0] = 0
        x[f] = -e0 + 0.5 * (g[kf[f]][torch.randperm(S, generator=generator)] + noise)
    return x, piv


def _attn_terms(q, k, v, table, heads, scale, row0, r1, row_chunk=1024):
    """(ref, A|v|, emulation) as fp64 tensors [len(table), r1 - row0, dim]."""
    _, S, dim = q.shape
    d = dim // heads
    R = r1 - row0
    shape = (len(table), R, dim)
    ref = torch.zeros(shape, dtype=torch.float64, device=q.device)
    absv = torch.zeros_like(ref)
    emu = torch.zeros_like(ref)
    for j, (qs, k0, v0, nkv) in enumerate(table):
        for h in range(heads):
            ch = slice(h * d, (h + 1) * d)
            kk = k[k0:k0 + nkv, :, ch].reshape(nkv * S, d)
            vv = v[v0:v0 + nkv, :, ch].reshape(nkv * S, d)
            k64, v64, k32, v32 = kk.double(), vv.double(), kk.float(), vv.float()
            for a in range(row0, r1, row_chunk):
                b = min(r1, a + row_chunk)
                qq = q[qs, a:b, ch]
                p64 = torch.softmax((qq.double() @ k64.T) * scale, dim=-1)
                ref[j, a - row0:b - row0, ch] = p64 @ v64
                absv[j, a - row0:b - row0, ch] = p64 @ v64.abs()
                s32 = (qq.float() @ k32.T) * scale
                p32 = torch.exp(s32 - s32.amax(dim=-1, keepdim=True))
                o = (p32.half().float() @ v32) / p32.sum(dim=-1, keepdim=True)
                emu[j, a - row0:b - row0, ch] = o.half().double()
    return ref, absv, emu


def check_ext_attn(got: torch.Tensor, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, table, heads: int,
                   scale: float, row0: int = 0, nrows: Optional[int] = None, *, atol: float = 1e-3,
                   rtol: float = 0.0, max_rel: Optional[float] = None) -> dict:
    """Assert that `got` is `ext_attn_table(q, k, v, table, heads, scale, row0, nrows)` computed correctly.

    q [Q, S, dim], k / v [KV, S, dim] fp16 (the kernel's inputs); `table[j] = (q slab, first k slab, first v
    slab, number of key slabs)` as in `OracleOps.ext_attn_table`.  `got` is [len(table), nrows, dim] fp16;
    only its rows of tokens < S are compared (the kernel leaves the rest unwritten).  `atol` / `rtol` set the
    fixed ceiling |got - ref| < atol + rtol * |ref|; `max_rel` optionally caps the relative RMS error.
    Returns the measured statistics, including the ratio of the relative RMS error to the emulation's."""
    _, S, dim = q.shape
    nrows = S if nrows is None else int(nrows)
    r1 = min(S, row0 + nrows)
    assert got.dtype == torch.float16, got.dtype
    assert tuple(got.shape) == (len(table), nrows, dim), (tuple(got.shape), (len(table), nrows, dim))
    assert q.dtype == k.dtype == v.dtype == torch.float16, "check the fp16 tensors the kernel read"
    if r1 <= row0:
        return {"rel": 0.0, "rel_emu": 0.0, "ratio": 1.0, "max_err": 0.0, "bound_use": 0.0}
    g = got[:, :r1 - row0].double()
    assert torch.isfinite(g).all(), "NaN or Inf in the attention output"
    ref, absv, emu = _attn_terms(q, k, v, table, heads, scale, row0, r1)

    err = (g - ref).abs()
    bound = ATTN_REL_ULP * (absv + ref.abs()) + ATTN_ABS_FLOOR
    use = err / bound
    worst = int(use.argmax())
    j, r, c = (worst // (use.shape[1] * use.shape[2]), (worst // use.shape[2]) % use.shape[1], worst % use.shape[2])
    stats = {"max_err": err.max().item(), "bound_use": use.max().item()}
    assert stats["bound_use"] <= 1.0, (
        f"outside the fp16 error model at sample {j} token {row0 + r} channel {c}: got {g[j, r, c].item():.6g}, "
        f"ref {ref[j, r, c].item():.6g}, bound {bound[j, r, c].item():.3g}; "
        f"{int((use > 1).sum())} of {use.numel()} elements exceed it")

    ref_norm = ref.norm().clamp_min(1e-300)
    rel = ((g - ref).norm() / ref_norm).item()
    rel_emu = ((emu - ref).norm() / ref_norm).item()
    stats.update(rel=rel, rel_emu=rel_emu, ratio=rel / rel_emu if rel_emu > 0 else math.inf)
    assert rel <= ATTN_EMU_FACTOR * rel_emu + ATTN_EMU_FLOOR, (
        f"relative RMS error {rel:.3g} vs {rel_emu:.3g} of the fp16-P emulation")
    assert (err < atol + rtol * ref.abs()).all(), f"max|got - ref| = {stats['max_err']:.3g} (ceiling {atol}, rtol {rtol})"
    if max_rel is not None:
        assert rel < max_rel, f"relative RMS error {rel:.3g} >= {max_rel}"
    return stats


def nn_similarity(x_unit: torch.Tensor, piv_unit: torch.Tensor) -> torch.Tensor:
    """fp16 similarities of fp16 unit rows, dot products accumulated in fp64: [R, dim] x [C, dim] -> [R, C]."""
    return (x_unit.double() @ piv_unit.double().T).float().half()


def tie_class(sim: torch.Tensor, rows: torch.Tensor, got: torch.Tensor, want: torch.Tensor,
              ulps: float = 1.0) -> torch.Tensor:
    """For rows whose index `got` differs from `want` (the argmax of `sim`): True where the two candidates'
    fp16 similarities lie within `ulps` fp16 ulps (at the winner's magnitude) of each other, i.e. the
    winner depends only on the accumulation order of the dot products."""
    s_want = sim[rows, want].float()
    s_got = sim[rows, got].float()
    ulp = 2.0 ** (torch.floor(torch.log2(s_want.abs().clamp_min(1e-8))) - 10)
    return (s_want - s_got).abs() <= ulps * ulp * 1.001


def check_nn_field(idx_a: torch.Tensor, idx_b: Optional[torch.Tensor], x_unit: torch.Tensor,
                   piv_unit: torch.Tensor, kf_a: Sequence[int], kf_b: Sequence[int],
                   max_tie_frac: float = 5e-3) -> dict:
    """Assert that (idx_a, idx_b) is `nn_field(x_unit, piv_unit, kf_a, kf_b)` computed correctly.

    x_unit [F, S, dim], piv_unit [K, S, dim] are the fp16 unit rows the kernel read.  idx_b is read only for
    frames with kf_b >= 0 (the kernel leaves the other rows unwritten).  Returns the tie-row count."""
    F, S, _ = x_unit.shape
    assert idx_a.dtype == torch.int32 and tuple(idx_a.shape) == (F, S), (idx_a.dtype, tuple(idx_a.shape))
    any_b = any(int(b) >= 0 for b in kf_b)
    if any_b:
        assert idx_b is not None and idx_b.dtype == torch.int32 and tuple(idx_b.shape) == (F, S)
    else:
        assert idx_b is None
    total = ties = 0
    for f in range(F):
        for kf, idx in ((int(kf_a[f]), idx_a), (int(kf_b[f]), idx_b)):
            if kf < 0:
                continue
            got = idx[f].long()
            assert got.min().item() >= 0 and got.max().item() < S, \
                f"frame {f}, keyframe {kf}: index outside [0, {S}) ({got.min().item()}..{got.max().item()})"
            sim = nn_similarity(x_unit[f], piv_unit[kf])
            want = sim.argmax(dim=-1)
            bad = (got != want).nonzero().flatten()
            total += S
            ties += bad.numel()
            if bad.numel():
                inside = tie_class(sim, bad, got[bad], want[bad])
                assert inside.all(), (f"frame {f}, keyframe {kf}: token {bad[~inside][0].item()} has an NN index "
                                      f"outside the fp16 tie class")
    assert ties <= max(2, int(max_tie_frac * total)), f"{ties}/{total} rows differ from the oracle"
    return {"ties": ties, "total": total}


# ------------------------------------------------------------------------------------------------
# GroupNorm (tf_group_norm_nhwc)
# ------------------------------------------------------------------------------------------------
GN_MAX_THREADS = 512            # tf_body.cu kGnMaxThreads
GN_STATS_CHUNK_BYTES = 64 << 10  # kGnStatsChunkBytes
GN_APPLY_CHUNK_BYTES = 128 << 10  # kGnApplyChunkBytes
GN_WS_REL_TOL = 2.0 ** -16       # observed on one H100 80GB HBM3 (400 W): at most 7.6e-8 (Σd) and 2.6e-7 (Σd²) over
                                 # the 222 shapes of tests/test_gpu_body_kernels.py, 4.9e-8 / 6.5e-8 at the real UNet
                                 # sites; a dropped pixel moves a chunk by >= 2^-12


def gn_layout(hw: int, c: int) -> dict:
    """tf_body.cu `gn_layout`: one thread per 8-channel column, `rows` pixel rows per CTA, and the pixel chunk of a
    statistics / apply CTA (a multiple of `rows` of about 64 / 128 KB of input)."""
    cols = c // 8
    rows = max(1, GN_MAX_THREADS // cols)

    def chunk(nbytes):
        px = nbytes // (2 * c)
        px = -(-px // rows) * rows
        return max(px, rows)

    stats_px, apply_px = chunk(GN_STATS_CHUNK_BYTES), chunk(GN_APPLY_CHUNK_BYTES)
    return {"cols": cols, "rows": rows, "threads": -(-cols * rows // 32) * 32, "stats_px": stats_px,
            "apply_px": apply_px, "stats_chunks": -(-hw // stats_px), "apply_chunks": -(-hw // apply_px)}


def ulp16(v: torch.Tensor) -> torch.Tensor:
    """fp16 spacing at |v| (fp32 tensor of magnitudes): 2^(e - 11) for v = m * 2^e, m in [0.5, 1); 2^-24 below."""
    _, e = torch.frexp(v.abs())
    return torch.clamp(torch.ldexp(torch.ones_like(v), e - 11), min=2.0 ** -24)


def _add_bias(x, bias):
    return x if bias is None else x + bias[:, :, None, None]      # the fp16 add, as the eager path rounds it


def group_norm_aten(x, norm, bias, silu):
    """The eager sequence tf_group_norm_nhwc replaces: fp16 add, ATen GroupNorm, SiLU."""
    y = F.group_norm(_add_bias(x, bias), norm.num_groups, norm.weight, norm.bias, norm.eps)
    return F.silu(y) if silu else y


def group_norm_fp64(x, norm, bias, silu):
    x = _add_bias(x, bias)
    n = x.shape[0]
    xd = x.double().reshape(n, norm.num_groups, -1)
    mean = xd.mean(-1, keepdim=True)
    var = ((xd - mean) ** 2).mean(-1, keepdim=True)
    y = ((xd - mean) / torch.sqrt(var + norm.eps)).reshape(x.shape)
    y = y * norm.weight.double()[None, :, None, None] + norm.bias.double()[None, :, None, None]
    return y * torch.sigmoid(y) if silu else y


def group_norm_stat_flip_bound(x, norm, bias, silu):
    """How far the output moves when ATen's fp16 mean or rstd (RowwiseMomentsCUDAKernel<Half> stores both in the input
    dtype) is one fp16 ulp away: a statistic computed slightly differently can land on the other side of an fp16
    rounding boundary, and then every output element of that group moves by up to
    |rstd * gamma| * ulp(mean) + |x - mean| * |gamma| * ulp(rstd); after SiLU, 1.1 (its largest slope) times that plus
    one ulp of the fp16 pre-activation."""
    x = _add_bias(x, bias)
    n, c, h, w = x.shape
    G = norm.num_groups
    _, mean, rstd = torch.ops.aten.native_group_norm(x.contiguous(), norm.weight, norm.bias, n, c, h * w, G, norm.eps)
    mean = mean.float().view(n, G, 1).expand(n, G, c // G).reshape(n, c, 1, 1)
    rstd = rstd.float().view(n, G, 1).expand(n, G, c // G).reshape(n, c, 1, 1)
    gamma = norm.weight.float().abs()[None, :, None, None]
    bound = rstd * gamma * ulp16(mean) + (x.float() - mean).abs() * gamma * ulp16(rstd)
    if not silu:
        return bound
    # SiLU maps a one-ulp difference of its fp16 input y to up to 1.1 ulp(y), more than ulp(silu(y)) for y < 0
    y = F.group_norm(x, G, norm.weight, norm.bias, norm.eps).float()
    return 1.1 * (bound + ulp16(y))


def aten_misrounded_groups(x, norm, bias) -> torch.Tensor:
    """[N, G] bool: groups whose ATen fp16 mean or rstd differs from the fp64 statistic rounded to fp16 (ATen's fp32
    Welford lands on the wrong side of an fp16 rounding boundary)."""
    x = _add_bias(x, bias)
    n, c, h, w = x.shape
    G = norm.num_groups
    _, mean, rstd = torch.ops.aten.native_group_norm(x.contiguous(), norm.weight, norm.bias, n, c, h * w, G, norm.eps)
    xd = x.double().reshape(n, G, -1)
    m = xd.mean(-1)
    var = ((xd - m[..., None]) ** 2).mean(-1)
    r = 1.0 / torch.sqrt(var + float(torch.tensor(norm.eps).half()))
    return (mean.view(n, G) != m.half()) | (rstd.view(n, G) != r.half())


def check_group_norm(got: torch.Tensor, x: torch.Tensor, norm, bias: Optional[torch.Tensor], silu: bool,
                     tag: str = "", exempt_aten_misrounded: bool = False) -> dict:
    """Assert that `got` is `[SiLU](GroupNorm(x [+ bias[:, :, None, None]]))` as tf_group_norm_nhwc computes it.

    x [N, C, H, W] fp16 (any H, W), bias fp16 [N, C] / [1, C] or None.  At least 99.9 % of the elements are within
    1 fp16 ulp of ATen; every element is within 1 ulp plus what a one-ulp change of ATen's fp16 mean / rstd explains
    (`group_norm_stat_flip_bound`); the error against fp64 is no worse than ATen's by more than the same amount.
    The 99.9 % rule is statistical: with few groups (tiny images, one group) or with statistics ATen's fp32 Welford
    rounds badly, a single group whose ATen fp16 statistic is misrounded (`aten_misrounded_groups`) exceeds 0.1 % on
    its own.  `exempt_aten_misrounded` leaves those groups out of the fraction; they still meet the other two bounds.
    Returns the bit-equal and within-1-ulp fractions."""
    assert got.dtype == torch.float16 and tuple(got.shape) == tuple(x.shape), (got.dtype, tuple(got.shape))
    want = group_norm_aten(x, norm, bias, silu)
    g32, w32 = got.float(), want.float()
    ulp = ulp16(torch.maximum(g32.abs(), w32.abs()))
    diff = (g32 - w32).abs()
    counted = torch.ones_like(diff, dtype=torch.bool)
    exempt = 0
    if exempt_aten_misrounded:
        n, c = x.shape[:2]
        G = norm.num_groups
        bad = aten_misrounded_groups(x, norm, bias)
        exempt = int(bad.sum())
        counted = ~bad.view(n, G, 1).expand(n, G, c // G).reshape(n, c, 1, 1).expand_as(diff)
    within = (diff <= ulp)[counted].float().mean().item() if counted.any() else 1.0
    stats = {"bit_equal": (got == want).float().mean().item(), "within_1ulp": within,
             "within_1ulp_all": (diff <= ulp).float().mean().item(), "max_ulps": (diff / ulp).max().item(),
             "exempt_groups": exempt}
    print(f"{tag}: bit-equal {stats['bit_equal']:.5f}, within 1 ulp {stats['within_1ulp']:.5f} "
          f"({stats['within_1ulp_all']:.5f} with every group), max |diff| / ulp {stats['max_ulps']:.2f}, "
          f"groups with misrounded ATen statistics left out {exempt}")
    assert stats["within_1ulp"] >= 0.999, f"{tag}: only {stats['within_1ulp']:.5f} of the elements within 1 ulp of ATen"
    flip = group_norm_stat_flip_bound(x, norm, bias, silu)
    assert (diff <= ulp + flip).all(), f"{tag}: {(diff > ulp + flip).sum().item()} elements off by more than 1 ulp " \
                                       "plus a one-ulp change of the fp16 statistics"
    ref = group_norm_fp64(x, norm, bias, silu)
    err_got = (g32.double() - ref).abs()
    err_aten = (w32.double() - ref).abs()
    ulp3 = ulp16(torch.maximum(torch.maximum(g32.abs(), w32.abs()), ref.float().abs())).double()
    assert (err_got <= err_aten + ulp3 + flip.double()).all(), f"{tag}: less accurate than ATen"
    return stats


def group_norm_partials(x: torch.Tensor, bias: Optional[torch.Tensor], groups: int, stats_px: int):
    """fp64 (Σd, Σd², Σ|d|), each [N, G, chunks], of d = fp16(x + bias) - shift over the pixel chunks
    [k * stats_px, min((k + 1) * stats_px, hw)); the shift is the group's element at pixel 0, channel g * cpg."""
    xv = _add_bias(x, bias)
    n, c, h, w = xv.shape
    hw, cpg = h * w, c // groups
    chunks = -(-hw // stats_px)
    xd = xv.permute(0, 2, 3, 1).reshape(n, hw, groups, cpg).double()
    d = xd - xd[:, :1, :, :1]
    d = torch.cat([d, d.new_zeros(n, chunks * stats_px - hw, groups, cpg)], dim=1).view(n, chunks, stats_px, groups, cpg)
    sums = [d.sum((2, 4)), (d * d).sum((2, 4)), d.abs().sum((2, 4))]
    return tuple(s.permute(0, 2, 1).contiguous() for s in sums)


def check_group_norm_workspace(ws: torch.Tensor, x: torch.Tensor, bias: Optional[torch.Tensor], groups: int, hw: int,
                               c: int, tol: float = GN_WS_REL_TOL, tag: str = "") -> dict:
    """Assert that the statistics workspace a tf_group_norm_nhwc call left behind holds the exact partial sums.

    ws: the workspace bytes (uint8, exactly what `tf_group_norm_nhwc_workspace` asked for), read as
    [N, G, stats_chunks] of double2 (Σd, Σd²).  Every entry must match `group_norm_partials` to `tol` of the chunk's
    Σ|d| (first sum) and Σd² (second sum).  Returns the largest error of each sum relative to its scale."""
    n = x.shape[0]
    L = gn_layout(hw, c)
    assert tuple(x.shape[1:2]) == (c,) and x.shape[2] * x.shape[3] == hw, (tuple(x.shape), c, hw)
    assert ws.dtype == torch.uint8 and ws.numel() == n * groups * L["stats_chunks"] * 16, \
        f"{tag}: workspace of {ws.numel()} bytes, layout [N={n}, G={groups}, chunks={L['stats_chunks']}] x 16"
    got = ws.view(torch.float64).view(n, groups, L["stats_chunks"], 2).to(x.device)
    s1, s2, sabs = group_norm_partials(x, bias, groups, L["stats_px"])
    e1, e2 = (got[..., 0] - s1).abs(), (got[..., 1] - s2).abs()
    ok1, ok2 = e1 <= tol * sabs, e2 <= tol * s2
    stats = {"rel1": (e1 / sabs.clamp_min(1e-300)).max().item(), "rel2": (e2 / s2.clamp_min(1e-300)).max().item()}
    for ok, name, ref in ((ok1, "sum d", s1), (ok2, "sum d^2", s2)):
        if not ok.all():
            i, g, k = (int(v) for v in (~ok).nonzero()[0])
            j = 0 if name == "sum d" else 1
            raise AssertionError(f"{tag}: {int((~ok).sum())} workspace entries off in {name}; first at sample {i} "
                                 f"group {g} chunk {k}: {got[i, g, k, j].item():.17g} vs fp64 {ref[i, g, k].item():.17g}")
    return stats


def guarded_group_norm(lib, x: torch.Tensor, norm, bias: Optional[torch.Tensor], silu: bool, guard: int = 256):
    """tf_group_norm_nhwc straight through the C ABI into a NaN-filled buffer with guard bands, with a workspace of
    exactly the size `tf_group_norm_nhwc_workspace` asks for.  Asserts that every output element was written and
    nothing outside.  Returns (out as a channels_last [N, C, H, W] view, workspace bytes)."""
    n, c, h, w = x.shape
    assert x.is_contiguous(memory_format=torch.channels_last)
    numel = x.numel()
    buf = torch.full((numel + 2 * guard,), float("nan"), dtype=torch.float16, device=x.device)
    out = buf[guard:guard + numel]
    ws = torch.empty(lib.tf_group_norm_nhwc_workspace(n, h * w, c, norm.num_groups), dtype=torch.uint8,
                     device=x.device)
    if bias is not None:
        assert bias.stride(1) == 1
        bias_stride = 0 if bias.shape[0] == 1 else bias.stride(0)
    st = lib.tf_group_norm_nhwc(x.data_ptr(), bias.data_ptr() if bias is not None else None,
                                bias_stride if bias is not None else 0, norm.weight.data_ptr(), norm.bias.data_ptr(),
                                n, h * w, c, norm.num_groups, float(norm.eps), int(silu), ws.data_ptr(), ws.numel(),
                                out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert st == 0, lib.tf_last_error()
    torch.cuda.synchronize()
    assert torch.isnan(buf[:guard]).all() and torch.isnan(buf[guard + numel:]).all(), "write outside the output"
    assert not torch.isnan(out).any(), "output element left unwritten"
    return out.view(n, h, w, c).permute(0, 3, 1, 2), ws


# ------------------------------------------------------------------------------------------------
# norm1 and unit rows (tf_unit_rows, tf_layernorm_rows, tf_layernorm_unit_rows)
# ------------------------------------------------------------------------------------------------
LN_SLOT_CHANNELS = 256          # tf_unit_rows.cu: one register slot of a row = 32 lanes x 8 channels
LN_MAX_DIM = 1280               # kLnMaxVecPerLane = 5 slots
U32 = 2.0 ** -24                # unit roundoff of fp32 (half an ulp, relative)
RSQRTF_ULPS = 2                 # rsqrtf: maximum error 2 ulp (CUDA C++ Programming Guide, single-precision functions)
UNIT_MAX_EXEMPT_FRAC = 2.0 ** -20


def _ord16(t: torch.Tensor) -> torch.Tensor:
    """fp16 values as integers in value order (+0 and -0 both 0; adjacent finite values differ by 1)."""
    b = t.contiguous().view(torch.int16).int()
    return torch.where(b < 0, -(b & 0x7FFF), b)


def _from_ord16(o: torch.Tensor) -> torch.Tensor:
    b = torch.where(o < 0, (-o) | 0x8000, o)
    return b.to(torch.int32).to(torch.int16).view(torch.float16)        # two's-complement wrap keeps the bits


def _ulp32(a: torch.Tensor) -> torch.Tensor:
    """fp32 spacing at |a| (fp64 tensor): 2^(e - 24) for |a| in [2^(e-1), 2^e); 2^-149 below the normal range."""
    _, e = torch.frexp(a.abs())
    return torch.clamp(torch.ldexp(torch.ones_like(a), e - 24), min=2.0 ** -149)


def unit_rows_exact(x: torch.Tensor):
    """tf_unit_rows' arithmetic, stated exactly: (fp16 output, fp32 quotient) of x [..., dim] fp32 / fp16."""
    dim = x.shape[-1]
    xd = x.reshape(-1, dim).double()
    nrm = torch.sqrt((xd * xd).sum(-1, keepdim=True)).float()
    q = (xd / nrm.double()).float()
    return q.half().view(x.shape), q.view(x.shape)


def _near_fp16_midpoint(q: torch.Tensor) -> torch.Tensor:
    """True where the fp32 value q lies within 1 fp32 ulp of a midpoint between two adjacent fp16 values."""
    a = q.double().abs()
    h = q.abs().half()
    o = _ord16(h)
    up, dn = _from_ord16(o + 1).double(), _from_ord16((o - 1).clamp_min(0)).double()
    hd = h.double()
    dist = torch.minimum((a - (hd + up) / 2).abs(), (a - (hd + dn) / 2).abs())
    return dist <= _ulp32(a)


def check_unit_rows(got: torch.Tensor, x: torch.Tensor, tag: str = "", max_exempt: Optional[int] = None) -> dict:
    """Assert that `got` is tf_unit_rows(x): equal to `unit_rows_exact(x)` element for element (±0 alike, NaN exactly
    where the reference is NaN), up to Markstein-case elements (see the module docstring), which are counted, printed
    and capped at `max_exempt` (default numel * 2^-20).  Returns {"exempt", "elements"}."""
    assert got.dtype == torch.float16 and tuple(got.shape) == tuple(x.shape), (got.dtype, tuple(got.shape))
    want, q = unit_rows_exact(x.detach())
    g = got.detach().to(want.device)
    nan_w, nan_g = torch.isnan(want), torch.isnan(g)
    assert torch.equal(nan_w, nan_g), (f"{tag}: {int((nan_g & ~nan_w).sum())} NaN outputs where the reference is "
                                       f"finite, {int((nan_w & ~nan_g).sum())} finite where it is NaN")
    fin = ~nan_w
    assert torch.isfinite(g[fin]).all(), f"{tag}: infinite output"
    d = (_ord16(g) - _ord16(want)).abs()
    d = torch.where(fin, d, torch.zeros_like(d))
    exempt = (d == 1) & _near_fp16_midpoint(q) & fin
    bad = (d != 0) & ~exempt
    n_ex = int(exempt.sum())
    if bad.any():
        dim = x.shape[-1]
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(
            f"{tag}: {int(bad.sum())} of {g.numel()} unit-row elements differ from fp16(x / fp32(||x||)); first at row "
            f"{i // dim} channel {i % dim}: got {g.flatten()[i].item():.8g}, want {want.flatten()[i].item():.8g} "
            f"(fp32 quotient {q.flatten()[i].item():.10g}, {int(d.flatten()[i])} fp16 ulps)")
    cap = int(g.numel() * UNIT_MAX_EXEMPT_FRAC) if max_exempt is None else max_exempt
    print(f"{tag}: unit rows equal to the exact quotient; Markstein-case elements {n_ex} of {g.numel()}")
    assert n_ex <= cap, f"{tag}: {n_ex} elements 1 fp16 ulp off next to a midpoint (at most {cap})"
    return {"exempt": n_ex, "elements": g.numel()}


def ln_affine_f32(norm):
    """The fp32 copies of γ and β the fused kernels read (`CudaOps._affine_f32`), and eps as the fp32 they get."""
    return (norm.weight.detach().float(), norm.bias.detach().float(),
            float(torch.tensor(float(norm.eps), dtype=torch.float32)))


def layernorm_fp64(x: torch.Tensor, norm) -> dict:
    """LayerNorm of fp16 x [..., dim] with the kernel's fp32 γ, β and eps, in fp64, as [rows, dim] tensors: y, the unit
    rows y / ||y||, z = (x - μ) rstd, and per row rstd, var + eps and mean |x|."""
    dim = x.shape[-1]
    g, b, eps = ln_affine_f32(norm)
    xd = x.detach().reshape(-1, dim).double()
    mu = xd.mean(-1, keepdim=True)
    v = ((xd - mu) ** 2).mean(-1, keepdim=True) + eps
    rstd = 1.0 / torch.sqrt(v)
    z = (xd - mu) * rstd
    g, b = g.to(xd.device).double(), b.to(xd.device).double()
    y = z * g + b
    return {"y": y, "unit": y / y.norm(dim=-1, keepdim=True), "z": z, "rstd": rstd, "v": v,
            "abs_mean": xd.abs().mean(-1, keepdim=True), "gamma": g}


def layernorm_deltas(ref: dict, dim: int):
    """(δ_y, δ_u) [rows, dim]: first-order bounds on |ŷ - y| of the kernel's fp32 y and on its fp32 unit-row quotient.

    With u = 2^-24 and s = ceil(dim / 256) register slots per lane (tf_layernorm_rows: one warp per row, lane l holding
    the 8-channel vectors l, l + 32, ...):
      * Σx: each element passes one pair add, at most 4s chained adds in its lane and 5 butterfly adds, so the fp32 sum
        is within (4s + 6) u Σ|x|; the mean multiplies by fp32(1/dim) (u) and rounds (u):
            |Δμ| <= (4s + 8) u A,  A = mean |x|.
      * Σd² (two-pass, d = x - μ̂): d rounds once (2u in d²), the square once (u), each term passes at most 8s chained
        adds and 5 butterfly adds, all terms >= 0; Σ(d_i - Δμ)² = Σd_i² + dim Δμ² because Σd_i = 0; then × fp32(1/dim)
        (2u) and + eps (u):
            |v̂ - v| / v <= (8s + 5 + 6) u + Δμ² / v,   v = var + eps.
      * rstd = rsqrtf(v̂): half the relative error of v̂ plus 2 ulp of rsqrtf (2 ulp <= 4u relative):
            ρ = |v̂ - v| / (2v) + 4u.
      * y = ((x - μ̂) · rstd) · γ + β in fp32 (d, × rstd, × γ, + β: one rounding each; FMA contraction only removes
        roundings):
            δ_y = rstd |γ| |Δμ| + |z γ| (3u + ρ) + u |y|.
      * unit = fp32(ŷ / fp32(sqrt(Σŷ² in fp64))): with ŷ = y + e, |e| <= δ_y, to first order
            δ_u = δ_y / N + |unit| Σ_j |unit_j| δ_y,j / N + 3u |unit|,  N = ||y||,
        the last term being the rounding of the norm (u) and a quotient within 1 ulp (2u).
    Both carry a relative 2^-20 for the neglected second-order terms and one fp32 ulp of the reference for the check's
    own fp64 -> fp32 -> fp16 conversion of the interval ends."""
    s = -(-dim // LN_SLOT_CHANNELS)
    dmu = (4 * s + 8) * U32 * ref["abs_mean"]
    rel_v = (8 * s + 11) * U32 + dmu ** 2 / ref["v"]
    rho = rel_v / 2 + 2 * RSQRTF_ULPS * U32
    zg = (ref["z"] * ref["gamma"]).abs()
    d_y = ref["rstd"] * ref["gamma"].abs() * dmu + zg * (3 * U32 + rho) + U32 * ref["y"].abs()
    unit = ref["unit"]
    n = ref["y"].norm(dim=-1, keepdim=True)
    d_u = d_y / n + unit.abs() * (unit.abs() * d_y).sum(-1, keepdim=True) / n + 3 * U32 * unit.abs()
    margin = lambda d, r: d * (1 + 2.0 ** -20) + _ulp32(r)
    return margin(d_y, ref["y"]), margin(d_u, unit)


def _interval_use(got: torch.Tensor, ref: torch.Tensor, delta: torch.Tensor, what: str, tag: str):
    """Largest fraction of δ that some t with fp16(t) == got must be from ref; asserts it is <= 1 and that got is
    finite.  Returns (max use, fraction of elements not equal to fp16(ref))."""
    g = got.detach().to(ref.device).reshape(ref.shape)
    assert torch.isfinite(g).all(), f"{tag}: {int((~torch.isfinite(g)).sum())} NaN / Inf {what} elements where the " \
                                    "fp64 value is finite"
    o = _ord16(g)
    gd = g.double()
    hi = (gd + _from_ord16(o + 1).double()) / 2          # the rounding interval of got (inf beyond 65504)
    lo = (gd + _from_ord16(o - 1).double()) / 2
    dist = torch.clamp(lo - ref, min=0) + torch.clamp(ref - hi, min=0)
    use = dist / delta
    worst = use.max().item() if use.numel() else 0.0
    if worst > 1.0:
        i = int(use.flatten().argmax())
        dim = ref.shape[-1]
        raise AssertionError(
            f"{tag}: {int((use > 1).sum())} of {use.numel()} {what} elements outside fp16([ref - δ, ref + δ]); worst at "
            f"row {i // dim} channel {i % dim}: got {gd.flatten()[i].item():.8g}, fp64 {ref.flatten()[i].item():.10g}, "
            f"δ {delta.flatten()[i].item():.3g} ({worst:.3g} δ)")
    miss = (g != ref.float().half()).double().mean().item() if g.numel() else 0.0
    return worst, miss


def check_layernorm_rows(y: Optional[torch.Tensor], unit: Optional[torch.Tensor], x: torch.Tensor, norm, n_unit: int,
                         tag: str = "") -> dict:
    """Assert that y = fp16(LN(x)) and unit = fp16 unit rows of LN(x) for x[:n_unit] are what tf_layernorm_rows
    computes: every element within the interval rule of `layernorm_deltas` around `layernorm_fp64`, no NaN / Inf.
    x is fp16 [b, ..., dim] (or [rows, dim]); y None (the frame pass writes none) or x's shape; unit None when
    n_unit == 0, else the shape of x[:n_unit].  Returns the largest fraction of δ used and the fraction of elements
    not correctly rounded, for y and for the unit rows."""
    dim = x.shape[-1]
    ref = layernorm_fp64(x, norm)
    d_y, d_u = layernorm_deltas(ref, dim)
    stats = {}
    if y is not None:
        assert y.dtype == torch.float16 and tuple(y.shape) == tuple(x.shape), (y.dtype, tuple(y.shape))
        stats["y_use"], stats["y_not_rn"] = _interval_use(y, ref["y"], d_y, "y", tag)
    if n_unit:
        assert unit is not None and unit.dtype == torch.float16 and tuple(unit.shape) == tuple(x[:n_unit].shape), \
            (None if unit is None else (unit.dtype, tuple(unit.shape)))
        r = unit.numel() // dim
        stats["u_use"], stats["u_not_rn"] = _interval_use(unit, ref["unit"][:r], d_u[:r], "unit-row", tag)
    return stats


NORM1_PROBES = ("randn", "var_10eps", "var_1eps", "var_0.1eps", "offset_200", "offset_-3000", "constant",
                "outlier_1000", "outlier_30000", "near_60000")


def norm1_probe(kind: str, rows: int, dim: int, generator=None) -> torch.Tensor:
    """fp16 [rows, dim] norm1 inputs of one statistics probe: well-conditioned ("randn": 2z + 0.3), variance near eps
    ("var_<f>eps": σ² = f * 1e-5, μ = 0), a large common offset (μ = 200, σ = 1; μ = -3000, σ = 16), constant rows,
    one outlier channel per row at ±1000 / ±30000, or values near ±60000."""
    z = torch.randn(rows, dim, generator=generator)
    if kind == "randn":
        x = 2 * z + 0.3
    elif kind.startswith("var_"):
        x = z * math.sqrt(float(kind[4:-3]) * 1e-5)
    elif kind == "offset_200":
        x = 200 + z
    elif kind == "offset_-3000":
        x = -3000 + 16 * z
    elif kind == "constant":
        x = (4 * torch.randn(rows, 1, generator=generator)).expand(rows, dim)
    elif kind.startswith("outlier_"):
        x = z.clone()
        col = torch.randint(0, dim, (rows,), generator=generator)
        sign = torch.where(torch.rand(rows, generator=generator) < 0.5, -1.0, 1.0)
        x[torch.arange(rows), col] = sign * float(kind[8:])
    elif kind == "near_60000":
        x = torch.sign(z) * (60000 - 3000 * torch.rand(rows, dim, generator=generator))
    else:
        raise ValueError(kind)
    return x.half()


def norm1_module(dim: int, gamma: str = "positive", generator=None) -> torch.nn.LayerNorm:
    """fp16 LayerNorm(dim) (CPU): γ uniform in [0.5, 1.5] ("positive") or standard normal with every 7th channel 0
    ("signed"); β uniform in [-0.3, 0.3]."""
    norm = torch.nn.LayerNorm(dim)
    with torch.no_grad():
        if gamma == "positive":
            norm.weight.copy_(0.5 + torch.rand(dim, generator=generator))
        else:
            w = torch.randn(dim, generator=generator)
            w[::7] = 0
            norm.weight.copy_(w)
        norm.bias.copy_(0.6 * torch.rand(dim, generator=generator) - 0.3)
    return norm.half()


def guarded_unit_rows(lib, x: torch.Tensor, guard: int = 256) -> torch.Tensor:
    """tf_unit_rows straight through the C ABI (x a [rows, dim] fp32 / fp16 view with unit last stride) into a
    NaN-filled buffer with guard bands.  Asserts that every output element was written and nothing outside, and that
    the call launched once.  Returns the output [rows, dim]."""
    rows, dim = x.shape
    assert x.stride(1) == 1
    buf = torch.full((rows * dim + 2 * guard,), float("nan"), dtype=torch.float16, device=x.device)
    out = buf[guard:guard + rows * dim]
    n0 = lib.tf_launch_count()
    st = lib.tf_unit_rows(x.data_ptr(), int(x.dtype == torch.float32), rows, dim, x.stride(0), out.data_ptr(),
                          torch.cuda.current_stream().cuda_stream)
    assert st == 0, lib.tf_last_error()
    torch.cuda.synchronize()
    assert lib.tf_launch_count() == n0 + (1 if rows else 0)
    assert torch.isnan(buf[:guard]).all() and torch.isnan(buf[guard + rows * dim:]).all(), "write outside the output"
    out = out.view(rows, dim)
    want_nan = torch.isnan(unit_rows_exact(x)[0])
    assert torch.equal(torch.isnan(out), want_nan), "output element left unwritten (or NaN where the reference is not)"
    return out


def guarded_layernorm_rows(lib, x: torch.Tensor, norm, unit_rows: int, y_pitch: Optional[int] = None,
                           unit_pitch: Optional[int] = None, with_y: bool = True, guard: int = 256):
    """tf_layernorm_rows (or, with `with_y=False` and unit rows of every row, tf_layernorm_unit_rows) straight through
    the C ABI, x a [rows, dim] fp16 view, into NaN-filled outputs of row pitch `y_pitch` / `unit_pitch` (default dim)
    with guard bands.  Asserts that exactly the [rows, dim] / [unit_rows, dim] elements were written: not the gap
    columns of a pitch > dim, not the guard bands.  Returns (y or None, unit or None) as [rows, dim] views."""
    rows, dim = x.shape
    assert x.stride(1) == 1 and x.dtype == torch.float16
    gamma, beta, eps = ln_affine_f32(norm)
    gamma, beta = gamma.to(x.device).contiguous(), beta.to(x.device).contiguous()

    def sentinel(n, pitch):
        buf = torch.full((n * pitch + 2 * guard,), float("nan"), dtype=torch.float16, device=x.device)
        return buf, buf[guard:guard + n * pitch].view(n, pitch)

    y_pitch, unit_pitch = y_pitch or dim, unit_pitch or dim
    ybuf, ymat = sentinel(rows, y_pitch) if with_y else (None, None)
    ubuf, umat = sentinel(unit_rows, unit_pitch) if unit_rows else (None, None)
    n0 = lib.tf_launch_count()
    stream = torch.cuda.current_stream().cuda_stream
    if with_y:
        st = lib.tf_layernorm_rows(x.data_ptr(), rows, dim, x.stride(0), gamma.data_ptr(), beta.data_ptr(), eps,
                                   ymat.data_ptr(), y_pitch, umat.data_ptr() if unit_rows else None, unit_pitch,
                                   unit_rows, stream)
    else:
        assert unit_rows == rows and unit_pitch == dim
        st = lib.tf_layernorm_unit_rows(x.data_ptr(), rows, dim, x.stride(0), gamma.data_ptr(), beta.data_ptr(), eps,
                                        umat.data_ptr(), stream)
    assert st == 0, lib.tf_last_error()
    torch.cuda.synchronize()
    assert lib.tf_launch_count() == n0 + (1 if rows and (with_y or unit_rows) else 0)
    outs = []
    for buf, mat, n in ((ybuf, ymat, rows), (ubuf, umat, unit_rows)):
        if buf is None:
            outs.append(None)
            continue
        assert torch.isnan(buf[:guard]).all() and torch.isnan(buf[guard + n * mat.shape[1]:]).all(), \
            "write outside the output"
        assert torch.isnan(mat[:, dim:]).all(), "write into the gap columns of a packed output"
        assert not torch.isnan(mat[:, :dim]).any(), "output element left unwritten"
        outs.append(mat[:, :dim])
    return tuple(outs)
