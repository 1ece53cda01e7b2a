"""ORACLE (test infrastructure) — calibrated checks of the CUDA kernels' outputs.

`check_ext_attn` compares an extended-attention output with the same sample table evaluated in fp64 on
the kernel's fp16 inputs.  Its bounds come from the kernel's arithmetic, not from a fixed tolerance.
tf_ext_attn computes, per query row of N keys in T tiles of B keys (B = 128, or 64 above d = 128),
P = exp2(s * scale * log2(e) - m + 8) with m the running row maximum, so P <= 2^8 (ATTN_P_OFFSET):

  * fp16 P, relative part: 2^-11 of each key's P while P is an fp16 normal (down to 2^-22 of the maximum);
  * fp16 P, absolute part: below that, fp16 subnormals are 2^-24 apart, so each key's P is off by up to
    2^-25 in units of P, i.e. 2^-33 of the row maximum (ATTN_P_ABS), whatever its own size.  Over N keys
    this is N * 2^-33 of the maximum -- not relative to anything, so it grows with the key count;
  * the fp32 normaliser l: each thread adds B / 8 pair sums of a tile into a fresh partial, then the partial
    into its running l (after l *= corr), then 2 shuffle additions and the reciprocal.  Every key passes
    at most B / 8 + 2T + 5 roundings of 2^-24, relative to l;
  * the fp32 numerator O: each tile's P V goes into a fresh tensor-core accumulator (B / 16 k-steps of 16
    products; the tensor core aligns products to the largest addend and keeps about 24 bits, so a product
    may lose 2^-23 of the tile's largest), then O = O * corr + tile with one rounding: T + 2B + 2 roundings
    of 2^-24 relative to A|v| (`attn_accum_rel` holds both sums);
  * the fp16 output (2^-11 relative).

Scaled by the output, with A|v| the same attention applied to |v| and Σ|v| / l the sum of |v| over the row's
keys divided by the row's exact normaliser (the maximum counts 1):

    |got - ref| <= 2^-10 (A|v| + |ref|) + ε(T) A|v| + 2^-33 Σ|v| / l + 2^-24        elementwise,

where 2^-10 is 2^-11 with a 2x margin.  At 204 800 keys (1 600 tiles) ε is 3.0e-4 and the absolute term at
most 2.4e-5 of max|v|.  With the kernel's earlier arithmetic (P <= 1, one fp32 addition per key into the
running l, every k-step's products straight into the running O) they were 2.4e-3 and 6.1e-3, and a row whose
maximum sits in its first tile and whose other keys all sit near 2^-25 of it lost that mass: 0.4 % of the
output on an H100, and the same in a restatement of the normaliser's arithmetic
(tests/test_kernel_checks_cpu.py).  A bound
that scales with the output keeps its power at large n*S, where the softmax averages over many keys and the
outputs shrink.  The relative RMS error is further compared with an emulation of the same rounding (fp32
scores, fp16 P with the offset, fp32 normaliser, fp16 output), which is scale-free.  The fixed north-star
bound max|got - ref| < 1e-3 (BASELINE.json) stays as a ceiling.  `row_chunk` sets how many query rows the
fp64 evaluation holds at once; by default as many as keep one fp64 [rows, keys] matrix near 256 MB.

`subnormal_tail_probe`, `staircase_probe` and `late_jump_probe` put every key of a row at a chosen log2
offset from the row maximum (a dominant key over a tail in a band; a maximum that rises in every tile; a
maximum that arrives in the last tile far above everything before it) and return the offsets the fp16 q and k
realise, so a test can assert that the band it meant was hit.

`check_nn_field` is the one implementation of the NN-field rule for realistic inputs: every index must be a
lawful winner of its row, given the kernel's own fp16 operands, the tensor core's fp32 accumulation error
(`nn_dot_delta`), one rounding to fp16 and the first index among equal fp16 values, with a NaN similarity above
every number as in torch.argmax (`nn_argmax`).  Rows with more than one lawful winner are counted.

`exact_similarity_probe` and `every_fp16_similarity_probe` build operands whose similarities the tensor core
computes exactly in any accumulation order, so that `nn_field_exact` states the one right index of every row;
`assert_exact_similarities` checks the premise.  See `exact_similarity_probe` for the cases its rows hold.

`propagate_exact` restates tf_propagate in numpy float32 from the reference expression, for bit-for-bit
comparison (`bit_equal`); `every_fp16_propagate_inputs` builds a call that feeds it every fp16 bit pattern.

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

import numpy as np
import torch
import torch.nn.functional as F

ATTN_REL_ULP = 2.0 ** -10       # fp16 rounding (2^-11 relative) of P and of the output, with a 2x margin
ATTN_ABS_FLOOR = 2.0 ** -24
ATTN_EMU_FACTOR = 2.0
ATTN_EMU_FLOOR = 1e-5
ATTN_P_OFFSET = 8               # tf_ext_attn.cu kPOffset: P = exp2(s * scale * log2(e) - m + 8) <= 2^8
ATTN_P_ABS = 2.0 ** -(25 + ATTN_P_OFFSET)   # half the fp16 subnormal spacing, in units of the row maximum
ATTN_ROW_CHUNK_BYTES = 256 << 20  # default size of one fp64 [rows, keys] matrix of the evaluation


def attn_block_n(d: int) -> int:
    """Keys per tile of tf_ext_attn at head dim d."""
    return 128 if d <= 128 else 64


def attn_accum_rel(tiles: int, block_n: int) -> float:
    """First-order relative error bound of the kernel's two fp32 running sums over `tiles` key tiles.  The
    normaliser: a thread's pair sums p0 + p1 (1 rounding), its block_n / 8 - 1 additions into the tile's partial,
    per tile one addition into l and one multiplication by corr, then 2 shuffle additions, the reciprocal and the
    product with O.  The numerator: up to 2^-23 of the tile's largest product for each of its block_n products,
    and one FMA per tile."""
    return (block_n // 8 + 2 * tiles + 5 + tiles + 2 * block_n + 2) * 2.0 ** -24


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


def _place_logits(q: torch.Tensor, k: torch.Tensor, heads: int, scale: float, target: torch.Tensor):
    """In place: every query row of q becomes (0, ..., 0, 1, 64) in each head and the last two channels of k carry
    (b2, b1) with 64 b1 + b2 as close to target / (scale log2 e) as fp16 allows, so that every query row sees the
    log2 logit `target[h, c]` (fp64 [heads, keys]) at key c of the flattened k slabs.  The other channels of k
    keep their values (they meet zeros in q).  Returns the realised log2 offsets from each head's row maximum,
    computed in fp64 from the fp16 q and k."""
    KV, S, dim = k.shape
    d = dim // heads
    assert d >= 2 and tuple(target.shape) == (heads, KV * S), (d, tuple(target.shape))
    x = target.double().cpu() / (scale * math.log2(math.e))
    b1 = (x / 64).half()
    b2 = (x - 64 * b1.double()).half()
    q.zero_()
    offsets = torch.empty(heads, KV * S, dtype=torch.float64)
    for h in range(heads):
        c1, c2 = h * d + d - 1, h * d + d - 2
        q[..., c1], q[..., c2] = 64.0, 1.0
        k[..., c1] = b1[h].view(KV, S).to(k.device)
        k[..., c2] = b2[h].view(KV, S).to(k.device)
        s = k[..., h * d:(h + 1) * d].reshape(KV * S, d).double().cpu() @ q[0, 0, h * d:(h + 1) * d].double().cpu()
        t = s * scale * math.log2(math.e)
        offsets[h] = t - t.max()
    return offsets


TAIL_BANDS = ((-25.5, -25.0), (-25.0, -24.0), (-24.0, -14.0))


def subnormal_tail_probe(q, k, v, heads: int, scale: float, band=(-25.5, -25.0), where: str = "first",
                         generator=None):
    """In place: one dominant key per row, the first key of the first k slab (`where="first"`, the first tile) or
    the last key of the last slab ("last", the last tile); every other key's log2 offset from it drawn uniformly
    inside `band` (1/64 octave in from each end).  v becomes constant per channel (±0.5..2), so the exact output
    of every row is that constant.  With P <= 1 the bands (-25.5, -25) and (-25, -24) are where fp16 P rounds to
    0 or 2^-24 and an fp32 sum near 1 drops the key; (-24, -14) is the fp16 subnormal range.  Returns the
    realised offsets (fp64 [heads, keys])."""
    KV, S, dim = k.shape
    lo, hi = band[0] + 2.0 ** -6, band[1] - 2.0 ** -6
    target = lo + (hi - lo) * torch.rand(heads, KV * S, generator=generator, dtype=torch.float64)
    target[:, 0 if where == "first" else -1] = 0.0
    offsets = _place_logits(q, k, heads, scale, target)
    c = (0.5 + 1.5 * torch.rand(dim, generator=generator)) * torch.where(torch.rand(dim, generator=generator) < 0.5,
                                                                       -1.0, 1.0)
    v.copy_(c.half().to(v.device).expand_as(v))
    return offsets


def _tile_index(KV: int, S: int, block_n: int) -> torch.Tensor:
    """Tile of each flattened key (k slab, token) in the kernel's order: slab-major, block_n keys per tile."""
    tps = -(-S // block_n)
    return (torch.arange(KV)[:, None] * tps + torch.arange(S)[None, :] // block_n).reshape(-1)


def staircase_probe(q, k, heads: int, scale: float, delta: float = 1.0, generator=None):
    """In place: the row maximum rises by `delta` octaves in every key tile, so every tile rescales the running
    sums.  Tile t of T has its first key at (t - T + 1) * delta and the rest up to 16 octaves below that.
    Returns the realised offsets (fp64 [heads, keys])."""
    KV, S, dim = k.shape
    tile = _tile_index(KV, S, attn_block_n(dim // heads))
    top = (tile - int(tile.max())).double() * delta
    target = top - 16.0 * torch.rand(heads, KV * S, generator=generator, dtype=torch.float64)
    first = torch.ones(KV * S, dtype=torch.bool)
    first[1:] = tile[1:] != tile[:-1]
    target[:, first] = top[first]
    return _place_logits(q, k, heads, scale, target)


def late_jump_probe(q, k, heads: int, scale: float, gap: float = 130.0, generator=None):
    """In place: the row maximum arrives in the last key tile, `gap` to `gap` + 10 octaves above every key before
    it, so the kernel's rescale factor exp2(m_old - m_new) underflows to zero.  The last tile's keys sit up to 12
    octaves below its maximum.  Returns the realised offsets (fp64 [heads, keys])."""
    KV, S, dim = k.shape
    tile = _tile_index(KV, S, attn_block_n(dim // heads))
    last = tile == tile.max()
    target = -gap - 10.0 * torch.rand(heads, KV * S, generator=generator, dtype=torch.float64)
    target[:, last] = -12.0 * torch.rand(heads, int(last.sum()), generator=generator, dtype=torch.float64)
    target[:, last.nonzero()[0, 0]] = 0.0
    return _place_logits(q, k, heads, scale, target)


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


def _attn_terms(q, k, v, table, heads, scale, row0, r1, row_chunk=None):
    """(ref, A|v|, Σ|v| / l, emulation) as fp64 tensors [len(table), r1 - row0, dim]; l is the row's exact
    normaliser with the maximum counted as 1."""
    _, S, dim = q.shape
    d = dim // heads
    R = r1 - row0
    shape = (len(table), R, dim)
    ref = torch.zeros(shape, dtype=torch.float64, device=q.device)
    absv = torch.zeros_like(ref)
    tail = torch.zeros_like(ref)
    emu = torch.zeros_like(ref)
    sl2 = float(torch.tensor(scale * math.log2(math.e), dtype=torch.float32))   # the kernel's fp32 scale * log2(e)
    for j, (qs, k0, v0, nkv) in enumerate(table):
        chunk = row_chunk or max(1, min(1024, ATTN_ROW_CHUNK_BYTES // (8 * nkv * S)))
        for h in range(heads):
            ch = slice(h * d, (h + 1) * d)
            kk = k[k0:k0 + nkv, :, ch].reshape(nkv * S, d)
            vv = v[v0:v0 + nkv, :, ch].reshape(nkv * S, d)
            k64, v64, k32, v32 = kk.double(), vv.double(), kk.float(), vv.float()
            vsum = v64.abs().sum(dim=0)
            for a in range(row0, r1, chunk):
                b = min(r1, a + chunk)
                qq = q[qs, a:b, ch]
                s64 = (qq.double() @ k64.T) * scale
                e64 = torch.exp(s64 - s64.amax(dim=-1, keepdim=True))
                l64 = e64.sum(dim=-1, keepdim=True)
                ref[j, a - row0:b - row0, ch] = (e64 @ v64) / l64
                absv[j, a - row0:b - row0, ch] = (e64 @ v64.abs()) / l64
                tail[j, a - row0:b - row0, ch] = vsum / l64
                del s64, e64
                t32 = (qq.float() @ k32.T) * sl2
                p32 = torch.exp2(t32 - t32.amax(dim=-1, keepdim=True) + ATTN_P_OFFSET)
                o = (p32.half().float() @ v32) / p32.sum(dim=-1, keepdim=True)
                emu[j, a - row0:b - row0, ch] = o.half().double()
    return ref, absv, tail, emu


def check_ext_attn(got: torch.Tensor, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, table, heads: int,
                   scale: float, row0: int = 0, nrows: Optional[int] = None, *, atol: float = 1e-3,
                   rtol: float = 0.0, max_rel: Optional[float] = None, row_chunk: Optional[int] = None) -> dict:
    """Assert that `got` is `ext_attn_table(q, k, v, table, heads, scale, row0, nrows)` computed correctly.

    q [Q, S, dim], k / v [KV, S, dim] fp16 (the kernel's inputs); `table[j] = (q slab, first k slab, first v
    slab, number of key slabs)` as in `OracleOps.ext_attn_table`.  `got` is [len(table), nrows, dim] fp16;
    only its rows of tokens < S are compared (the kernel leaves the rest unwritten).  `atol` / `rtol` set the
    fixed ceiling |got - ref| < atol + rtol * |ref|; `max_rel` optionally caps the relative RMS error;
    `row_chunk` is the number of query rows evaluated at once (default: about 256 MB per fp64 [rows, keys]).
    Returns the measured statistics, including the ratio of the relative RMS error to the emulation's and
    `max_err_scaled` = max |got - ref| / max(1, |ref|)."""
    _, S, dim = q.shape
    nrows = S if nrows is None else int(nrows)
    r1 = min(S, row0 + nrows)
    assert got.dtype == torch.float16, got.dtype
    assert tuple(got.shape) == (len(table), nrows, dim), (tuple(got.shape), (len(table), nrows, dim))
    assert q.dtype == k.dtype == v.dtype == torch.float16, "check the fp16 tensors the kernel read"
    if r1 <= row0:
        return {"rel": 0.0, "rel_emu": 0.0, "ratio": 1.0, "max_err": 0.0, "bound_use": 0.0, "max_err_scaled": 0.0}
    g = got[:, :r1 - row0].double()
    assert torch.isfinite(g).all(), "NaN or Inf in the attention output"
    ref, absv, tail, emu = _attn_terms(q, k, v, table, heads, scale, row0, r1, row_chunk)

    err = (g - ref).abs()
    block_n = attn_block_n(dim // heads)
    eps_l = torch.tensor([attn_accum_rel(nkv * -(-S // block_n), block_n) for (_, _, _, nkv) in table],
                         dtype=torch.float64, device=ref.device).view(-1, 1, 1)
    bound = ATTN_REL_ULP * (absv + ref.abs()) + eps_l * absv + ATTN_P_ABS * tail + ATTN_ABS_FLOOR
    use = err / bound
    worst = int(use.argmax())
    j, r, c = (worst // (use.shape[1] * use.shape[2]), (worst // use.shape[2]) % use.shape[1], worst % use.shape[2])
    stats = {"max_err": err.max().item(), "bound_use": use.max().item(),
             "max_err_scaled": (err / ref.abs().clamp_min(1.0)).max().item()}
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
    """fp16 similarities of fp16 unit rows, dot products accumulated in fp64: [R, dim] x [C, dim] -> [R, C].
    The unit row of a zero token is NaN (0 / 0), so its similarity row or column is NaN."""
    return (x_unit.double() @ piv_unit.double().T).float().half()


def nn_argmax(sim: torch.Tensor) -> torch.Tensor:
    """Index of each row's maximum in the order of torch.argmax, which the reference takes over its similarities:
    a NaN ranks above every number, and the first of equal values, or of several NaNs, wins.  A row that is all NaN
    (a zero frame token) gives 0, a NaN column (a zero pivot token) wins every row it reaches."""
    nan = torch.isnan(sim)
    first_nan = nan.to(torch.uint8).argmax(dim=-1)
    best = torch.where(nan, torch.full_like(sim, -math.inf), sim).argmax(dim=-1)
    return torch.where(nan.any(dim=-1), first_nan, best)


def tie_class(sim: torch.Tensor, rows: torch.Tensor, got: torch.Tensor, want: torch.Tensor,
              ulps: float = 1.0) -> torch.Tensor:
    """For rows whose index `got` differs from `want` (the argmax of `sim`): True where the two candidates'
    fp16 similarities lie within `ulps` fp16 ulps (at the winner's magnitude) of each other, i.e. the
    winner depends only on the accumulation order of the dot products."""
    s_want = sim[rows, want].float()
    s_got = sim[rows, got].float()
    ulp = 2.0 ** (torch.floor(torch.log2(s_want.abs().clamp_min(1e-8))) - 10)
    return (s_want - s_got).abs() <= ulps * ulp * 1.001


NN_BLOCK_N = 128                # tf_nn_field.cu kBlockN: key columns per tile
NN_CHUNK = 64                   # kChunkK: channels per shared-memory chunk
NN_KSTEP = 16                   # channels per wgmma k-step
NN_GRID_BITS = 17               # exact probes: every partial sum of a dot stays below 2^17 steps of its grid


def fp16_rn(v: torch.Tensor) -> torch.Tensor:
    """fp64 -> fp16 with a single round-to-nearest-even (`.half()` of a double rounds through fp32, which can round
    twice).  v = m 2^e with m in [0.5, 1) sits in an fp16 binade of spacing 2^(e - 11), 2^-24 below the normal range;
    torch.round is round-half-even, and a result past 65504 becomes inf in the final conversion."""
    _, e = torch.frexp(v)
    q = torch.ldexp(torch.ones_like(v), e - 11).clamp_min(2.0 ** -24)
    return (torch.round(v / q) * q).half()


def nn_dot_delta(dim: int, abs_dot: torch.Tensor) -> torch.Tensor:
    """Bound on |ŝ - s| of the kernel's fp32 similarity ŝ, s the exact dot product of fp16 rows, with
    `abs_dot` = Σ|x_i y_i| (fp64).  The tensor-core model of `attn_accum_rel`: each wgmma k-step adds 16 products
    to the running accumulator, every one of the 17 addends aligned to the largest of them and losing up to 2^-23
    of it, and the sum is rounded to fp32 (2^-24).  Every addend, the accumulator included, is at most Σ|x_i y_i|,
    so one k-step errs by at most (17 * 2^-23 + 2^-24) Σ|x_i y_i| = 35 * 2^-24 Σ|x_i y_i|, and ceil(dim / 16)
    k-steps by ceil(dim / 16) times that.  δ is twice the sum: 2 * ceil(dim / 16) * 35 * 2^-24 * Σ|x_i y_i|.
    (The fp16 rounding of the epilogue is not part of δ: `nn_lawful_winners` maps the interval through it.)"""
    return (2 * -(-dim // NN_KSTEP) * 35 * 2.0 ** -24) * abs_dot


def nn_lawful_winners(sim64: torch.Tensor, abs_dot: torch.Tensor, dim: int) -> torch.Tensor:
    """[R, C] bool for rows without NaN: column c is a lawful winner when some fp32 similarities within δ
    (`nn_dot_delta`) of the exact ones, each rounded to fp16, make c the first maximum.  With [lo16, hi16] the fp16
    values an interval [s - δ, s + δ] can round to, that is hi16(c) > lo16(c') for every c' < c and
    hi16(c) >= lo16(c') for every c' > c."""
    d = nn_dot_delta(dim, abs_dot)
    lo, hi = fp16_rn(sim64 - d).float(), fp16_rn(sim64 + d).float()
    pad = torch.full_like(lo[:, :1], -math.inf)
    before = torch.cat([pad, lo[:, :-1]], dim=1).cummax(dim=1).values
    after = torch.cat([lo[:, 1:], pad], dim=1).flip(1).cummax(dim=1).values.flip(1)
    return (hi > before) & (hi >= after)


def check_nn_field(idx_a: torch.Tensor, idx_b: Optional[torch.Tensor], x_unit: torch.Tensor,
                   piv_unit: torch.Tensor, kf_a: Sequence[int], kf_b: Sequence[int], tag: str = "") -> dict:
    """Assert that (idx_a, idx_b) is `nn_field(x_unit, piv_unit, kf_a, kf_b)` computed correctly.

    x_unit [F, S, dim], piv_unit [K, S, dim] are the fp16 rows the kernel read.  idx_b is read only for frames with
    kf_b >= 0 (the kernel leaves the other rows unwritten).  Every index must be a lawful winner of its row
    (`nn_lawful_winners`); a row with a NaN similarity (a zero token's unit row is NaN) is exact: its first NaN column
    must win, index 0 for a row that is all NaN.  Returns {"ties": the number of rows with more than one lawful winner
    (tie rows: the accumulation order may decide their index), "total": the number of rows}."""
    F, S, dim = x_unit.shape
    assert idx_a.dtype == torch.int32 and tuple(idx_a.shape) == (F, S), (idx_a.dtype, tuple(idx_a.shape))
    any_b = any(int(b) >= 0 for b in kf_b)
    if any_b:
        assert idx_b is not None and idx_b.dtype == torch.int32 and tuple(idx_b.shape) == (F, S)
    else:
        assert idx_b is None
    chunk = max(1, (1 << 24) // max(S, 1))              # rows per evaluation: a few [rows, S] fp64 matrices
    total = multi = 0
    for f in range(F):
        for kf, idx in ((int(kf_a[f]), idx_a), (int(kf_b[f]), idx_b)):
            if kf < 0:
                continue
            got = idx[f].long().to(x_unit.device)
            assert got.min().item() >= 0 and got.max().item() < S, \
                f"frame {f}, keyframe {kf}: index outside [0, {S}) ({got.min().item()}..{got.max().item()})"
            y = piv_unit[kf].double()
            for r0 in range(0, S, chunk):
                xr = x_unit[f, r0:r0 + chunk].double()
                s64 = xr @ y.T
                lawful = nn_lawful_winners(s64, xr.abs() @ y.abs().T, dim)
                nan_row = torch.isnan(s64).any(dim=1)
                g = got[r0:r0 + chunk]
                ok = torch.where(nan_row, g == nn_argmax(s64), lawful.gather(1, g[:, None]).squeeze(1))
                if not ok.all():
                    r = int((~ok).nonzero()[0])
                    sim = fp16_rn(s64[r])
                    want = int(nn_argmax(sim[None])[0])
                    raise AssertionError(
                        f"{tag} frame {f}, keyframe {kf}: {int((~ok).sum())} of the rows {r0}..{r0 + len(g) - 1} have "
                        f"an index that is not a lawful winner; token {r0 + r} has {int(g[r])} (similarity "
                        f"{s64[r, g[r]].item():.9g}, fp16 {sim[g[r]].item():.6g}); its first fp16 maximum is {want} "
                        f"({s64[r, want].item():.9g}, fp16 {sim[want].item():.6g}), lawful winners "
                        f"{lawful[r].nonzero().flatten()[:8].tolist()}")
                multi += int(((lawful.sum(dim=1) > 1) & ~nan_row).sum())
            total += S
    print(f"{tag} nn_field: {multi} of {total} rows with more than one lawful winner")
    return {"ties": multi, "total": total}


# ------------------------------------------------------------------------------------------------
# NN field: probes whose similarities are exact in every accumulation order
# ------------------------------------------------------------------------------------------------
def _token_grid(t: torch.Tensor) -> torch.Tensor:
    """Per row of fp16 t [N, dim]: the largest power of two dividing every channel, in units of 2^-24 (int64; 2^62
    for a zero row).  Every finite fp16 value is a multiple of 2^-24 below 2^16."""
    n = (t.double() * 2.0 ** 24).long()
    low = torch.where(n == 0, torch.full_like(n, 1 << 62), n & -n)
    return low.min(dim=1).values


def _unique_rows(t: torch.Tensor):
    """(distinct rows by bit pattern, inverse map) of fp16 t [N, dim]."""
    u, inv = torch.unique(t.contiguous().view(torch.int16), dim=0, return_inverse=True)
    return u.view(torch.float16), inv


def assert_exact_similarities(x: torch.Tensor, piv: torch.Tensor):
    """Assert the premise of the exact probes for fp16 x [F, S, dim] and piv [K, S, dim]: for every frame token r and
    keyframe token c, with g_r and g_c the power-of-two grids of their channels (`_token_grid`), every product
    x_i y_i is a multiple of g_r g_c and Σ|x_i y_i| < 2^17 g_r g_c.  Every partial sum of the dot, in any order, is
    then a multiple of g_r g_c below 2^17 of them: 17 significant bits, exact in an accumulator that keeps 24 bits of
    its largest addend, and exact in fp32 and fp64."""
    dim = x.shape[-1]
    xs, _ = _unique_rows(x.reshape(-1, dim).cpu())
    ys = piv.reshape(-1, dim).cpu()
    assert torch.isfinite(xs).all() and torch.isfinite(ys).all(), "the exact premise needs finite operands"
    gx, gy = _token_grid(xs).double() * 2.0 ** -24, _token_grid(ys).double() * 2.0 ** -24
    a = xs.double().abs() @ ys.double().abs().T
    bound = 2.0 ** NN_GRID_BITS * gx[:, None] * gy[None, :]
    if not (a < bound).all():
        r, c = (int(v) for v in (a >= bound).nonzero()[0])
        raise AssertionError(f"exact-similarity premise: Σ|x_i y_i| = {a[r, c].item():.9g} for distinct frame row {r} "
                             f"and keyframe token {c}, not below 2^{NN_GRID_BITS} grid steps ({bound[r, c].item():.3g})")


def nn_field_exact(x: torch.Tensor, piv: torch.Tensor, kf_a: Sequence[int], kf_b: Sequence[int]):
    """The NN field stated outright: per frame f and keyframe kf, the dot products in fp64, one rounding to fp16
    (`fp16_rn`), then `nn_argmax`.  It is the kernel's one right answer where `assert_exact_similarities` holds, or
    where every dot has a single nonzero product (`every_fp16_similarity_probe`).  Evaluated once per distinct frame
    row.  Returns CPU int32 (idx_a, idx_b) [F, S]; idx_b is None when no frame has a second keyframe, and -1 in the
    rows of frames without one."""
    F, S, dim = x.shape
    x, piv = x.cpu(), piv.cpu()
    idx_a = torch.full((F, S), -1, dtype=torch.int32)
    idx_b = idx_a.clone() if any(int(b) >= 0 for b in kf_b) else None
    for f in range(F):
        u, inv = _unique_rows(x[f])
        for kf, idx in ((int(kf_a[f]), idx_a), (int(kf_b[f]), idx_b)):
            if kf >= 0:
                idx[f] = nn_argmax(fp16_rn(u.double() @ piv[kf].double().T))[inv].int()
    return idx_a, idx_b


# Each case: the similarities of its candidate columns, in grid steps of 2^-14 relative to a base b (an fp16 value
# in [1, 2) with an even mantissa: b = 2^14 + 32 j, one fp16 ulp = 16 steps), in increasing column order, each
# with a placement rule, and which candidate must win.  The fp16 value each rounds to is noted.
#   first: in the first key tile          last: in the last key tile            end: the last column, S - 1
#   pair: c_prev + 1, same thread         thread: same thread as candidate 0 (same c mod 8), a later tile
#   other: same tile as c_prev, another thread of the row's 4-thread merge (another (c mod 8) // 2)
#   any: anywhere after c_prev
NN_PROBE_CASES = {
    # an fp16 tie class inside one thread, within a tile and across tiles: the later exact values are larger
    "tie_same_thread": ([(2, "first"), (4, "pair"), (7, "thread"), (-9, "any")], 0),          # b, b, b, b - 16
    # an fp16 tie class across two threads of the merge; truncation would drop the first to b - 16
    "tie_cross_threads": ([(-3, "any"), (3, "other"), (-23, "any")], 0),                     # b, b, b - 16
    # a midpoint below an odd neighbour rounds down to the even b; rounding half up would pick it
    "rne_midpoint_down": ([(-16, "any"), (1, "any"), (8, "other"), (7, "any")], 1),          # b - 16, b, b, b
    # a midpoint above an odd value rounds up to the even b + 32; truncation leaves b + 16 everywhere
    "rne_midpoint_up": ([(16, "any"), (23, "any"), (24, "any"), (25, "any")], 2),            # b + 16, b + 16, b + 32, b + 32
    # every real similarity negative (near -0.3125, ulp 4 steps, b not used): a padding column (0) would win
    "negative_last_tile": ([(-5124, "first"), (-5121, "any"), (-5116, "last")], 2),           # n - 4, n, n + 4
    "first_tile_winner": ([(80, "first"), (87, "any")], 0),                                  # b + 80, b + 80
    "last_column_winner": ([(0, "first"), (15, "end")], 1),                                  # b, b + 16
}
NN_PROBE_SMALL = ([(90, "any"), (113, "any"), (113, "other"), (112, "any"), (5, "any")], 1)  # exact below 2^-7
NN_PROBE_ABSOLUTE = {"negative_last_tile"}
_PROBE_SEL = 2048               # selector entry of a keyframe token (units 2^-7): -2^15 steps against other groups
_PROBE_ROW_SEL = 16


def _placement(rule: str, chosen: list, S: int, n_tiles: int) -> torch.Tensor:
    """[S] bool: the columns where the next candidate of a case may go (see NN_PROBE_CASES)."""
    c = torch.arange(S)
    prev = chosen[-1] if chosen else -1
    tile = c // NN_BLOCK_N
    ok = c > prev
    if rule == "first":
        return ok & (tile == 0)
    if rule == "last":
        return ok & (tile == n_tiles - 1)
    if rule == "end":
        return ok & (c == S - 1)
    if rule == "pair":
        return ok & (c == prev + 1) & (prev % 2 == 0)
    if rule == "thread":
        return ok & (c % 8 == chosen[0] % 8) & (tile > chosen[0] // NN_BLOCK_N)
    if rule == "other":
        return ok & (tile == prev // NN_BLOCK_N) & ((c % 8) // 2 != (prev % 8) // 2)
    assert rule == "any", rule
    return ok


def exact_similarity_probe(F: int, K: int, S: int, dim: int, generator=None) -> dict:
    """fp16 frame tokens x [F, S, dim] and keyframe tokens piv [K, S, dim] whose similarities the kernel computes
    exactly (`assert_exact_similarities`, asserted here), so every index has one right answer (`nn_field_exact`).

    Layout, in integers times 2^-7 (products in grid steps of 2^-14): channels [0, G) select a group (G = 8, 6 at
    dim 8), then mass channels up to dim - 3, a level channel dim - 2 and a fine channel dim - 1.  Frame tokens are
    copies of G + 1 prototypes, permuted per frame: prototype g < G has 16 in selector channel g, random ±1 / ±2 in
    every mass channel, 16 in the level channel and 1 in the fine channel; prototype G is prototype 0 times 2^-7.
    A keyframe token of group g has -2048 in every selector channel but g (-2^15 steps against every other group),
    random ±1 / ±2 mass, and a level ℓ and fine value t chosen so that its similarity with prototype g is the target
    of its role: 16 ℓ + t = target - mass.  The fine channel holds the low 4 bits that settle ties and midpoints;
    the mass spreads every similarity over every 64-channel chunk and 16-channel k-step, with different amounts for
    the candidates of a case, so that skipping, repeating or misaddressing one changes some index.

    In every keyframe, group 0 holds `NN_PROBE_SMALL`: exact similarities below 2^-7, fp16 subnormals for
    prototype G.  Groups 1 .. G-1 hold the cases of `NN_PROBE_CASES`, rotated from keyframe to keyframe; a case that
    does not fit S is left out.  Every other keyframe token is a filler well below its group's candidates.  Returns
    {"x", "piv" (CPU fp16), "proto" [F, S] (each frame token's prototype), "groups" (G), "cases": [(keyframe,
    prototype, name, candidate columns, winning column)]}."""
    assert dim % 8 == 0 and dim >= 8 and S >= 1
    g_ = generator
    G = 6 if dim == 8 else 8
    n_proto = G + 1
    mass = slice(G, dim - 2)
    n_mass = dim - 2 - G
    n_tiles = -(-S // NN_BLOCK_N)

    def pm12(*shape):
        v = torch.randint(1, 3, shape, generator=g_) * (2 * torch.randint(0, 2, shape, generator=g_) - 1)
        return v.long()

    proto = torch.zeros(n_proto, dim, dtype=torch.long)
    proto[torch.arange(G), torch.arange(G)] = _PROBE_ROW_SEL
    proto[:G, mass] = pm12(G, n_mass)
    proto[:G, dim - 2], proto[:G, dim - 1] = 16, 1
    proto[G] = proto[0]
    proto16 = (proto.double() * 2.0 ** -7).half()
    proto16[G] = (proto[G].double() * 2.0 ** -14).half()
    assert torch.equal(proto16[G].double() * 2 ** 7, proto16[0].double())

    menu = sorted(NN_PROBE_CASES)
    piv = torch.empty(K, S, dim, dtype=torch.float16)
    cases = []
    for k in range(K):
        group = torch.randint(0, G, (S,), generator=g_)
        target = torch.zeros(S, dtype=torch.long)
        free = torch.ones(S, dtype=torch.bool)
        floor = {}
        plan = [(0, "small", NN_PROBE_SMALL)] + [
            (gi, name, NN_PROBE_CASES[name])
            for gi, name in ((gi, menu[((gi - 1) + k * (G - 1)) % len(menu)]) for gi in range(1, G))]
        # place the cases with the tightest rules first
        plan.sort(key=lambda p: (0 if any(r in ("end", "last", "thread") for _, r in p[2][0]) else 1))
        for gi, name, (cands, win) in plan:
            base = 0 if name == "small" or name in NN_PROBE_ABSOLUTE else 2 ** 14 + 32 * int(torch.randint(0, 64, (1,),
                                                                                                             generator=g_))
            chosen = []
            for _, rule in cands:
                options = (free & _placement(rule, chosen, S, n_tiles)).nonzero().flatten()
                if rule == "first" and len(cands) > 1 and cands[1][1] == "pair":
                    options = options[options % 2 == 0]
                if not len(options):
                    break
                room = max(1, len(options) // (len(cands) - len(chosen) + 1))
                chosen.append(int(options[int(torch.randint(0, room, (1,), generator=g_))]))
                free[chosen[-1]] = False
            if len(chosen) < len(cands):
                free[chosen] = True
                continue
            for c, (t, _) in zip(chosen, cands):
                group[c], target[c] = gi, base + t
            floor[gi] = base + min(t for t, _ in cands)
            cases.append((k, gi, name, chosen, chosen[win]))
            if name == "small":
                cases.append((k, G, "small_subnormal", chosen, chosen[win]))
        rest = free.nonzero().flatten()
        fg = group[rest]
        fl = torch.tensor([floor.get(int(g), 2 ** 14 if g else 80) for g in fg], dtype=torch.long)
        drop = torch.where(fg == 0, torch.randint(0, 208, (len(rest),), generator=g_),
                           600 + torch.randint(0, 2000, (len(rest),), generator=g_))
        target[rest] = fl - drop
        target[rest[fg == 0]] = target[rest[fg == 0]].clamp_min(-127)

        y = torch.zeros(S, dim, dtype=torch.long)
        y[:, :G] = -_PROBE_SEL
        y[torch.arange(S), group] = 0
        y[:, mass] = pm12(S, n_mass)
        r = target - (proto[group][:, mass] * y[:, mass]).sum(dim=1)
        lvl = torch.div(r, 16, rounding_mode="floor")
        y[:, dim - 2], y[:, dim - 1] = lvl, r - 16 * lvl
        assert lvl.abs().max() <= 2047, "probe level channel out of fp16 integer range"
        piv[k] = (y.double() * 2.0 ** -7).half()
        assert torch.equal(piv[k].double() * 2 ** 7, y.double())

    x = torch.empty(F, S, dim, dtype=torch.float16)
    pmap = torch.empty(F, S, dtype=torch.long)
    for f in range(F):
        pmap[f] = torch.randperm(S, generator=g_) % n_proto
        x[f] = proto16[pmap[f]]
    assert_exact_similarities(x, piv)
    # the cases decide as designed
    for k, p, name, cols, win in cases:
        got = int(nn_argmax(fp16_rn(proto16[p:p + 1].double() @ piv[k].double().T))[0])
        assert got == win, f"probe case {name} in keyframe {k}: column {got} wins, not {win}"
    return {"x": x, "piv": piv, "proto": pmap, "groups": G, "cases": cases}


FP16_SIM_TOKENS = 65536                 # every fp16 bit pattern once
FP16_SIM_DIM = 8
FP16_SIM_SETS = ("all_patterns", "no_nan", "finite", "signed_zeros")


def every_fp16_similarity_probe(generator=None) -> dict:
    """Keyframes of S = 65 536 tokens whose channel 0 carries fp16 values (every other channel 0), against frame rows
    ±2^k e0, k in [-24, 15]: every dot is a single exact product, so its fp16 rounding is the kernel's similarity in
    any order.  Keyframe 0 holds every bit pattern once (a permutation); 1 the same with each NaN replaced by a
    random non-NaN pattern; 2 with each NaN and ±inf replaced by a random finite one; 3 only ±0.  This pins the
    kernel's total order: the first NaN above +inf, products that overflow fp16 to ±inf, products that round to
    fp16 subnormals or to ±0 (RN-even), -0 equal to +0 so that the first index wins, and duplicates.  Every frame
    holds all 80 multipliers, in its own order.  Returns {"x" [4, S, 8], "piv" [4, S, 8] (CPU fp16), "kf_a",
    "kf_b"}."""
    g_ = generator
    S, dim = FP16_SIM_TOKENS, FP16_SIM_DIM
    pats = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.float16)
    nan, inf = torch.isnan(pats), torch.isinf(pats)

    def refill(bad):
        v = pats.clone()
        good = (~bad).nonzero().flatten()
        v[bad] = pats[good[torch.randint(0, len(good), (int(bad.sum()),), generator=g_)]]
        return v

    sets = [pats, refill(nan), refill(nan | inf),
            (torch.randint(0, 2, (S,), generator=g_, dtype=torch.int32) * -32768).to(torch.int16).view(torch.float16)]
    piv = torch.zeros(len(sets), S, dim, dtype=torch.float16)
    for k, v in enumerate(sets):
        piv[k, :, 0] = v[torch.randperm(S, generator=g_)]
    mult = torch.tensor([s * 2.0 ** e for e in range(-24, 16) for s in (1.0, -1.0)]).half()
    x = torch.zeros(4, S, dim, dtype=torch.float16)
    for f in range(4):
        x[f, :, 0] = mult[torch.randperm(S, generator=g_) % len(mult)]
    return {"x": x, "piv": piv, "kf_a": [0, 1, 2, 3], "kf_b": [1, -1, 3, 0]}


# ------------------------------------------------------------------------------------------------
# NN-indexed propagation (tf_propagate)
# ------------------------------------------------------------------------------------------------
def propagate_exact(A: torch.Tensor, idx_a: torch.Tensor, idx_b: Optional[torch.Tensor], kf_a: Sequence[int],
                    kf_b: Sequence[int], w: Sequence[float], residual: Optional[torch.Tensor],
                    out_dtype: torch.dtype) -> torch.Tensor:
    """tf_propagate restated in numpy float32 from the reference expression (tokenflow_utils.py:361-397).

    A [3, K, S, dim] fp16, idx_a / idx_b [F, S], residual [3F, S, dim] fp16 or None.  For frame f and stream s the
    gathered rows a = A[s, kf_a[f], idx_a[f]] and, when kf_b[f] >= 0, b = A[s, kf_b[f], idx_b[f]] give
    fp32(w * a) + fp32((1 - w) * b): two fp32 products and one fp32 addition, with w and 1 - w in fp32 and no fused
    multiply-add (the reference's `w1 * attn_output1 + (1 - w1) * attn_output2` on an fp32 weight tensor).  A frame
    without a second keyframe is a.  The residual is added in fp32 and the sum rounded once to `out_dtype`
    (float16 or float32).  Returns a CPU tensor [3F, S, dim]."""
    a16 = A.detach().cpu().to(torch.float16).numpy()
    _, K, S, dim = a16.shape
    ia = idx_a.detach().cpu().long().numpy()
    ib = idx_b.detach().cpu().long().numpy() if idx_b is not None else None
    F_ = ia.shape[0]
    out = np.empty((3, F_, S, dim), dtype=np.float32)
    with np.errstate(all="ignore"):          # 0 * inf, inf - inf and overflow are part of the arithmetic
        for f in range(F_):
            a = a16[:, int(kf_a[f])][:, ia[f]].astype(np.float32)
            if int(kf_b[f]) >= 0:
                wf = np.float32(w[f])
                b = a16[:, int(kf_b[f])][:, ib[f]].astype(np.float32)
                a = wf * a + (np.float32(1.0) - wf) * b
            out[:, f] = a
        if residual is not None:
            out += residual.detach().cpu().to(torch.float16).numpy().reshape(3, F_, S, dim).astype(np.float32)
        res = out.reshape(3 * F_, S, dim).astype({torch.float16: np.float16, torch.float32: np.float32}[out_dtype])
    return torch.from_numpy(res)


def bit_equal(got: torch.Tensor, want: torch.Tensor) -> torch.Tensor:
    """Elementwise: both NaN, or the same bit pattern (so +0 and -0 differ).  Both fp16 or both fp32."""
    assert got.dtype == want.dtype and tuple(got.shape) == tuple(want.shape), (got.dtype, want.dtype, got.shape,
                                                                              want.shape)
    got, want = got.detach().cpu(), want.detach().cpu()
    bits = {torch.float16: torch.int16, torch.float32: torch.int32}[got.dtype]
    return (got.view(bits) == want.view(bits)) | (torch.isnan(got) & torch.isnan(want))


FP16_PATTERN_SIDE = 256                # S = dim = 256: one [S, dim] slab holds all 65 536 fp16 bit patterns


def every_fp16_propagate_inputs(weights: Sequence[float], generator=None) -> dict:
    """A tf_propagate call whose operands hold every fp16 bit pattern: ±0, subnormals, ±inf, NaNs, the largest
    finite values (whose sums overflow) and values whose blend lands on fp16 midpoints.  One keyframe slab is
    S x dim = 256 x 256 = 65 536 elements.  Stream a (keyframe 1, identity indices) holds the patterns in order in
    stream 0 and in two fixed permutations in streams 1 and 2; stream b (keyframe 0) holds another permutation per
    stream, gathered through a different row permutation in every frame; the residual is an independent permutation
    per frame and stream.  Frames: one per entry of `weights`, then w = 1 with a second keyframe (1 - w = 0, so
    0 * inf gives NaN), then one frame without a second keyframe.  Returns CPU tensors, keyword arguments of
    `propagate_exact` and `CudaOps.propagate` (without `out_dtype`)."""
    S = dim = FP16_PATTERN_SIDE
    pats = torch.arange(-32768, 32768, dtype=torch.int16).view(torch.float16)
    perm = lambda: torch.randperm(S * dim, generator=generator)
    kf_a = [1] * (len(weights) + 2)
    kf_b = [0] * (len(weights) + 1) + [-1]
    w = [float(x) for x in weights] + [1.0, 1.0]
    F_ = len(kf_a)
    A = torch.empty(3, 2, S, dim, dtype=torch.float16)
    for s in range(3):
        A[s, 1] = (pats if s == 0 else pats[perm()]).view(S, dim)
        A[s, 0] = pats[perm()].view(S, dim)
    idx_a = torch.arange(S, dtype=torch.int32).repeat(F_, 1)
    idx_b = torch.stack([torch.randperm(S, generator=generator) for _ in range(F_)]).int()
    residual = torch.stack([pats[perm()].view(S, dim) for _ in range(3 * F_)])
    return dict(A=A, idx_a=idx_a, idx_b=idx_b, kf_a=kf_a, kf_b=kf_b, w=w, residual=residual)


# ------------------------------------------------------------------------------------------------
# GroupNorm (tf_group_norm_nhwc)
# ------------------------------------------------------------------------------------------------
GN_MAX_THREADS = 512            # tf_body.cu kGnMaxThreads
GN_STATS_CHUNK_BYTES = 64 << 10  # kGnStatsChunkBytes
GN_APPLY_CHUNK_BYTES = 128 << 10  # kGnApplyChunkBytes
GN_G4_APPLY_CHUNKS_PER_SAMPLE = 64  # kGnG4ApplyChunksPerSample
GN_WS_REL_TOL = 2.0 ** -16       # observed on one H100 80GB HBM3 (400 W): at most 7.6e-8 (Σd) and 2.6e-7 (Σd²) over
                                 # the 222 shapes of tests/test_gpu_body_kernels.py, 4.9e-8 / 6.5e-8 at the real UNet
                                 # sites; a dropped pixel moves a chunk by >= 2^-12


def gn_layout(hw: int, c: int, groups: Optional[int] = None) -> dict:
    """tf_body.cu `gn_layout`: one thread per 8-channel column, `rows` pixel rows per CTA, and the pixel chunk of a
    statistics / apply CTA (a multiple of `rows` of about 64 / 128 KB of input).  At 4 channels per group
    (c == 4 * groups) the library takes `gn_layout_g4`: the apply chunk is at least 1/64 of the sample, rounded up to
    whole CTA rows."""
    cols = c // 8
    rows = max(1, GN_MAX_THREADS // cols)

    def chunk(nbytes):
        px = nbytes // (2 * c)
        px = -(-px // rows) * rows
        return max(px, rows)

    stats_px, apply_px = chunk(GN_STATS_CHUNK_BYTES), chunk(GN_APPLY_CHUNK_BYTES)
    if groups is not None and c == 4 * groups:
        px = -(-hw // GN_G4_APPLY_CHUNKS_PER_SAMPLE)
        apply_px = max(apply_px, -(-px // rows) * rows)
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
