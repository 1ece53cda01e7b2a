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
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import torch

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
