"""ORACLE — test infrastructure, not product code.

A restatement, in plain PyTorch ops, of the arithmetic of TokenFlow's per-denoise-step hot path as
the reference (omerbt/TokenFlow @ 5dd6a69) computes it.  Only `tests/`, `__graft_entry__.smoke()`
and `bench.py`'s CPU-baseline / `--impl reference` legs may import this package; the product
(`tokenflow_b200/`) never does and has no CPU fallback.

Pinning: the reference has no tests / golden vectors of its own (SURVEY.md §4), so this oracle is
pinned against the *unmodified* reference hooks, executed through `oracle/ref_shim.py` by
`oracle/gen_golden.py`; the vectors that run produced are committed under `tests/golden/`, and
`tests/test_oracle_golden.py` re-checks the oracle against them everywhere.

Each function cites the reference lines it restates.  The functions are device agnostic: on CPU
they run in the dtype they are given (fp32 for BASELINE config C1, fp64 for closed-form checks); on
a GPU under `torch.autocast(float16)` they launch exactly the library kernels the reference
launches (cuBLAS bmm → fp16, softmax → fp32, matmul → fp16, argmax first-index), which is the
dtype flow the CUDA kernels must reproduce (SURVEY.md Appendix A, "GPU dtype flow").
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch


# ---------------------------------------------------------------------------------------------
# extended attention  (reference tokenflow_utils.py:114-199 PnP flavour, :224-281 SDEdit flavour)
# ---------------------------------------------------------------------------------------------
def inject_qk(q: torch.Tensor, k: torch.Tensor, n: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """PnP q/k injection, reference tokenflow_utils.py:124-130: the uncond and cond thirds of q
    and k are overwritten with the source third (v is left alone)."""
    q = q.clone()
    k = k.clone()
    q[n:2 * n] = q[:n]
    k[n:2 * n] = k[:n]
    q[2 * n:] = q[:n]
    k[2 * n:] = k[:n]
    return q, k


def extended_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, scale: float,
                       inject: bool = False) -> torch.Tensor:
    """q, k, v: [3n, S, dim] (already projected).  Returns the head-merged attention output
    [3n, S, dim] *before* `to_out` (reference :196-197 / :278-279).

    Source stream: each frame attends to its own S keys (:173,:177 / :266,:270).  Uncond and cond
    streams: each frame's queries attend to the n·S keys of all frames of the same stream, frame
    major (:133-138,:174-175,:178-179 / :235-239,:267-268,:271-272).  Per head: sim = q·kᵀ·scale,
    softmax over keys, ·v.  The K>12 per-frame loop (:165-168,:184-190) is the same arithmetic per
    frame and is therefore not restated separately.
    """
    b, S, dim = q.shape
    n = b // 3
    d = dim // heads
    if inject:
        q, k = inject_qk(q, k, n)

    def split(t):  # [m, S, dim] -> [m, heads, S, d]   (head_to_batch_dim, :140-159)
        return t.reshape(t.shape[0], S, heads, d).permute(0, 2, 1, 3)

    out = []
    for s in range(3):
        qs, ks, vs = (split(t[s * n:(s + 1) * n]) for t in (q, k, v))
        if s > 0:  # extended: keys/values of all n frames, frame-major
            ks = ks.permute(1, 0, 2, 3).reshape(1, heads, n * S, d).expand(n, heads, n * S, d)
            vs = vs.permute(1, 0, 2, 3).reshape(1, heads, n * S, d).expand(n, heads, n * S, d)
        per_head = []
        for j in range(heads):
            sim = torch.bmm(qs[:, j], ks[:, j].transpose(-1, -2)) * scale
            per_head.append(torch.bmm(sim.softmax(dim=-1), vs[:, j]))
        o = torch.stack(per_head, dim=1)                       # [n, heads, S, d]
        out.append(o.permute(0, 2, 1, 3).reshape(n, S, dim))  # batch_to_head_dim (:197)
    return torch.cat(out, dim=0)


# ---------------------------------------------------------------------------------------------
# nearest-neighbour field  (reference tokenflow_utils.py:329-348, util.py:61-69)
# ---------------------------------------------------------------------------------------------
def cosine_sim(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """util.py:66-68: row L2-normalise (no epsilon) then x @ y.T."""
    x = x / x.norm(dim=-1, keepdim=True)
    y = y / y.norm(dim=-1, keepdim=True)
    return x @ y.T


def nn_field(x_src: torch.Tensor, pivots_src: torch.Tensor, batch_idx: int
             ) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """x_src: norm1 output of the SOURCE stream for the B frames of this batch, [B, S, dim].
    pivots_src: cached norm1 output of the source stream for all K keyframes, [K, S, dim].
    Returns (idx1, idx2): int64 [B*S] argmax of cosine similarity against keyframe `batch_idx`,
    and against keyframe `batch_idx-1` (None for batch 0).  `torch.argmax` returns the first
    maximal index (reference :335-343)."""
    dim = x_src.shape[-1]
    batch_idxs = [batch_idx] + ([batch_idx - 1] if batch_idx > 0 else [])
    sim = cosine_sim(x_src.reshape(-1, dim), pivots_src[batch_idxs].reshape(-1, dim))
    if len(batch_idxs) == 2:
        sim1, sim2 = sim.chunk(2, dim=1)
        return sim1.argmax(dim=-1), sim2.argmax(dim=-1)
    return sim.argmax(dim=-1), None


def nn_sim_fp16_emulated(x_src: torch.Tensor, piv: torch.Tensor) -> torch.Tensor:
    """The GPU-autocast value of the similarity matrix, emulated on any device without fp16 GEMM:
    fp32 normalise → RNE to fp16 → dot products accumulated wider than fp32 (fp64) → RNE to fp16.
    x_src [R, dim], piv [C, dim] → fp16 [R, C].  Used by the tests to classify an index mismatch:
    two candidates whose emulated fp16 similarity is equal form a tie class, inside which the
    winner depends only on the fp32 accumulation order of the GEMM (SURVEY.md §7 hard part 1)."""
    xh = (x_src.float() / x_src.float().norm(dim=-1, keepdim=True)).half()
    yh = (piv.float() / piv.float().norm(dim=-1, keepdim=True)).half()
    return (xh.double() @ yh.double().T).float().half()


# ---------------------------------------------------------------------------------------------
# propagation  (reference tokenflow_utils.py:361-397)
# ---------------------------------------------------------------------------------------------
def blend_weights(batch_idx: int, n_frames: int, device=None) -> torch.Tensor:
    """w1[f] = sigmoid(d2/(d1+d2)), reference :375-383.  Depends on f and B only."""
    s = torch.arange(0, n_frames, device=device) + batch_idx * n_frames
    p1 = batch_idx * n_frames + n_frames // 2
    p2 = (batch_idx - 1) * n_frames + n_frames // 2
    d1 = torch.abs(s - p1)
    d2 = torch.abs(s - p2)
    return torch.sigmoid(d2 / (d1 + d2))


def propagate(kf_attn_output: torch.Tensor, idx1: torch.Tensor, idx2: Optional[torch.Tensor],
              batch_idx: int, n_frames: int) -> torch.Tensor:
    """kf_attn_output: cached attn1 output of the pivotal pass, [3K, S, dim].
    idx1/idx2: [B*S] NN indices.  Returns attn_output [3B, S, dim] (reference :362-393):
    batch 0 → rows of keyframe 0 gathered by idx1; otherwise w·A[i][idx1] + (1-w)·A[i-1][idx2]."""
    threeK, S, dim = kf_attn_output.shape
    K = threeK // 3
    A = kf_attn_output.view(3, K, S, dim)
    B = n_frames

    def gather(kf: int, idx: torch.Tensor) -> torch.Tensor:  # [3, B*S, dim]
        return A[:, kf][:, idx.reshape(-1)]

    if idx2 is None:
        out = gather(batch_idx, idx1)
    else:
        w1 = blend_weights(batch_idx, B, device=kf_attn_output.device)
        w1 = w1.view(1, B, 1, 1)
        a1 = gather(batch_idx, idx1).view(3, B, S, dim)
        a2 = gather(batch_idx - 1, idx2).view(3, B, S, dim)
        out = w1 * a1 + (1 - w1) * a2
    return out.reshape(3 * B, S, dim)


# ---------------------------------------------------------------------------------------------
# whole self-attention stage of TokenFlowBlock.forward (reference :311-397), functional form
# ---------------------------------------------------------------------------------------------
class BlockState:
    """What the reference keeps as module attributes between passes (Appendix B)."""
    pivot_hidden_states: Optional[torch.Tensor] = None  # (3, K, S, dim), norm1 output
    kf_attn_output: Optional[torch.Tensor] = None       # [3K, S, dim], attn1 output (after to_out)


def block_self_attention(state: BlockState, hidden_states: torch.Tensor, norm_hidden: torch.Tensor,
                         pivotal_pass: bool, batch_idx: int, attn1) -> torch.Tensor:
    """Returns hidden_states + self-attention contribution (reference :325-397).
    `attn1` is the callable installed on the block's attn1 (the extended-attention closure)."""
    b, S, dim = hidden_states.shape
    n = b // 3
    norm_hidden = norm_hidden.view(3, n, S, dim)
    if pivotal_pass:
        state.pivot_hidden_states = norm_hidden                                  # :326-327
        state.kf_attn_output = attn1(norm_hidden.view(b, S, dim))                # :354-360
        attn_output = state.kf_attn_output
    else:
        idx1, idx2 = nn_field(norm_hidden[0], state.pivot_hidden_states[0], batch_idx)   # :329-348
        attn_output = propagate(state.kf_attn_output, idx1, idx2, batch_idx, n)          # :361-393
    return attn_output + hidden_states                                           # :396-397
