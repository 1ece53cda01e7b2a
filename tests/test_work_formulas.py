"""CPU tier: the algorithmic work formulas behind every roofline number (bench.py, ops.py timing hooks)
reproduce the per-step totals of BASELINE.md §2 / SURVEY.md Appendix D, and the host-side shard / frame
tables hold their invariants for arbitrary sizes."""
import math

import pytest
import torch
from hypothesis import given, settings, strategies as st

from oracle import tokenflow_oracle as O
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.ops import blend_weights, propagate_bytes

SD15_LEVELS = [(4096, 320, 5), (1024, 640, 5), (256, 1280, 5), (64, 1280, 1)]      # (S, dim, blocks)
SD21_768_LEVELS = [(9216, 320, 5), (2304, 640, 5), (576, 1280, 5), (144, 1280, 1)]


def _per_step(levels, N, B):
    K = N // B
    attn = sum(4.0 * K * S * S * dim * (2 * K + 1) * blocks for S, dim, blocks in levels)
    nn = sum(2.0 * B * S * S * dim * (2 * N / B - 1) * blocks for S, dim, blocks in levels)
    prop = 0.0
    for S, dim, blocks in levels:
        per_block = 0.0
        for i in range(K):                                       # one tf_propagate launch per batch, no residual
            kf_a, kf_b = [i] * B, [i - 1 if i > 0 else -1] * B
            per_block += propagate_bytes(B, S, dim, kf_a, kf_b, with_residual=False)
        prop += per_block * blocks
    return attn, nn, prop


@pytest.mark.parametrize("levels,N,B,attn_tf,nn_tf,prop_gb", [
    (SD15_LEVELS, 40, 8, 6.74, 4.41, 3.40),          # C2
    (SD15_LEVELS, 80, 8, 25.72, 9.31, 6.88),         # C3
    (SD21_768_LEVELS, 40, 8, 34.11, 22.32, 7.66),    # C4
    (SD15_LEVELS, 200, 4, 618.6, 24.25, 20.76),      # C5 stride 4
])
def test_per_step_work_matches_baseline_md(levels, N, B, attn_tf, nn_tf, prop_gb):
    attn, nn, prop = _per_step(levels, N, B)
    assert attn / 1e12 == pytest.approx(attn_tf, rel=2e-3)
    assert nn / 1e12 == pytest.approx(nn_tf, rel=2e-3)
    assert prop / 1e9 == pytest.approx(prop_gb, rel=5e-3)


def test_ops_flop_accounting_matches_formula():
    """The flops `CudaOps.ext_attn` / `nn_field` attribute to a launch (timing hooks) are the §8d formulas."""
    n, S, dim = 5, 4096, 320
    assert 4.0 * n * S * S * dim * (2 * n + 1) == pytest.approx(1181.1e9, rel=1e-3)     # Appendix D, C2 top level
    B, pairs = 8, 8 * 2
    per_batch = 2.0 * pairs * S * S * dim
    assert per_batch * (2 * 40 / B - 1) / 2 == pytest.approx(773.1e9, rel=1e-3)


@given(K=st.integers(1, 50), G=st.sampled_from([1, 2, 3, 4, 8]), S=st.integers(1, 10000))
@settings(max_examples=60, deadline=None)
def test_pivotal_shard_covers_every_sample_and_row_once(K, G, S):
    seen, rows = [], []
    m = -(-3 * K // G)
    for r in range(G):
        sh = tfu.PivotalShard(G, r, K)
        assert len(sh.slots) == m
        seen += sh.slots
        for inject in (False, True):
            tab = sh.global_attention_table(inject)
            assert len(tab) == 3 * K
            for i, (qs, k0, v0, nkv) in enumerate(tab):
                assert 0 <= k0 and k0 + nkv <= G * m and 0 <= v0 and v0 + nkv <= G * m
                assert 0 <= qs < G * m
                if i >= K:                                     # extended streams see all K keyframes of the stream
                    assert nkv == K and v0 == (i // K) * K
        row0, nrows = sh.row_split(S)
        rows += range(row0, min(S, row0 + nrows))
    assert seen == list(range(G * m)) and G * m >= 3 * K
    assert rows == list(range(S))                              # every query row on exactly one rank, in order


@given(B=st.integers(1, 16), batches=st.integers(1, 12))
@settings(max_examples=60, deadline=None)
def test_frame_table_is_the_reference_batch_arithmetic(B, batches):
    from tokenflow_b200.editor import TokenFlowEditor
    ed = TokenFlowEditor.__new__(TokenFlowEditor)
    ed.config = {"batch_size": B}
    N = B * batches
    kf_a, kf_b, w = TokenFlowEditor.frame_table(ed, list(range(N)))
    for i in range(batches):
        ref_w = O.blend_weights(i, B) if i > 0 else None
        for f in range(B):
            g = i * B + f
            assert kf_a[g] == i and kf_b[g] == (i - 1 if i > 0 else -1)
            if i > 0:
                assert w[g] == pytest.approx(float(ref_w[f]), abs=1e-7)


@given(B=st.integers(1, 32))
@settings(max_examples=32, deadline=None)
def test_blend_weights_bounds(B):
    w = blend_weights(B)
    assert len(w) == B and all(0.5 < x < 0.7311 + 1e-6 for x in w)          # sigmoid of a ratio in (0, 1]
    assert torch.allclose(torch.tensor(w), O.blend_weights(3, B).float(), atol=1e-7)
