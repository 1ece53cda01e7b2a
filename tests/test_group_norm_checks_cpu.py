"""CPU tier: `check_group_norm_workspace` (oracle/kernel_checks.py) has the power to reject wrong GroupNorm statistics.

tf_group_norm_nhwc's statistics kernel leaves its per-chunk partial sums (Σd, Σd² of d = fp16(x + bias) - shift)
in the caller's workspace.  Here `gn_layout` is tied to the library's workspace size, a plain-torch restatement of
the statistics pass (fp32 sums over one thread's load batch of <= 4 pixels x 8 channels, then fp64, in the
kernel's chunk / row / column order) must pass the checker, and the same pass with one deliberate mistake each
must fail it.  Nothing here needs a GPU."""
import pytest
import torch

from oracle.kernel_checks import check_group_norm_workspace, gn_layout
from tokenflow_b200 import ops as tf_ops


@pytest.fixture(scope="module")
def lib():
    from tokenflow_b200 import _build
    if not tf_ops.library_path().exists():
        _build.build()
    return tf_ops.load_library()


@pytest.mark.parametrize("c,g", [(8, 1), (64, 1), (72, 8), (80, 8), (256, 32), (320, 32), (2040, 255), (4000, 500),
                                 (4096, 32), (4096, 512), (8, 2), (128, 32), (4096, 1024)])
def test_gn_layout_matches_the_library_workspace_size(lib, c, g):
    L0 = gn_layout(1, c, g)
    hws = {1, 3, 64, 4096, 9216, L0["rows"], L0["stats_px"] - 1, L0["stats_px"], L0["stats_px"] + 1,
           L0["apply_px"] + 1, 2 * L0["apply_px"] + L0["rows"] - 1, 7 * L0["stats_px"] + 5, 64 * L0["apply_px"] + 1}
    for hw in sorted(h for h in hws if h >= 1):
        L = gn_layout(hw, c, g)
        assert L["stats_px"] % L["rows"] == 0 and L["apply_px"] % L["rows"] == 0
        assert L["cols"] * L["rows"] <= L["threads"] <= 512
        for n in (1, 3):
            assert lib.tf_group_norm_nhwc_workspace(n, hw, c, g) == n * g * L["stats_chunks"] * 16, (n, hw)


def _stats_pass(x, bias, groups, *, drop_last_px=False, drop_last_rows=False, chunk_twice=False,
                straddle_to_low_group=False, previous_sample_bias=False):
    """tf_body.cu gn_stats_kernel on CPU: the workspace bytes [N, G, stats_chunks] x (Σd, Σd²).  Each keyword is one
    plausible kernel bug (applied to every sample's last chunk, or to all chunks where noted)."""
    n, c, h, w = x.shape
    hw, cpg = h * w, c // groups
    L = gn_layout(hw, c)
    rows, spx, chunks, cols = L["rows"], L["stats_px"], L["stats_chunks"], L["cols"]
    unroll = 2 if bias is not None else 4
    b = bias
    if previous_sample_bias:
        b = torch.cat([bias[:1], bias[:-1]])                       # sample i reads sample i-1's bias row
    xv = x if b is None else x + b[:, :, None, None]             # fp16 add
    v = xv.permute(0, 2, 3, 1).reshape(n, hw, c).float()
    grp = torch.arange(c) // cpg
    d = v - v[:, :1, grp * cpg]                                   # shift: the group's pixel-0 element, first channel
    credit = grp.clone()
    if straddle_to_low_group:                                     # a group's first channel mid-column -> previous group
        first = torch.arange(groups) * cpg
        first = first[first % 8 != 0]
        credit[first] = grp[first] - 1
    keep = torch.ones(hw, dtype=torch.bool)
    last0 = (chunks - 1) * spx
    if drop_last_px:
        keep[hw - 1] = False
    if drop_last_rows:
        keep[max(last0, hw - rows):] = False
    d = d * keep[None, :, None]
    # a thread's 8-channel column splits into (at most two) group parts; sum each part's channels of one pixel
    col = torch.arange(c) // 8
    part = credit - credit[col * 8]                               # 0: the column's first group, 1: the next one
    pair = col * 2 + part
    d1 = torch.zeros(n, hw, 2 * cols)
    d2 = torch.zeros(n, hw, 2 * cols)
    d1.index_add_(2, pair, d)
    d2.index_add_(2, pair, d * d)
    pair_group = (credit[torch.arange(cols) * 8].repeat_interleave(2) + torch.arange(2).repeat(cols)).clamp_max(groups - 1)
    # pixel q of chunk k at offset j belongs to thread row j % rows and load batch (j // rows) // unroll
    batch = -(-spx // (rows * unroll)) * rows * unroll
    pad = torch.zeros(n, chunks * spx - hw, 2 * cols)
    out = torch.zeros(n, groups, chunks, 2, dtype=torch.float64)
    for j, s in enumerate((d1, d2)):
        s = torch.cat([s, pad], dim=1).view(n, chunks, spx, 2 * cols)
        s = torch.cat([s, s.new_zeros(n, chunks, batch - spx, 2 * cols)], dim=2)
        s = s.view(n, chunks, batch // (rows * unroll), unroll, rows, 2 * cols).sum(3)       # fp32, <= 4 pixels
        s = s.double().sum((2, 3))                                                            # fp64
        per_group = torch.zeros(n, chunks, groups, dtype=torch.float64)
        per_group.index_add_(2, pair_group, s)
        out[..., j] = per_group.permute(0, 2, 1)
    if chunk_twice:
        out[:, :, -1] += out[:, :, 0]                             # chunk 0 counted again in the last chunk
    return out.flatten().view(torch.uint8)


def _case(n, h, w, c, groups, bias, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(n, c, h, w, generator=g) * 1.5 + 3.0 * torch.randn(1, c, 1, 1, generator=g)).half()
    b = (torch.randn(n, c, generator=g) * 2).half() if bias else None
    return x, b


ACCEPT = [(3, 34, 41, 80, 8, True), (3, 34, 41, 80, 8, False), (2, 8, 12, 72, 8, False), (2, 1, 7, 4000, 500, True),
          (2, 33, 33, 256, 32, True), (1, 64, 96, 8, 1, False), (2, 3, 5, 4096, 512, True), (3, 20, 30, 2040, 255, False)]


@pytest.mark.parametrize("n,h,w,c,groups,bias", ACCEPT)
def test_check_group_norm_workspace_accepts_the_kernels_arithmetic(n, h, w, c, groups, bias):
    x, b = _case(n, h, w, c, groups, bias, seed=c + h)
    stats = check_group_norm_workspace(_stats_pass(x, b, groups), x, b, groups, h * w, c)
    assert stats["rel1"] < 2.0 ** -19 and stats["rel2"] < 2.0 ** -19, stats


MUTANTS = ["drop_last_px", "drop_last_rows", "chunk_twice", "straddle_to_low_group", "previous_sample_bias"]


@pytest.mark.parametrize("mutant", MUTANTS)
@pytest.mark.parametrize("c,groups", [(80, 8), (72, 8)])
def test_check_group_norm_workspace_rejects_wrong_statistics(mutant, c, groups):
    """C = 80 / 72 in 8 groups: 10 / 9 channels per group, so columns straddle two groups; 3 samples over 3 chunks
    and a ragged last chunk."""
    n, h, w = 3, 34, 41
    x, b = _case(n, h, w, c, groups, True, seed=5)
    assert gn_layout(h * w, c)["stats_chunks"] >= 3
    check_group_norm_workspace(_stats_pass(x, b, groups), x, b, groups, h * w, c)
    with pytest.raises(AssertionError):
        check_group_norm_workspace(_stats_pass(x, b, groups, **{mutant: True}), x, b, groups, h * w, c)


def test_check_group_norm_workspace_rejects_a_wrong_size():
    n, h, w, c, groups = 2, 8, 12, 72, 8
    x, _ = _case(n, h, w, c, groups, False, seed=1)
    ws = _stats_pass(x, None, groups)
    with pytest.raises(AssertionError):
        check_group_norm_workspace(torch.cat([ws, torch.zeros(16, dtype=torch.uint8)]), x, None, groups, h * w, c)
