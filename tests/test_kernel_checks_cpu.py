"""CPU tier: the kernel checkers of oracle/kernel_checks.py have the power to reject wrong kernels.

A plain-torch restatement of tf_ext_attn's arithmetic (128- or 64-key tiles per slab, zero-filled
padding keys masked, online softmax with fp16 P and an fp32 normaliser, fp16 output) must pass
`check_ext_attn`; the same computation with one deliberate mistake each must fail it.  At 204 800 keys
(1 600 tiles) a thread-by-thread restatement of the normaliser shows that the kernel's earlier arithmetic
(P <= 1, one fp32 addition per key) fails the error model on a subnormal-tail probe, that the current one
(P <= 2^8, one addition per tile) meets it on every probe, and that one dropped or stale tile out of 1 600 is
rejected.  Likewise for `check_nn_field` and the NN field's padding guard, first-index rule, fp16 rounding and NaN
order (torch's argmax, which the reference uses, ranks a NaN similarity above every number).  Everything
here is CPU torch: no wrong computation is compiled into the library or run on a GPU."""
import math

import pytest
import torch

from oracle.kernel_checks import (ATTN_P_OFFSET, TAIL_BANDS, attn_block_n, check_ext_attn, check_nn_field,
                                  ext_attn_samples, fp16_rn, late_jump_probe, logit_shift_probe,
                                  negative_similarity_probe, nn_argmax, nn_dot_delta, nn_similarity, staircase_probe,
                                  subnormal_tail_probe, tie_class)


def _flash(q, k, v, table, heads, scale, row0=0, nrows=None, *, leak_pad=False, drop_last_key=False,
           drop_last_partial_tile=False, double_first_tile=False, k_slab_shift=0, scale_factor=1.0,
           v_hi_next_head=False):
    """tf_ext_attn's arithmetic on CPU; each keyword is one plausible kernel bug."""
    _, S, dim = q.shape
    d = dim // heads
    block_n = 128 if d <= 128 else 64
    nrows = S if nrows is None else nrows
    r1 = min(S, row0 + nrows)
    KV = k.shape[0]
    tiles_per_slab = -(-S // block_n)
    sc = scale * scale_factor
    out = torch.zeros(len(table), nrows, dim, dtype=torch.float16)
    for j, (qs, k0, v0, nkv) in enumerate(table):
        for h in range(heads):
            ch = torch.arange(h * d, (h + 1) * d)
            vch = ch.clone()
            if v_hi_next_head and d > 64:
                vch[64:] = ((h + 1) % heads) * d + torch.arange(64, d)
            qq = q[qs, row0:r1][:, ch].float()
            m = torch.full((r1 - row0, 1), -math.inf)
            l = torch.zeros(r1 - row0, 1)
            o = torch.zeros(r1 - row0, d)
            tiles = [(slab, t) for slab in range(nkv) for t in range(tiles_per_slab)]
            if double_first_tile:
                tiles = tiles[:1] + tiles
            for slab, t in tiles:
                n0 = t * block_n
                valid = min(block_n, S - n0)
                last_slab = slab == nkv - 1
                if drop_last_partial_tile and last_slab and valid < block_n:
                    continue
                ks = (k0 + slab + k_slab_shift) % KV
                kt = torch.zeros(block_n, d)
                vt = torch.zeros(block_n, d)
                kt[:valid] = k[ks, n0:n0 + valid][:, ch].float()
                vt[:valid] = v[v0 + slab, n0:n0 + valid][:, vch].float()
                s = qq @ kt.T
                masked = torch.arange(block_n) >= valid
                if leak_pad and valid < block_n:
                    masked[valid] = False
                if drop_last_key and last_slab and t == tiles_per_slab - 1:
                    masked[valid - 1] = True
                s[:, masked] = -math.inf
                m_new = torch.maximum(m, s.amax(dim=-1, keepdim=True) * sc)
                corr = torch.exp(m - m_new)
                p = torch.exp(s * sc - m_new)
                l = l * corr + p.sum(dim=-1, keepdim=True)
                o = o * corr + p.half().float() @ vt
                m = m_new
            out[j, :r1 - row0, h * d:(h + 1) * d] = (o / l).half()
    return out


def _inputs(n, S, heads, d, kind, seed=0):
    g = torch.Generator().manual_seed(seed)
    dim = heads * d
    q, k, v = (torch.randn(3 * n, S, dim, generator=g) for _ in range(3))
    scale = d ** -0.5
    if kind == "peaked":
        q = q * 2.5
    elif kind == "onehot":
        q = q * 7
    q, k, v = q.half(), k.half(), v.half()
    if kind == "probe":
        logit_shift_probe(q, k, heads, scale, generator=g)
    return q, k, v, scale


ACCEPT_SHAPES = [(2, 100, 2, 40), (2, 150, 2, 80), (2, 4, 1, 8), (3, 70, 2, 144), (2, 130, 1, 24)]


@pytest.mark.parametrize("kind", ["flat", "peaked", "onehot", "probe"])
@pytest.mark.parametrize("n,S,heads,d", ACCEPT_SHAPES)
@pytest.mark.parametrize("inject", [False, True])
def test_check_ext_attn_accepts_the_fp16_p_arithmetic(n, S, heads, d, kind, inject):
    q, k, v, scale = _inputs(n, S, heads, d, kind, seed=S + d)
    table = ext_attn_samples(n, inject)
    # near one-hot rows carry |O| ~ |v| ~ 3, where one fp16 ulp is 2e-3: the fixed ceiling scales above unit magnitude
    rtol = 1.5e-3 if kind in ("peaked", "onehot") else 0.0
    stats = check_ext_attn(_flash(q, k, v, table, heads, scale), q, k, v, table, heads, scale, rtol=rtol)
    assert stats["bound_use"] < 0.6, stats
    row0 = 128 if S > 128 else 0
    rows = _flash(q, k, v, table, heads, scale, row0=row0, nrows=S)
    check_ext_attn(rows, q, k, v, table, heads, scale, row0=row0, nrows=S, rtol=rtol)


MUTANTS = {
    "leaked_padding_key": dict(leak_pad=True),
    "dropped_last_key": dict(drop_last_key=True),
    "dropped_last_partial_tile": dict(drop_last_partial_tile=True),
    "first_tile_twice": dict(double_first_tile=True),
    "neighbouring_k_slab": dict(k_slab_shift=1),
    "scale_1pct_off": dict(scale_factor=1.01),
    "v_channels_64_up_from_next_head": dict(v_hi_next_head=True),
}


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
@pytest.mark.parametrize("inject", [False, True])
def test_check_ext_attn_rejects_wrong_kernels_on_the_probe(mutant, inject):
    n, S, heads, d = 2, 150, 2, 80                      # ragged last key tile, d > 64
    q, k, v, scale = _inputs(n, S, heads, d, "probe", seed=7)
    table = ext_attn_samples(n, inject)
    check_ext_attn(_flash(q, k, v, table, heads, scale), q, k, v, table, heads, scale)
    with pytest.raises(AssertionError):
        check_ext_attn(_flash(q, k, v, table, heads, scale, **MUTANTS[mutant]), q, k, v, table, heads, scale)


@pytest.mark.parametrize("mutant", ["neighbouring_k_slab", "scale_1pct_off", "v_channels_64_up_from_next_head",
                                    "first_tile_twice"])
def test_check_ext_attn_rejects_wrong_kernels_on_random_inputs(mutant):
    n, S, heads, d = 3, 300, 2, 72
    q, k, v, scale = _inputs(n, S, heads, d, "flat", seed=3)
    table = ext_attn_samples(n, False)
    with pytest.raises(AssertionError):
        check_ext_attn(_flash(q, k, v, table, heads, scale, **MUTANTS[mutant]), q, k, v, table, heads, scale)


def test_check_ext_attn_rejects_nan_and_wrong_shape():
    n, S, heads, d = 2, 40, 1, 16
    q, k, v, scale = _inputs(n, S, heads, d, "flat")
    table = ext_attn_samples(n, False)
    good = _flash(q, k, v, table, heads, scale)
    bad = good.clone()
    bad[1, 3, 2] = float("nan")
    with pytest.raises(AssertionError):
        check_ext_attn(bad, q, k, v, table, heads, scale)
    with pytest.raises(AssertionError):
        check_ext_attn(good[:, :-1], q, k, v, table, heads, scale)
    with pytest.raises(AssertionError):
        check_ext_attn(good.float(), q, k, v, table, heads, scale)


# ------------------------------------------------------------------------------------------------
# NN field
# ------------------------------------------------------------------------------------------------
def _unit(x):
    return (x / x.norm(dim=-1, keepdim=True)).half()


def _nn(xu, pu, kf_a, kf_b, *, pad_leak=False, clamp_leak=False, last_on_ties=False, fp32_compare=False):
    """tf_nn_field's arithmetic on CPU (fp16 similarities, 128-column tiles, zero padding columns); `fp32_compare`
    takes the argmax of the fp32 similarities without rounding them to fp16."""
    F, S, _ = xu.shape
    S_pad = -(-S // 128) * 128
    idx_a = torch.full((F, S), -0x7f7f7f7f, dtype=torch.int32)
    idx_b = idx_a.clone() if any(b >= 0 for b in kf_b) else None
    for f in range(F):
        for kf, idx in ((kf_a[f], idx_a), (kf_b[f], idx_b)):
            if kf < 0:
                continue
            sim = nn_similarity(xu[f], pu[kf]).float()
            if fp32_compare:
                sim = (xu[f].double() @ pu[kf].double().T).float()
            if pad_leak or clamp_leak:
                sim = torch.cat([sim, torch.zeros(S, S_pad - S)], dim=1)
            if last_on_ties:
                best = sim.shape[1] - 1 - sim.flip(1).argmax(dim=-1)
            else:
                best = sim.argmax(dim=-1)
            if clamp_leak:
                best = best.clamp_max(S - 1)
            idx[f] = best.int()
    return idx_a, idx_b


def test_check_nn_field_accepts_argmax_and_ignores_rows_without_second_keyframe():
    g = torch.Generator().manual_seed(0)
    kf_a, kf_b = [0, 1, 1, 2], [-1, 0, -1, 1]
    x, piv = negative_similarity_probe(4, 3, 100, 72, kf_a, generator=g)
    xu, pu = _unit(x), _unit(piv)
    idx_a, idx_b = _nn(xu, pu, kf_a, kf_b)
    assert check_nn_field(idx_a, idx_b, xu, pu, kf_a, kf_b)["ties"] == 0
    assert idx_b[0].eq(-0x7f7f7f7f).all()                  # rows of frames without a second keyframe: never read


@pytest.mark.parametrize("mutant", ["pad_leak", "clamp_leak"])
def test_check_nn_field_rejects_padding_column_leaks(mutant):
    g = torch.Generator().manual_seed(1)
    kf_a, kf_b = [0, 1], [-1, 0]
    x, piv = negative_similarity_probe(2, 2, 100, 64, kf_a, generator=g)
    xu, pu = _unit(x), _unit(piv)
    assert (nn_similarity(xu.view(-1, 64), pu.view(-1, 64)).float() < 0).all()
    idx_a, idx_b = _nn(xu, pu, kf_a, kf_b, **{mutant: True})
    with pytest.raises(AssertionError):
        check_nn_field(idx_a, idx_b, xu, pu, kf_a, kf_b)


def test_check_nn_field_rejects_last_index_on_exact_ties():
    S, dim = 256, 64
    g = torch.Generator().manual_seed(1)
    base = torch.randn(S // 2, dim, generator=g)
    pu = _unit(torch.cat([base, base]).unsqueeze(0))             # token c and c + S/2 are identical
    xu = _unit(base[torch.randperm(S // 2, generator=g)].repeat(2, 1).unsqueeze(0))
    check_nn_field(*_nn(xu, pu, [0], [-1]), xu, pu, [0], [-1])
    with pytest.raises(AssertionError):
        check_nn_field(*_nn(xu, pu, [0], [-1], last_on_ties=True), xu, pu, [0], [-1])


def test_check_nn_field_rejects_a_wrong_index_outside_the_tie_class():
    g = torch.Generator().manual_seed(2)
    x, piv = negative_similarity_probe(1, 1, 64, 32, [0], generator=g)
    xu, pu = _unit(x), _unit(piv)
    idx_a, _ = _nn(xu, pu, [0], [-1])
    idx_a[0, 5] = (idx_a[0, 5] + 1) % 64
    with pytest.raises(AssertionError):
        check_nn_field(idx_a, None, xu, pu, [0], [-1])


def _tie_rows(S=256, dim=320, seed=6):
    """Unit rows of video-like frames (keyframe tokens plus noise) at dim 320, and keyframe tokens c + S/2 that are
    copies of tokens c with every other channel moved one fp16 ulp away from zero: for a frame token near token c the
    copy's exact similarity is larger by about half an fp16 ulp, and often rounds to the same fp16 value."""
    g = torch.Generator().manual_seed(seed)
    base = torch.nn.functional.layer_norm(torch.randn(S // 2, dim, generator=g), (dim,))
    b16 = _unit(base)
    bump = (torch.arange(dim) % 2 == 0).to(torch.int16)                 # every other channel
    away = (b16.view(torch.int16) + bump).view(torch.float16)          # sign and magnitude: one ulp away from 0
    pu = torch.cat([b16, away]).unsqueeze(0)
    x = base[torch.randperm(S // 2, generator=g)].repeat(2, 1) + 0.05 * torch.randn(S, dim, generator=g)
    return _unit(x).unsqueeze(0), pu


def test_check_nn_field_rejects_fp32_compare_on_unit_rows():
    """A kernel that compares its fp32 similarities without rounding them to fp16 picks the later, exactly larger
    column of an fp16 tie.  The old rule (a 1-ulp tie class and a 0.5 % allowance) excused such rows; every one of
    them whose two exact values lie more than 2δ apart is a violation now."""
    xu, pu = _tie_rows()
    S, dim = xu.shape[1:]
    check_nn_field(*_nn(xu, pu, [0], [-1]), xu, pu, [0], [-1])
    got, _ = _nn(xu, pu, [0], [-1], fp32_compare=True)
    want, _ = _nn(xu, pu, [0], [-1])
    s64 = xu[0].double() @ pu[0].double().T
    d = nn_dot_delta(dim, xu[0].double().abs() @ pu[0].double().abs().T)
    rows = (got[0] != want[0]).nonzero().flatten()
    g, w = got[0, rows].long(), want[0, rows].long()
    # every such row is an fp16 tie whose later column is larger by more than both intervals
    s16 = fp16_rn(s64)
    assert (s16[rows, g] == s16[rows, w]).all() and (g > w).all()
    outside = (s64[rows, g] - d[rows, g]) - (s64[rows, w] + d[rows, w])
    clear = int((outside > 0).sum())
    print(f"fp32-compare mutant: {len(rows)} of {S} rows differ, {clear} of them outside the δ band")
    assert clear >= 5
    assert tie_class(s16.float(), rows, g, w).all()                    # the old rule's tie class excuses them all
    with pytest.raises(AssertionError, match="not a lawful winner"):
        check_nn_field(got, None, xu, pu, [0], [-1])


def test_video_like_unit_rows_and_the_delta_band():
    """How many fp16 tie rows video-like data at dim 320 has, and how wide δ is against an fp16 ulp: printed, and δ
    stays below 1/4 ulp of a similarity near 1."""
    g = torch.Generator().manual_seed(8)
    S, dim = 1024, 320
    piv = torch.nn.functional.layer_norm(torch.randn(S, dim, generator=g), (dim,))
    x = piv[torch.randperm(S, generator=g)] + 0.3 * torch.randn(S, dim, generator=g)
    xu, pu = _unit(x), _unit(piv)
    s64 = xu.double() @ pu.double().T
    s16 = fp16_rn(s64).float()
    top = s16.max(dim=1, keepdim=True).values
    ties = int(((s16 == top).sum(dim=1) > 1).sum())
    d = nn_dot_delta(dim, xu.double().abs() @ pu.double().abs().T)
    print(f"video-like dim {dim}: {ties} of {S} rows with an fp16 tie at the maximum; δ at most {d.max().item():.3g}")
    assert d.max().item() < 2.0 ** -11 / 4
    assert check_nn_field(nn_argmax(s16).int()[None], None, xu[None], pu[None], [0], [-1])["total"] == S


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_torch_argmax_returns_the_first_nan_and_nn_argmax_agrees(dtype):
    """The reference takes torch.argmax over its similarities: a NaN ranks above every number, +inf included, and
    the first NaN of a row wins; `nn_argmax` states that order without relying on it."""
    nan, inf = float("nan"), float("inf")
    sim = torch.tensor([[0.1, nan, 0.9, nan], [nan, nan, nan, nan], [0.2, 0.7, 0.7, -0.1], [inf, 0.3, nan, 1.0],
                        [-1.0, -2.0, -1.0, -3.0]], dtype=dtype)
    want = [1, 0, 1, 2, 0]
    assert sim.argmax(dim=-1).tolist() == want
    assert nn_argmax(sim).tolist() == want
    g = torch.Generator().manual_seed(5)
    big = torch.randn(64, 700, generator=g).to(dtype)
    big[torch.rand(64, 700, generator=g) < 0.004] = nan
    big[3] = nan
    big[7, 699] = nan
    assert torch.isnan(big).any(dim=-1).sum() > 10
    assert torch.equal(big.argmax(dim=-1), nn_argmax(big))


def _zero_token_inputs(S=200, dim=64, seed=4):
    """Unit rows of a video-like pair of frames with zero tokens: pivot token 150 of keyframe 1 and tokens 21 and
    130 of keyframe 0 (NaN columns), and token 77 of frame 1 (a NaN row)."""
    g = torch.Generator().manual_seed(seed)
    piv = torch.nn.functional.layer_norm(torch.randn(2, S, dim, generator=g), (dim,))
    x = piv[[1, 0]][:, torch.randperm(S, generator=g)] + 0.3 * torch.randn(2, S, dim, generator=g)
    piv[1, 150] = 0
    piv[0, [21, 130]] = 0
    x[1, 77] = 0
    return _unit(x), _unit(piv)


def test_check_nn_field_requires_the_first_nan_column_and_index_0_for_a_nan_row():
    xu, pu = _zero_token_inputs()
    kf_a, kf_b = [1, 1], [-1, 0]
    assert torch.isnan(pu[1, 150]).all() and torch.isnan(xu[1, 77]).all()
    idx_a, idx_b = _nn(xu, pu, kf_a, kf_b)
    assert idx_a[0].eq(150).all() and idx_b[1, :77].eq(21).all() and idx_b[1, 77] == 0
    check_nn_field(idx_a, idx_b, xu, pu, kf_a, kf_b)
    # a kernel that never picks a NaN similarity (`h > best` alone) gives the best finite candidate instead
    skip_nan = [torch.where(torch.isnan(s), torch.full_like(s, -float("inf")), s).argmax(dim=-1).int()
                for s in (nn_similarity(xu[0], pu[1]).float(), nn_similarity(xu[1], pu[0]).float())]
    wrong_a = idx_a.clone()
    wrong_a[0] = skip_nan[0]
    with pytest.raises(AssertionError):
        check_nn_field(wrong_a, idx_b, xu, pu, kf_a, kf_b)
    # ... or, with two NaN columns, keeps the later one
    wrong_b = idx_b.clone()
    wrong_b[1, :77] = 130
    with pytest.raises(AssertionError):
        check_nn_field(idx_a, wrong_b, xu, pu, kf_a, kf_b)
    # a NaN row must give index 0
    wrong_row = idx_a.clone()
    wrong_row[1, 77] = skip_nan[1][77] if skip_nan[1][77] != 0 else 1
    with pytest.raises(AssertionError):
        check_nn_field(wrong_row, idx_b, xu, pu, kf_a, kf_b)


# ------------------------------------------------------------------------------------------------
# long rows: the kernel's per-thread arithmetic at 204 800 keys (1 600 tiles)
# ------------------------------------------------------------------------------------------------
def _per_thread(q, k, v, scale, nrows, *, p_offset=ATTN_P_OFFSET, tile_local=True, drop_tile=None, stale_tile=None):
    """tf_ext_attn's arithmetic for the table [(0, 0, 0, KV)], one head, query rows [0, nrows), thread by thread.

    `_flash` sums each tile in one torch sum; here the normaliser is what the kernel adds: 4 threads share a row,
    thread t owning columns 8j + 2t and 8j + 2t + 1 of every tile; each adds its pair sums p0 + p1 in fp32 either
    into a fresh per-tile partial that then goes into its l (`tile_local`, the kernel's arithmetic) or straight
    into l (the earlier kernel, with `p_offset=0`); the final shuffles add (l0 + l1) + (l2 + l3).  Scores,
    m, corr and P are fp32 (exp2 flushing results below 2^-126 to zero, as ex2.approx.ftz does), P is rounded
    to fp16 with P <= 2^p_offset, the P V accumulation is fp64, the output fp16(fp32(O) * fp32(1 / l)).
    `drop_tile` skips one tile; `stale_tile` reads the previous tile's keys and values in its place."""
    KV, S, d = k.shape
    block_n = attn_block_n(d)
    tps = -(-S // block_n)
    sl2 = torch.tensor(scale * math.log2(math.e), dtype=torch.float32)
    qq = q[0, :nrows].float()
    m = torch.full((nrows, 1), -math.inf)
    l = torch.zeros(nrows, 4)
    o = torch.zeros(nrows, d, dtype=torch.float64)
    tiny = 2.0 ** -126
    for t in range(KV * tps):
        if t == drop_tile:
            continue
        slab, n0 = divmod(t - 1 if t == stale_tile else t, tps)
        n0 *= block_n
        valid = min(block_n, S - n0)
        kt, vt = torch.zeros(block_n, d), torch.zeros(block_n, d)
        kt[:valid], vt[:valid] = k[slab, n0:n0 + valid].float(), v[slab, n0:n0 + valid].float()
        s = qq @ kt.T
        s[:, valid:] = -math.inf
        m_new = torch.maximum(m, s.amax(dim=-1, keepdim=True) * sl2)
        corr = torch.exp2(m - m_new)
        corr[corr < tiny] = 0.0
        m = m_new
        l = l * corr
        mneg = p_offset - m_new
        p = (s.double() * sl2.double() + mneg.double()).float().exp2()      # fmaf: one rounding
        p[p < tiny] = 0.0
        pairs = p.view(nrows, block_n // 8, 4, 2)
        pairs = pairs[..., 0] + pairs[..., 1]
        if tile_local:
            part = pairs[:, 0]
            for j in range(1, block_n // 8):
                part = part + pairs[:, j]
            l = l + part
        else:
            for j in range(block_n // 8):
                l = l + pairs[:, j]
        o = o * corr.double() + p.half().double() @ vt.double()
    lsum = (l[:, 0] + l[:, 1]) + (l[:, 2] + l[:, 3])
    return (o.float() * (1.0 / lsum)[:, None]).half().unsqueeze(0)


LONG_S, LONG_KV, LONG_D, LONG_ROWS = 4096, 50, 40, 8          # C5 stride 4: 204 800 keys per row, 1 600 tiles


def _long_inputs(seed, video=True):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(1, LONG_S, LONG_D, generator=g)
    k = torch.randn(LONG_KV, LONG_S, LONG_D, generator=g) + (1.5 * q if video else 0)
    v = torch.randn(LONG_KV, LONG_S, LONG_D, generator=g)
    return q.half(), k.half(), v.half(), LONG_D ** -0.5, g


def _check_long(got, q, k, v, scale):
    return check_ext_attn(got, q, k, v, [(0, 0, 0, LONG_KV)], 1, scale, 0, LONG_ROWS, row_chunk=LONG_ROWS)


@pytest.mark.parametrize("band", [(-25.5, -25.0), (-25.0, -24.0)])
def test_earlier_normaliser_fails_the_error_model_on_the_subnormal_tail(band):
    """P <= 1 and one fp32 addition per key: the thread holding the maximum drops every tail key from l while the
    numerator rounds them to 0 or 2^-24.  At 204 800 keys that is several 1e-3 of the output."""
    q, k, v, scale, g = _long_inputs(1)
    offsets = subnormal_tail_probe(q, k, v, 1, scale, band, "first", generator=g)
    assert band[0] < offsets[0, 1:].min().item() and offsets[0, 1:].max().item() < band[1]
    got = _per_thread(q, k, v, scale, LONG_ROWS, p_offset=0, tile_local=False)
    err = (got.double() - v[0, 0].double()).abs().max().item()
    assert err > 2e-3, err
    with pytest.raises(AssertionError, match="outside the fp16 error model"):
        _check_long(got, q, k, v, scale)
    # the offset alone or the tile partial alone does not repair it
    for p_offset, tile_local in ((ATTN_P_OFFSET, False), (0, True)):
        with pytest.raises(AssertionError):
            _check_long(_per_thread(q, k, v, scale, LONG_ROWS, p_offset=p_offset, tile_local=tile_local),
                        q, k, v, scale)


@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("band", TAIL_BANDS)
def test_kernel_normaliser_meets_the_error_model_on_the_subnormal_tail(band, where):
    q, k, v, scale, g = _long_inputs(2)
    subnormal_tail_probe(q, k, v, 1, scale, band, where, generator=g)
    got = _per_thread(q, k, v, scale, LONG_ROWS)
    stats = _check_long(got, q, k, v, scale)
    assert stats["max_err_scaled"] < 1e-3 and stats["bound_use"] < 0.3, stats


@pytest.mark.parametrize("probe", ["video", "staircase_0.0625", "staircase_1", "late_jump"])
def test_kernel_normaliser_meets_the_error_model_at_1600_tiles(probe):
    q, k, v, scale, g = _long_inputs(3)
    if probe.startswith("staircase"):
        staircase_probe(q, k, 1, scale, float(probe.split("_")[1]), generator=g)
    elif probe == "late_jump":
        offsets = late_jump_probe(q, k, 1, scale, generator=g)
        assert offsets[0, :-128].max().item() < -126
    stats = _check_long(_per_thread(q, k, v, scale, LONG_ROWS), q, k, v, scale)
    assert stats["max_err_scaled"] < 1e-3, stats


@pytest.mark.parametrize("mutant,probe", [("drop_tile", "video"), ("stale_tile", "video"),
                                          ("drop_last_tile", "late_jump"), ("stale_tile", "staircase_1")])
def test_check_ext_attn_rejects_one_wrong_tile_out_of_1600(mutant, probe):
    """One tile dropped or read stale (the previous tile's keys and values) out of 1 600: tile 800 is the first
    tile of slab 25, which holds the key correlated with query rows 0..7 (video-like inputs)."""
    q, k, v, scale, g = _long_inputs(4)
    if probe == "late_jump":
        late_jump_probe(q, k, 1, scale, generator=g)
    elif probe == "staircase_1":
        staircase_probe(q, k, 1, scale, 1.0, generator=g)
    T = LONG_KV * LONG_S // 128
    kw = {"drop_tile": dict(drop_tile=800), "stale_tile": dict(stale_tile=T - 1 if probe != "video" else 800),
          "drop_last_tile": dict(drop_tile=T - 1)}[mutant]
    with pytest.raises(AssertionError):
        _check_long(_per_thread(q, k, v, scale, LONG_ROWS, **kw), q, k, v, scale)
