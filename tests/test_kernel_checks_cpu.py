"""CPU tier: the kernel checkers of oracle/kernel_checks.py have the power to reject wrong kernels.

A plain-torch restatement of tf_ext_attn's arithmetic (128- or 64-key tiles per slab, zero-filled
padding keys masked, online softmax with fp16 P and an fp32 normaliser, fp16 output) must pass
`check_ext_attn`; the same computation with one deliberate mistake each must fail it.  Likewise for
`check_nn_field` and the NN field's padding guard and first-index rule.  Everything here is CPU torch:
no wrong computation is compiled into the library or run on a GPU."""
import math

import pytest
import torch

from oracle.kernel_checks import (check_ext_attn, check_nn_field, ext_attn_samples, logit_shift_probe,
                                  negative_similarity_probe, nn_similarity)


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


def _nn(xu, pu, kf_a, kf_b, *, pad_leak=False, clamp_leak=False, last_on_ties=False):
    """tf_nn_field's arithmetic on CPU (fp16 similarities, 128-column tiles, zero padding columns)."""
    F, S, _ = xu.shape
    S_pad = -(-S // 128) * 128
    idx_a = torch.full((F, S), -0x7f7f7f7f, dtype=torch.int32)
    idx_b = idx_a.clone() if any(b >= 0 for b in kf_b) else None
    for f in range(F):
        for kf, idx in ((kf_a[f], idx_a), (kf_b[f], idx_b)):
            if kf < 0:
                continue
            sim = nn_similarity(xu[f], pu[kf]).float()
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
