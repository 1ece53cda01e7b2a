"""CPU tier: the exact NN-field probes of oracle/kernel_checks.py pin every index, and have the power to reject wrong
kernels.

`_restated` states tf_nn_field's arithmetic in numpy: fp16 operands, key columns zero-padded to 128-column tiles, an fp32 dot product in one of three accumulation orders, one fp16 rounding, then the
kernel's scan: each of the 4 threads of a row visits its columns (c mod 8 in {2t, 2t + 1}) tile by tile in increasing
order and takes a value when `!(h <= best) && best == best`, and the 4 threads merge by XOR shuffles (offsets 1, 2),
NaN above every number and the smaller index among equal values or NaNs.  The orders are sequential fp32 additions,
a pairwise fp32 tree, and 16-channel k-steps that truncate every addend to 24 bits of the step's largest before one
fp32 rounding (the tensor-core model of `nn_dot_delta`).  On the probes every order gives `nn_field_exact`'s
indices, so the expectation does not depend on the order.  Each keyword of `_restated` is one plausible kernel bug,
and each must change an index on a probe that tests/test_gpu_nn_field.py runs: the test names the probe case that
catches it.  Everything here is CPU numpy / torch."""
import numpy as np
import pytest
import torch

from oracle.kernel_checks import (NN_BLOCK_N, NN_CHUNK, NN_KSTEP, assert_exact_similarities, every_fp16_similarity_probe,
                                  exact_similarity_probe, fp16_rn, nn_argmax, nn_field_exact)

# the probe of the row-width sweep in tests/test_gpu_nn_field.py
KF_A, KF_B = [0, 1, 1, 2, 0, 1], [-1, 0, 2, -1, 1, -1]
NAN_PIVOT = (2, 141)            # keyframe 2, token 141: last key tile, thread 2 of the merge (141 mod 8 = 5)
NAN_FRAME = (1, 77)


def width_probe(dim, S=200, seed=None):
    """The GPU file's row-width probe: F = 6, K = 3, S = 200, with a NaN pivot token (a zero token's unit row) in
    keyframe 2 and a NaN frame token."""
    pr = exact_similarity_probe(len(KF_A), 3, S, dim, generator=torch.Generator().manual_seed(dim if seed is None
                                                                                                 else seed))
    x, piv = pr["x"].clone(), pr["piv"].clone()
    if S > NAN_PIVOT[1]:
        piv[NAN_PIVOT] = float("nan")
    if S > NAN_FRAME[1]:
        x[NAN_FRAME] = float("nan")
    return dict(pr, x=x, piv=piv, kf_a=KF_A, kf_b=KF_B)


# ------------------------------------------------------------------------------------------------
# the kernel restated
# ------------------------------------------------------------------------------------------------
def _dots(xr, y, order, kmask=None):
    """fp32 dots of one fp16 row xr [D] with y [C, D] in an accumulation order; kmask [D] zeroes skipped channels."""
    p = xr.astype(np.float32)[None, :] * y.astype(np.float32)          # exact: 11 x 11 significant bits
    if kmask is not None:
        p = np.where(kmask[None, :], p, np.float32(0))
    C, D = p.shape
    if order == "sequential":
        acc = np.zeros(C, np.float32)
        for i in range(D):
            acc = acc + p[:, i]
        return acc
    if order == "pairwise":
        n = 1 << (D - 1).bit_length()
        q = np.concatenate([p, np.zeros((C, n - D), np.float32)], axis=1)
        while q.shape[1] > 1:
            q = q[:, 0::2] + q[:, 1::2]
        return q[:, 0]
    assert order == "kstep_truncated"
    acc = np.zeros(C, np.float64)
    for k in range(0, D, NN_KSTEP):
        a = np.concatenate([acc[:, None], p[:, k:k + NN_KSTEP].astype(np.float64)], axis=1)
        big = np.abs(a).max(axis=1, keepdims=True)
        _, e = np.frexp(np.where(np.isfinite(big), big, 1.0))
        q = np.ldexp(1.0, e - 24)                                        # 24 bits of the largest addend
        a = np.where(np.isfinite(a), np.trunc(a / q) * q, a)
        acc = a.sum(axis=1).astype(np.float32).astype(np.float64)
    return acc.astype(np.float32)


def _round16(acc, mutant):
    if mutant == "fp32_compare":
        return acc
    h = acc.astype(np.float16)
    if mutant == "fp16_truncation":
        over = np.abs(h.astype(np.float32)) > np.abs(acc)
        h = np.where(over, np.nextafter(h, np.float16(0)), h)
    return h.astype(np.float32)


def _scan(h, S, mutant):
    """The kernel's epilogue and merge on fp16 similarities h [U, S_pad]: the index thread 0 of each row writes."""
    U, S_pad = h.shape
    best = np.full((U, 4), -np.inf, np.float32)
    idx = np.zeros((U, 4), np.int64)
    lane = np.arange(4)
    limit = S + 1 if mutant == "tile_bound_le_S" else S
    for n0 in range(0, S_pad, NN_BLOCK_N):
        for jb in range(NN_BLOCK_N // 8):
            for e in range(2):
                c = n0 + 8 * jb + 2 * lane + e
                hc = h[:, c]
                keep = (hc < best) if mutant == "ge_epilogue" else (hc <= best)
                take = (c < limit)[None, :] & ~keep & (best == best)
                best = np.where(take, hc, best)
                idx = np.where(take, c[None, :], idx)
    for off in (1, 2):
        ob, oi = best[:, lane ^ off], idx[:, lane ^ off]
        o_nan, b_nan = ob != ob, best != best
        if mutant == "merge_no_nan_rule":
            take = (ob > best) | ((ob == best) & (oi < idx))
        else:
            first = (oi > idx) if mutant == "merge_larger_index" else (oi < idx)
            take = (~b_nan & ~(ob <= best)) | (((ob == best) | (o_nan & b_nan)) & first)
        best, idx = np.where(take, ob, best), np.where(take, oi, idx)
    return idx[:, 0]


def _restated(x, piv, kf_a, kf_b, order="sequential", mutant=None):
    """tf_nn_field on CPU: (idx_a, idx_b) as nn_field_exact returns them."""
    F, S, dim = x.shape
    nkc = dim // NN_CHUNK if mutant == "skip_last_partial_chunk" else -(-dim // NN_CHUNK)
    S_pad = -(-S // NN_BLOCK_N) * NN_BLOCK_N
    # the zero-filled channels past dim add exact zeros: the dots run over the real ones
    xs = x.numpy()
    ys = np.zeros((piv.shape[0], S_pad, dim), np.float16)
    ys[:, :S] = piv.numpy()
    kmask = np.arange(dim) < nkc * NN_CHUNK
    if mutant == "kstep_wrong_swizzle_row":
        # the second k-step of every chunk reads the B operand of the neighbouring token row of the swizzle atom
        ks = (np.arange(dim) % NN_CHUNK) // NN_KSTEP == 1
        ys[:, :, ks] = ys[:, np.arange(S_pad) ^ 1][:, :, ks]
    idx_a = torch.full((F, S), -1, dtype=torch.int32)
    idx_b = idx_a.clone() if any(b >= 0 for b in kf_b) else None
    for f in range(F):
        u, inv = np.unique(xs[f].view(np.int16), axis=0, return_inverse=True)
        u = u.view(np.float16)
        for kf, idx in ((kf_a[f], idx_a), (kf_b[f], idx_b)):
            if kf < 0:
                continue
            with np.errstate(all="ignore"):
                h = np.stack([_round16(_dots(u[i], ys[kf], order, kmask), mutant) for i in range(len(u))])
            idx[f] = torch.from_numpy(_scan(h, S, mutant)[inv.reshape(-1)]).int()
    return idx_a, idx_b


def _cases_caught(pr, got, want):
    """Names of the probe cases (and the NaN tokens) on whose rows `got` differs from `want`."""
    caught = set()
    diff = [(got[i] != want[i]) if want[i] is not None else None for i in range(2)]
    for k, p, name, _, _ in pr.get("cases", []):
        for tab, d in ((pr["kf_a"], diff[0]), (pr["kf_b"], diff[1])):
            for f, kf in enumerate(tab):
                if kf == k and bool((d[f] & (pr["proto"][f] == p)).any()):
                    caught.add(name)
    if bool(diff[0].any()) or (diff[1] is not None and bool(diff[1].any())):
        caught.add("any")
    return caught


# ------------------------------------------------------------------------------------------------
# the expectation is the restated kernel's, in every accumulation order
# ------------------------------------------------------------------------------------------------
ORDERS = ["sequential", "pairwise", "kstep_truncated"]
WIDTHS = [8, 16, 24, 56, 64, 72, 120, 136, 320, 640, 648, 1280, 2560, 4096]


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("dim", WIDTHS)
def test_restatement_gives_the_exact_indices_in_every_order(dim, order):
    pr = width_probe(dim)
    want = nn_field_exact(pr["x"], pr["piv"], KF_A, KF_B)
    got = _restated(pr["x"], pr["piv"], KF_A, KF_B, order)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    # the NaN rule: the NaN pivot token wins every row against keyframe 2, the NaN frame token gets 0
    assert (want[1][2] == NAN_PIVOT[1]).all() and (want[0][3] == NAN_PIVOT[1]).all()
    assert want[0][NAN_FRAME] == 0 and want[1][NAN_FRAME] == 0


@pytest.mark.parametrize("S", [1, 2, 7, 127, 129, 257])
def test_restatement_gives_the_exact_indices_at_small_token_counts(S):
    pr = width_probe(64, S=S, seed=S)
    want = nn_field_exact(pr["x"], pr["piv"], KF_A, KF_B)
    for order in ORDERS:
        got = _restated(pr["x"], pr["piv"], KF_A, KF_B, order)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), order


@pytest.fixture(scope="module")
def fp16_probe():
    pr = every_fp16_similarity_probe(generator=torch.Generator().manual_seed(0))
    return dict(pr, want=nn_field_exact(pr["x"], pr["piv"], pr["kf_a"], pr["kf_b"]))


@pytest.mark.parametrize("order", ["sequential", "kstep_truncated"])
def test_restatement_gives_the_exact_indices_on_every_fp16_similarity(fp16_probe, order):
    pr = fp16_probe
    got = _restated(pr["x"], pr["piv"], pr["kf_a"], pr["kf_b"], order)
    assert torch.equal(got[0], pr["want"][0]) and torch.equal(got[1], pr["want"][1])


def test_every_fp16_similarity_probe_covers_the_total_order(fp16_probe):
    """What the probe pins: the first NaN wins; +inf from an fp16 overflow of a finite product wins over every finite
    value; -0 and +0 tie (the first index wins); products that round to subnormals or to zero."""
    pr = fp16_probe
    x, piv = pr["x"], pr["piv"]
    ia, ib = pr["want"]
    mult = x[:, :, 0]
    v = piv[:, :, 0]
    nan0 = torch.isnan(v[0]).nonzero().flatten()
    assert (ia[0] == nan0[0]).all()                                  # all patterns: the first NaN, every row
    fin2 = v[2].float()
    assert torch.isfinite(fin2).all() and not torch.isnan(v[1]).any()
    # keyframe 2 (finite values) against the largest multiplier: products overflow to ±inf, the first +inf wins
    big = (mult[2] == 2.0 ** 15).nonzero().flatten()
    prod = fp16_rn(fin2.double() * 2.0 ** 15)
    first_inf = int((prod == np.inf).nonzero()[0])
    assert (ia[2, big] == first_inf).all() and (fin2[:first_inf] * 2.0 ** 15 < 65520).all()
    # keyframe 3 (only ±0) ties everywhere: index 0
    assert torch.equal(ia[3], torch.zeros_like(ia[3])) and (v[3] == 0).all() and torch.signbit(v[3]).any()
    # the smallest multiplier rounds most products to zero or a subnormal
    small = fp16_rn(fin2.double() * 2.0 ** -24)
    assert (small == 0).any() and ((small != 0) & (small.abs() < 2.0 ** -14)).any()


def test_the_probe_asserts_its_premise():
    """A single channel off the 2^-7 grid gives a dot with more than 17 significant bits: the builder's premise
    check refuses it."""
    pr = exact_similarity_probe(2, 1, 40, 64, generator=torch.Generator().manual_seed(3))
    assert_exact_similarities(pr["x"], pr["piv"])
    piv = pr["piv"].clone()
    piv[0, 5, 20] += 2.0 ** -9
    with pytest.raises(AssertionError, match="premise"):
        assert_exact_similarities(pr["x"], piv)


# ------------------------------------------------------------------------------------------------
# every chunk and k-step decides
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [8, 16, 24, 40, 56, 64, 72, 128, 136, 200, 320, 640, 648, 1280, 2560, 4096])
def test_every_chunk_and_k_step_decides_some_index(dim):
    """Dropping or doubling any one 16-channel k-step or 64-channel chunk changes at least one index of the width
    probe (evaluated exactly per prototype row and keyframe).  Doubling a block that holds the whole row only scales
    every similarity by 2, which keeps every index."""
    pr = exact_similarity_probe(6, 3, 200, dim, generator=torch.Generator().manual_seed(dim))
    x, piv = pr["x"], pr["piv"]
    protos = torch.stack([x[pr["proto"] == p][0] for p in range(pr["groups"] + 1)]).double()
    y = piv.reshape(-1, dim).double()

    def winners(s):
        return torch.stack([nn_argmax(fp16_rn(s[:, k * 200:(k + 1) * 200])) for k in range(3)])

    want = winners(protos @ y.T)
    for width in (NN_KSTEP, NN_CHUNK):
        for c0 in range(0, dim, width):
            part = protos[:, c0:c0 + width] @ y[:, c0:c0 + width].T
            for sign, what in ((-1, "dropped"), (1, "doubled")):
                if sign > 0 and c0 == 0 and width >= dim:
                    continue
                assert not torch.equal(winners(protos @ y.T + sign * part), want), \
                    f"dim {dim}: channels {c0}..{min(dim, c0 + width) - 1} {what} change no index"


# ------------------------------------------------------------------------------------------------
# planted mutants
# ------------------------------------------------------------------------------------------------
# mutant -> (probe, widths, the probe case that must catch it)
MUTANTS = {
    "fp32_compare": ("width", [64, 648], "tie_same_thread"),
    "fp16_truncation": ("width", [64, 648], "rne_midpoint_up"),
    "ge_epilogue": ("width", [64, 648], "tie_same_thread"),
    "merge_larger_index": ("width", [64, 648], "tie_cross_threads"),
    "merge_no_nan_rule": ("width", [64, 648], "nan_pivot"),
    "skip_last_partial_chunk": ("width", [72, 648], "small"),
    "tile_bound_le_S": ("width", [64, 648], "negative_last_tile"),
    "kstep_wrong_swizzle_row": ("width", [64, 648], "any"),
}


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_planted_mutant_fails_on_a_probe(mutant):
    probe, widths, case = MUTANTS[mutant]
    for dim in widths:
        pr = width_probe(dim)
        want = nn_field_exact(pr["x"], pr["piv"], KF_A, KF_B)
        assert torch.equal(_restated(pr["x"], pr["piv"], KF_A, KF_B)[0], want[0])
        got = _restated(pr["x"], pr["piv"], KF_A, KF_B, mutant=mutant)
        caught = _cases_caught(pr, got, want)
        if case == "nan_pivot":
            # frame 2 reads keyframe 2 as its second keyframe, frame 3 as its first: the NaN token must win
            caught |= {"nan_pivot"} if (got[1][2] != NAN_PIVOT[1]).any() or (got[0][3] != NAN_PIVOT[1]).any() else set()
        print(f"{mutant} at dim {dim}: caught by {sorted(caught)}")
        assert case in caught, f"{mutant} at dim {dim} passes the {case} probe (caught by {sorted(caught)})"


@pytest.mark.parametrize("mutant", ["merge_no_nan_rule", "fp16_truncation", "ge_epilogue"])
def test_planted_mutant_fails_on_every_fp16_similarity(fp16_probe, mutant):
    pr = fp16_probe
    got = _restated(pr["x"], pr["piv"], pr["kf_a"], pr["kf_b"], mutant=mutant)
    assert not torch.equal(got[0], pr["want"][0]) or not torch.equal(got[1], pr["want"][1])
