"""GPU tier (-m gpu): extended attention at the key counts the BASELINE configurations run, against fp64.

* Every UNet level at production head counts (SD1.5 at n = 5 and 10 keyframes, SD2.1 at 768² and n = 5), with
  and without PnP injection: every query row of an uncond, a cond and a source slab, the last head included,
  through `check_ext_attn`'s error model; two launches give identical bits.
* Long rows through `ext_attn_table` with few samples and 2 heads: 40 960 keys (C3), 46 080 (C4, d = 64, single
  and paired kernels), 102 400 and 204 800 (C5 stride 8 / 4), on random and video-like inputs and on the three
  probes of oracle/kernel_checks.py (a dominant key over a tail in the fp16-P rounding bands, a maximum that
  rises in every tile, a maximum that arrives in the last tile more than 126 octaves up).  Each must stay within
  the error model and within 1e-3 * max(1, |ref|).
* One full C5 stride-4 top-level launch (n = 50, S = 4096, 8 heads x 40): with constant V every output equals V
  within the error model; with random V sampled row ranges match fp64.
"""
import pytest
import torch

from oracle.kernel_checks import (ATTN_ABS_FLOOR, ATTN_P_ABS, ATTN_REL_ULP, TAIL_BANDS, attn_accum_rel,
                                  attn_block_n, check_ext_attn, ext_attn_samples, late_jump_probe,
                                  staircase_probe, subnormal_tail_probe)

pytestmark = pytest.mark.gpu

CEILING = 1e-3                      # max |got - ref| / max(1, |ref|) of every long-row and probe case


@pytest.fixture(scope="module")
def ops():
    from tokenflow_b200.ops import CudaOps
    return CudaOps()


def _video_like(shape_q, shape_kv, g, video):
    """q, k, v fp16 on the GPU; `video`: k = randn + 1.5 q of the same token (peaked rows)."""
    q = torch.randn(*shape_q, generator=g, device="cuda")
    k = torch.randn(*shape_kv, generator=g, device="cuda")
    if video:
        reps = -(-shape_kv[0] // shape_q[0])
        k = k + 1.5 * q.repeat(reps, 1, 1)[:shape_kv[0]]
    v = torch.randn(*shape_kv, generator=g, device="cuda")
    return q.half(), k.half(), v.half()


# ------------------------------------------------------------------------------------------------
# every UNet level at production head counts
# ------------------------------------------------------------------------------------------------
SD15 = [(4096, 8, 40), (1024, 8, 80), (256, 8, 160), (64, 8, 160)]
SD21_768 = [(9216, 5, 64), (2304, 10, 64), (576, 20, 64), (144, 20, 64)]
LEVELS = [(S, h, d, n) for n in (5, 10) for (S, h, d) in SD15] + [(S, h, d, 5) for (S, h, d) in SD21_768]


@pytest.mark.parametrize("inject", [False, True])
@pytest.mark.parametrize("S,heads,d,n", LEVELS)
def test_every_unet_level_against_fp64(ops, S, heads, d, n, inject):
    g = torch.Generator(device="cuda").manual_seed(S * n + d)
    dim = heads * d
    q, k, v = _video_like((3 * n, S, dim), (3 * n, S, dim), g, video=True)
    scale = d ** -0.5
    out = ops.ext_attn(q, k, v, heads, scale, inject)
    assert torch.equal(out, ops.ext_attn(q, k, v, heads, scale, inject)), "two launches differ"
    table = ext_attn_samples(n, inject)
    for smp, head in ((n, heads - 1), (3 * n - 1, heads // 2), (n // 2, heads - 1), (2 * n, 0)):
        ch = slice(head * d, (head + 1) * d)
        # video-like rows carry |O| up to ~4, where one fp16 ulp of P and of the output is 2e-3
        check_ext_attn(out[smp:smp + 1, :, ch], q[..., ch], k[..., ch], v[..., ch], [table[smp]], 1, scale,
                       atol=2.5e-3, max_rel=1e-3)


# ------------------------------------------------------------------------------------------------
# long rows: 40 960 to 204 800 keys per query row
# ------------------------------------------------------------------------------------------------
LONG = {"c3_40960": (4096, 10, 40), "c4_46080": (9216, 5, 64), "c5s8_102400": (4096, 25, 40),
        "c5s4_204800": (4096, 50, 40)}
INPUTS = (["random", "video"] + [f"tail_{lo}_{where}" for (lo, _) in TAIL_BANDS for where in ("first", "last")]
          + ["staircase_0.0625", "staircase_0.25", "staircase_1", "late_jump"])


def _long_case(S, KV, d, kind, paired, seed):
    """(q [1, S, 2d], k, v [KV or 2 KV, S, 2d], table, offsets or None) of one long-row case."""
    heads, dim = 2, 2 * d
    scale = d ** -0.5
    g = torch.Generator(device="cuda").manual_seed(seed)
    slabs = 2 * KV if paired else KV
    q, k, v = _video_like((1, S, dim), (slabs, S, dim), g, video=kind == "video")
    table = [(0, 0, 0, KV), (0, 0, KV, KV)] if paired else [(0, 0, 0, KV)]
    gc = torch.Generator().manual_seed(seed)
    offsets = None
    if kind.startswith("tail_"):
        band = next(b for b in TAIL_BANDS if str(b[0]) == kind.split("_")[1])
        offsets = subnormal_tail_probe(q, k[:KV], v, heads, scale, band, kind.split("_")[2], generator=gc)
    elif kind.startswith("staircase_"):
        offsets = staircase_probe(q, k[:KV], heads, scale, float(kind.split("_")[1]), generator=gc)
    elif kind == "late_jump":
        offsets = late_jump_probe(q, k[:KV], heads, scale, generator=gc)
    return q, k, v, table, offsets, heads, scale


def _assert_probe_hit(kind, offsets, S, KV, d):
    """The fp16 q and k realise the offsets the probe was built for."""
    assert offsets.max().item() == 0.0
    if kind.startswith("tail_"):
        lo, hi = next(b for b in TAIL_BANDS if str(b[0]) == kind.split("_")[1])
        top = 0 if kind.endswith("first") else offsets.shape[1] - 1
        assert offsets[:, top].eq(0).all()
        rest = torch.cat([offsets[:, :top], offsets[:, top + 1:]], dim=1)
        assert lo < rest.min().item() and rest.max().item() < hi, (rest.min().item(), rest.max().item())
    elif kind.startswith("staircase_"):
        delta = float(kind.split("_")[1])
        block_n = attn_block_n(d)
        tiles = offsets.view(2, KV, -(-S // block_n), block_n).amax(dim=-1).reshape(2, -1)
        steps = tiles[:, 1:] - tiles[:, :-1]
        assert (steps - delta).abs().max().item() < 0.02 * delta + 1e-3, (steps.min().item(), steps.max().item())
    elif kind == "late_jump":
        block_n = attn_block_n(d)
        assert offsets[:, :-block_n].max().item() < -126.0
        assert offsets[:, -block_n:].max().item() == 0.0


@pytest.mark.parametrize("kind", INPUTS)
@pytest.mark.parametrize("case", sorted(LONG) + ["c4_46080_paired"])
def test_long_rows_against_fp64(ops, case, kind):
    paired = case.endswith("_paired")
    S, KV, d = LONG[case.replace("_paired", "")]
    q, k, v, table, offsets, heads, scale = _long_case(S, KV, d, kind, paired, seed=KV * 131 + len(kind))
    if offsets is not None:
        _assert_probe_hit(kind, offsets, S, KV, d)
    n0 = ops.launch_count()
    out = ops.ext_attn_table(q, k, v, table, heads, scale)
    assert ops.launch_count() - n0 == 1                 # one launch: the paired table runs as one pair
    if offsets is None:
        stats = check_ext_attn(out, q, k, v, table, heads, scale, atol=CEILING, rtol=CEILING)
    else:
        # every query row reads the same logits: all rows equal, and the first and last query tiles are checked
        assert torch.equal(out, out[:, :1].expand_as(out)), "query rows of one probe row differ"
        stats = check_ext_attn(out[:, :128], q, k, v, table, heads, scale, 0, 128, atol=CEILING, rtol=CEILING)
        check_ext_attn(out[:, S - 128:], q, k, v, table, heads, scale, S - 128, 128, atol=CEILING, rtol=CEILING)
    assert stats["max_err_scaled"] < CEILING, stats
    print(f"{case} {kind}: {stats}")


# ------------------------------------------------------------------------------------------------
# one full C5 stride-4 top-level launch: 50 keyframes, 204 800 keys per extended row
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("inject", [False, True])
def test_c5_stride4_top_level(ops, inject):
    n, S, heads, d = 50, 4096, 8, 40
    dim = heads * d
    scale = d ** -0.5
    g = torch.Generator(device="cuda").manual_seed(54 + inject)
    q, k, v = _video_like((3 * n, S, dim), (3 * n, S, dim), g, video=True)
    # constant V: the exact output of every row is V, no oracle needed
    c = (0.5 + 1.5 * torch.rand(dim, generator=g, device="cuda")) * torch.where(
        torch.rand(dim, generator=g, device="cuda") < 0.5, -1.0, 1.0)
    c = c.half()
    out = ops.ext_attn(q, k, c.expand(3 * n, S, dim).contiguous(), heads, scale, inject)
    c64 = c.double().abs()
    for smp, (_, _, _, nkv) in enumerate(ext_attn_samples(n, inject)):
        keys = nkv * S
        eps_l = attn_accum_rel(nkv * -(-S // attn_block_n(d)), attn_block_n(d))
        # A|v| = |ref| = |c|, l >= 1
        bound = 2 * ATTN_REL_ULP * c64 + eps_l * c64 + ATTN_P_ABS * keys * c64 + ATTN_ABS_FLOOR
        err = (out[smp].double() - c.double()).abs()
        assert (err <= bound).all(), f"sample {smp}: {(err / bound).max().item():.3g} of the error model"
        assert (err / c64.clamp_min(1.0)).max().item() < CEILING
    # random V: sampled row ranges against fp64
    out = ops.ext_attn(q, k, v, heads, scale, inject)
    table = ext_attn_samples(n, inject)
    for smp in (0, n, 2 * n - 1, 3 * n - 1):
        for row0 in (0, 1920, S - 128):
            check_ext_attn(out[smp:smp + 1, row0:row0 + 128], q, k, v, [table[smp]], heads, scale, row0, 128,
                           atol=2.5e-3, max_rel=1e-3)
