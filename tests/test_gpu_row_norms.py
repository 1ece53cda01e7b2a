"""GPU tier (-m gpu): tf_unit_rows, tf_layernorm_rows and tf_layernorm_unit_rows (norm1 and the NN field's unit
rows) against `check_unit_rows` (bit for bit) and `check_layernorm_rows` (fp64, interval rule) of
oracle/kernel_checks.py.

* Every width: each multiple of 8 up to 1280 (the LayerNorm kernel holds a row in 5 register slots of 256 channels,
  so slots 3 and 4 and every partly filled slot run), and past 1280, where tf_unit_rows has no limit and the LayerNorm
  route falls back to `norm(x)` + unit rows.
* Rows: 1, 7, 8 and 64 * SMs +- 1 (one row per warp of the capped grid, then the row loop), the C2 frame pass and
  the C5s4 pivotal pass.
* Statistics probes (variance near eps, large offsets, constant rows, outliers, values near ±60000, γ with zeros and
  negative entries) and exact unit-row probes (scale invariance, one-hot, equal elements, subnormal norms, zero rows).
* Layouts: strided and misaligned inputs, packed outputs, and NaN-filled outputs with guard bands through the C ABI.
* Real sites: the hidden_states of all 16 transformer blocks of SD1.5 and SD2.1.
"""
import pytest
import torch

from oracle.kernel_checks import (LN_MAX_DIM, LN_SLOT_CHANNELS, NORM1_PROBES, check_layernorm_rows, check_unit_rows,
                                  guarded_layernorm_rows, guarded_unit_rows, norm1_module, norm1_probe)
from tokenflow_b200 import ops as tf_ops
from tokenflow_b200 import sd_unet

pytestmark = pytest.mark.gpu

SLOT_EDGE_DIMS = [8, 248, 256, 264, 512, 520, 768, 776, 1016, 1024, 1032, 1272, 1280]


@pytest.fixture(scope="module")
def ops():
    return tf_ops.CudaOps()


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _case(rows, dim, kind="randn", gamma="positive", seed=0):
    g = _gen(seed * 7919 + dim)
    x = norm1_probe(kind, rows, dim, generator=g).cuda()
    return x, norm1_module(dim, gamma, generator=g).cuda()


def _grid_rows():
    return 64 * torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------
# every width
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", range(8, LN_MAX_DIM + 1, 8))
def test_every_width(ops, dim):
    x, norm = _case(24, dim, gamma="signed" if dim % 16 else "positive", seed=1)
    y, unit = ops.layernorm_rows(x.view(3, 8, dim), norm, 1)
    check_layernorm_rows(y, unit, x.view(3, 8, dim), norm, 1, tag=f"layernorm_rows dim {dim}")
    u2 = ops.layernorm_unit_rows(x, norm)
    check_layernorm_rows(None, u2, x, norm, 24, tag=f"layernorm_unit_rows dim {dim}")
    assert torch.equal(u2[:8], unit.view(8, dim))                 # one kernel, one arithmetic
    x32 = (torch.randn(24, dim, generator=_gen(dim)) * 3 + 0.5).cuda()
    check_unit_rows(ops.unit_rows(x32), x32, tag=f"unit_rows fp32 dim {dim}")
    check_unit_rows(ops.unit_rows(x), x, tag=f"unit_rows fp16 dim {dim}")


@pytest.mark.parametrize("dim", [1288, 1536, 2048])
def test_widths_past_the_layernorm_kernel(ops, dim):
    x, norm = _case(24, dim, seed=2)
    x32 = (torch.randn(40, dim, generator=_gen(dim)) * 3 + 0.5).cuda()
    check_unit_rows(ops.unit_rows(x32), x32, tag=f"unit_rows fp32 dim {dim}")
    check_unit_rows(guarded_unit_rows(ops.lib, x), x, tag=f"unit_rows fp16 dim {dim}")
    # the op falls back to norm(x) (ATen, fp16 out) + unit rows of that
    y, unit = ops.layernorm_rows(x.view(3, 8, dim), norm, 1)
    want_y = norm(x.view(3, 8, dim))
    assert torch.equal(y, want_y)
    check_unit_rows(unit, want_y[:1], tag=f"fallback unit rows dim {dim}")
    check_unit_rows(ops.layernorm_unit_rows(x, norm), norm(x), tag=f"fallback layernorm_unit_rows dim {dim}")
    # the kernel itself refuses, without launching
    g32, b32 = norm.weight.float(), norm.bias.float()
    out = torch.empty_like(x)
    n0 = ops.launch_count()
    st = ops.lib.tf_layernorm_rows(x.data_ptr(), 24, dim, dim, g32.data_ptr(), b32.data_ptr(), 1e-5, out.data_ptr(),
                                   dim, out.data_ptr(), dim, 8, torch.cuda.current_stream().cuda_stream)
    assert st == 3 and b"not supported" in ops.lib.tf_last_error()             # TF_ERR_UNSUPPORTED
    st = ops.lib.tf_layernorm_unit_rows(x.data_ptr(), 24, dim, dim, g32.data_ptr(), b32.data_ptr(), 1e-5,
                                        out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert st == 3
    assert ops.launch_count() == n0


# ------------------------------------------------------------------------------------------------
# rows: the capped grid and its row loop; the C2 frame pass and the C5s4 pivotal pass
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [320, 1032])
@pytest.mark.parametrize("which", ["few", "grid"])
def test_row_counts(ops, dim, which):
    G = _grid_rows()
    for rows in ([1, 7, 8] if which == "few" else [G - 1, G, G + 1]):
        x, norm = _case(rows, dim, gamma="signed", seed=rows)
        tag = f"rows {rows} dim {dim}"
        y, unit = guarded_layernorm_rows(ops.lib, x, norm, rows)
        check_layernorm_rows(y, unit, x, norm, rows, tag=tag)
        _, u2 = guarded_layernorm_rows(ops.lib, x, norm, rows, with_y=False)
        assert torch.equal(u2, unit), tag
        y3, _ = guarded_layernorm_rows(ops.lib, x, norm, 0)
        assert torch.equal(y3, y), tag
        check_unit_rows(guarded_unit_rows(ops.lib, x), x, tag=tag)
        x32 = y.float() * 3 + 0.25
        check_unit_rows(guarded_unit_rows(ops.lib, x32), x32, tag=tag + " fp32")


def _check_chunked(y, unit, x, norm, n_unit, chunk, tag):
    use = {"y_use": 0.0, "u_use": 0.0}
    for a in range(0, x.shape[0], chunk):
        b = min(x.shape[0], a + chunk)
        nu = max(0, min(n_unit, b) - a)
        st = check_layernorm_rows(None if y is None else y[a:b], unit[a:a + nu] if nu else None, x[a:b], norm, nu,
                                  tag=f"{tag} samples {a}:{b}")
        for k in use:
            use[k] = max(use[k], st.get(k, 0.0))
    print(f"{tag}: largest use of δ: y {use['y_use']:.3f}, unit rows {use['u_use']:.3f}")
    return use


def test_c2_frame_pass(ops):
    """norm1 + unit rows of the source stream at C2's largest level: 8 frames x 4096 tokens x 320, taken from the
    first third of a [3F, S, dim] hidden_states."""
    hs, norm = _case(3 * 8 * 4096, 320, seed=3)
    hs = hs.view(24, 4096, 320)
    unit = ops.layernorm_unit_rows(hs[:8], norm)
    _check_chunked(None, unit, hs[:8], norm, 8, 4, "C2 frame pass")
    assert torch.equal(ops.layernorm_unit_rows(hs[:8].contiguous(), norm), unit)


def test_c5s4_pivotal_pass(ops):
    """norm1 of the C5s4 pivotal pass: 150 samples x 4096 tokens x 320, unit rows of the 50 source samples."""
    g = torch.Generator(device="cuda").manual_seed(4)
    hs = (torch.randn(150, 4096, 320, device="cuda", generator=g) * 2 + 0.3).half()
    norm = norm1_module(320, "signed", generator=_gen(4)).cuda()
    y, unit = ops.layernorm_rows(hs, norm, 50)
    _check_chunked(y, unit, hs, norm, 50, 10, "C5s4 pivotal pass")


# ------------------------------------------------------------------------------------------------
# statistics probes
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", NORM1_PROBES)
@pytest.mark.parametrize("dim,gamma", [(40, "signed"), (320, "positive"), (776, "signed"), (1032, "positive"),
                                       (1280, "signed")])
def test_statistics_probes(ops, kind, dim, gamma):
    x, norm = _case(32, dim, kind, gamma, seed=5)
    tag = f"{kind} dim {dim} γ {gamma}"
    y, unit = ops.layernorm_rows(x.view(4, 8, dim), norm, 2)
    st = check_layernorm_rows(y, unit, x.view(4, 8, dim), norm, 2, tag=tag)
    u2 = ops.layernorm_unit_rows(x, norm)
    st2 = check_layernorm_rows(None, u2, x, norm, 32, tag=tag)
    if kind == "constant":                  # the fp64 values are β and β / ||β||: y is fp16(β) up to δ
        assert torch.allclose(y.float(), norm.bias.float().expand_as(y), rtol=0, atol=2.0 ** -9), tag
    print(f"{tag}: δ use y {st['y_use']:.3f} unit {max(st['u_use'], st2['u_use']):.3f}, not correctly rounded "
          f"y {st['y_not_rn']:.4f} unit {st2['u_not_rn']:.4f}")


# ------------------------------------------------------------------------------------------------
# exact unit-row probes
# ------------------------------------------------------------------------------------------------
def _fp32_scale_sweep(x):
    import math
    lo = max(math.ceil(-126 - math.log2(x.abs().min().item())),
             math.ceil(-126 - math.log2(x.double().norm(dim=-1).min().item())))
    hi = math.floor(127 - math.log2(x.double().norm(dim=-1).max().item()))
    return sorted(set(range(-100, 101, 10)) | {lo, hi})


@pytest.mark.parametrize("dim", [40, 320, 1280])
def test_unit_rows_scale_invariance_fp32(ops, dim):
    g = _gen(dim)
    x = (torch.sign(torch.randn(64, dim, generator=g)) * (0.5 + 1.5 * torch.rand(64, dim, generator=g))).cuda()
    base = ops.unit_rows(x)
    check_unit_rows(base, x, tag=f"dim {dim}")
    for k in _fp32_scale_sweep(x):
        xs = x * 2.0 ** k
        assert torch.equal(xs * 2.0 ** -k, x)
        got = ops.unit_rows(xs)
        check_unit_rows(got, xs, tag=f"dim {dim} x 2^{k}")
        assert torch.equal(got, base), f"dim {dim}: unit_rows(x * 2^{k}) != unit_rows(x)"


@pytest.mark.parametrize("dim", [40, 320, 1280])
def test_unit_rows_scale_invariance_fp16(ops, dim):
    g = _gen(dim)
    x = (torch.sign(torch.randn(64, dim, generator=g)) * (0.5 + 1.5 * torch.rand(64, dim, generator=g))).half().cuda()
    base = ops.unit_rows(x)
    check_unit_rows(base, x, tag=f"fp16 dim {dim}")
    ks = []
    for k in range(-40, 41):
        xs = (x.float() * 2.0 ** k).half()
        if torch.isfinite(xs).all() and torch.equal(xs.float() * 2.0 ** -k, x.float()):
            ks.append(k)
            got = ops.unit_rows(xs)
            check_unit_rows(got, xs, tag=f"fp16 dim {dim} x 2^{k}")
            assert torch.equal(got, base), f"fp16 dim {dim}: unit_rows(x * 2^{k}) != unit_rows(x)"
    assert min(ks) <= -13 and max(ks) >= 14, ks           # |x| in [0.5, 2]: exact from 2^-13 up, finite to 2^14


def test_unit_rows_subnormal_norm_rows(ops):
    """Rows whose fp32 norm is subnormal (below 2^-126): 1 / norm overflows, x / fp32(norm) does not."""
    x = (torch.randn(48, 320, generator=_gen(9)) * 2.0 ** -136).cuda()
    n = x.double().norm(dim=-1)
    assert (n < 2.0 ** -126).all() and (n > 2.0 ** -149).all()
    check_unit_rows(ops.unit_rows(x), x, tag="subnormal norms")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("dim", [8, 320, 1032, 1280, 2048])
def test_unit_rows_special_rows(ops, dtype, dim):
    rows = 3 * 8
    x = torch.zeros(rows, dim, dtype=dtype, device="cuda")
    cols = torch.randint(0, dim, (8,), generator=_gen(dim)).cuda()
    x[torch.arange(8, device="cuda"), cols] = torch.tensor([1, -1, 3, -0.5, 1000, -2.0 ** -10, 7, -60000],
                                                           dtype=dtype, device="cuda")
    x[8:16] = torch.tensor([1, -1, 0.5, 4, -8, 2.0 ** -10, 2.0 ** -14, 256], dtype=dtype, device="cuda")[:, None]
    got = ops.unit_rows(x)
    check_unit_rows(got, x, tag=f"special rows {dtype} dim {dim}")
    onehot = torch.zeros(8, dim, dtype=torch.float16, device="cuda")
    onehot[torch.arange(8, device="cuda"), cols] = torch.tensor([1, -1, 1, -1, 1, -1, 1, -1], dtype=torch.float16,
                                                                device="cuda")
    assert torch.equal(got[:8], onehot)                               # exactly ±1 and 0
    want = torch.tensor(dim ** -0.5, dtype=torch.float64).half().item()
    sign = torch.sign(x[8:16, :1].float()).half()
    assert torch.equal(got[8:16], (sign * want).expand(8, dim))        # RN16(±1/sqrt(dim))
    assert torch.isnan(got[16:]).all()                                # 0 / 0, like x / x.norm()


# ------------------------------------------------------------------------------------------------
# layouts
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [40, 320, 1032, 1280])
def test_strided_and_misaligned_inputs(ops, dim):
    rows = 40
    g = _gen(dim)
    # fp32 rows with pitch dim + 4 are read in place
    buf = (torch.randn(rows, dim + 4, generator=g) * 2).cuda()
    x = buf[:, :dim]
    got = ops.unit_rows(x)
    check_unit_rows(got, x, tag="pitch dim + 4")
    assert torch.equal(got, ops.unit_rows(x.contiguous()))
    # a pitch the kernel cannot take (dim + 2 fp32), and a data_ptr 4 / 2 bytes off 16: copied first, same bits
    buf2 = (torch.randn(rows, dim + 2, generator=g) * 2).cuda()
    for v in (buf2[:, :dim], buf2.view(-1)[1:1 + rows * dim].view(rows, dim)):
        assert torch.equal(ops.unit_rows(v), ops.unit_rows(v.contiguous()))
    h = (torch.randn(rows * dim + 8, generator=g) * 2).half().cuda()
    mis = h[1:1 + rows * dim].view(rows, dim)
    assert mis.data_ptr() % 16
    assert torch.equal(ops.unit_rows(mis), ops.unit_rows(mis.contiguous()))
    norm = norm1_module(dim, "signed", generator=g).cuda()
    assert torch.equal(ops.layernorm_unit_rows(mis, norm), ops.layernorm_unit_rows(mis.contiguous(), norm))
    y1, u1 = ops.layernorm_rows(mis.view(5, 8, dim), norm, 2)
    y2, u2 = ops.layernorm_rows(mis.contiguous().view(5, 8, dim), norm, 2)
    assert torch.equal(y1, y2) and torch.equal(u1, u2)
    # column slices of a packed [b, S, 3 dim] buffer, read in place
    pack = (torch.randn(5, 8, 3 * dim, generator=g) * 2 + 0.3).half().cuda()
    xs = pack[..., dim:2 * dim]
    y, unit = ops.layernorm_rows(xs, norm, 2)
    check_layernorm_rows(y, unit, xs, norm, 2, tag=f"packed input dim {dim}")
    assert torch.equal(ops.layernorm_unit_rows(xs, norm), ops.layernorm_unit_rows(xs.contiguous(), norm))
    assert torch.equal(ops.unit_rows(xs), ops.unit_rows(xs.contiguous()))


@pytest.mark.parametrize("dim", SLOT_EDGE_DIMS)
@pytest.mark.parametrize("n_unit", [0, 1, 6])
def test_layernorm_rows_into_packed_outputs(ops, dim, n_unit):
    b, S = 6, 16
    x, norm = _case(b * S, dim, gamma="signed", seed=n_unit)
    x = x.view(b, S, dim)
    pack = torch.full((b, S, 3 * dim), float("nan"), dtype=torch.float16, device="cuda")
    y, unit = ops.layernorm_rows(x, norm, n_unit, y_out=pack[..., :dim], unit_out=pack[:n_unit, :, 2 * dim:])
    torch.cuda.synchronize()
    assert torch.isnan(pack[..., dim:2 * dim]).all(), "write into the gap columns"
    assert torch.isnan(pack[n_unit:, :, 2 * dim:]).all(), "unit rows past n_unit written"
    check_layernorm_rows(pack[..., :dim], pack[:n_unit, :, 2 * dim:] if n_unit else None, x, norm, n_unit,
                         tag=f"packed outputs dim {dim} n_unit {n_unit}")
    y0, u0 = ops.layernorm_rows(x, norm, n_unit)
    assert torch.equal(y0, pack[..., :dim]) and (n_unit == 0 or torch.equal(u0, pack[:n_unit, :, 2 * dim:]))


@pytest.mark.parametrize("dim", SLOT_EDGE_DIMS)
def test_sentinel_outputs_with_pitch(ops, dim):
    """NaN-filled outputs with guard bands and a row pitch of dim + 16 (gap columns)."""
    x, norm = _case(40, dim, seed=6)
    y, unit = guarded_layernorm_rows(ops.lib, x, norm, 13, y_pitch=dim + 16, unit_pitch=dim + 16)
    check_layernorm_rows(y, unit, x, norm, 13, tag=f"sentinel dim {dim}")
    _, u2 = guarded_layernorm_rows(ops.lib, x, norm, 40, with_y=False)
    assert torch.equal(u2[:13], unit)
    check_unit_rows(guarded_unit_rows(ops.lib, x), x, tag=f"sentinel unit rows dim {dim}")


# ------------------------------------------------------------------------------------------------
# real sites: norm1 of every transformer block of SD1.5 and SD2.1
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["sd15", "sd21"])
def test_real_norm1_sites(ops, kind):
    unet = sd_unet.build_unet(kind, seed=1, device="cuda", dtype=torch.float16, init_on_device=True)
    unet = unet.to(memory_format=torch.channels_last)
    g = torch.Generator(device="cuda").manual_seed(0)
    sample = torch.randn(3, 4, 64, 64, device="cuda", generator=g).half().contiguous(memory_format=torch.channels_last)
    ctx = torch.randn(3, 77, unet.config.cross_attention_dim, device="cuda", generator=g).half()
    captured = []
    blocks = [m for m in unet.modules() if isinstance(m, sd_unet.BasicTransformerBlock)]
    hooks = [blk.register_forward_pre_hook(lambda m, args, kw=None, i=i: captured.append((i, m.norm1, args[0].clone())))
             for i, blk in enumerate(blocks)]
    try:
        with torch.no_grad():
            unet(sample, torch.tensor([501], device="cuda"), encoder_hidden_states=ctx)
    finally:
        for h in hooks:
            h.remove()
    torch.cuda.synchronize()
    assert len(blocks) == 16 and len(captured) == 16
    worst = {"y_use": 0.0, "u_use": 0.0}
    for i, norm, hs in captured:
        b, S, dim = hs.shape
        tag = f"{kind} block {i}: {b}x{S}x{dim}"
        y, unit = ops.layernorm_rows(hs, norm, b // 3)
        st = check_layernorm_rows(y, unit, hs, norm, b // 3, tag=tag)
        st2 = check_layernorm_rows(None, ops.layernorm_unit_rows(hs, norm), hs, norm, b, tag=tag)
        print(f"{tag}: largest use of δ: y {st['y_use']:.3f}, unit rows {max(st['u_use'], st2['u_use']):.3f}")
        worst = {"y_use": max(worst["y_use"], st["y_use"]), "u_use": max(worst["u_use"], st["u_use"], st2["u_use"])}
    print(f"{kind}: largest use of δ over the 16 sites: y {worst['y_use']:.3f}, unit rows {worst['u_use']:.3f}")
    del unet
    torch.cuda.empty_cache()
