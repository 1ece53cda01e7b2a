"""GPU tier (-m gpu): the two kernels that write every latent of every step, and operands at any element offset.

* Every fp16 input.  tf_cfg_ddim with u over all 65 536 fp16 bit patterns against a structured set of c and x (signed
  zeros, subnormals, the smallest normal, +-1, +-65504, +-inf, NaN, magnitudes where g (c - u) overflows, N(0, 1)
  values), and again with the roles of u and c swapped, at every step of a 50-step schedule and five guidances; tf_ddim
  with eps over all patterns against structured x and the other way round, at every step of both 500-step inversion
  tables, out of place and in place.  References: the scheduler's eager fp16 step on the same GPU (bit for bit, NaN
  equal to NaN) and oracle/latent_step.py's numpy restatement on a sample of every sweep.
* Lengths 1 ... 40 and 8k + r for every residue r over several blocks, with the outputs between guard bands.
* Offsets.  Every operand of the step ops 0 ... 7 elements into a larger buffer, independently; every tensor operand of
  every other op 1 ... 7 fp16 (1 ... 3 fp32 / int32, 1 ... 15 uint8) elements in: the same bytes as the aligned call.
* Odd latent sizes end to end: 13 x 21 latents (an odd h * w, so a slice of an odd number of frames starts 8 bytes
  off) through the tiny UNet on one rank and on two rank threads, and 45 x 75 through SD1.5 channels_last.
"""
import importlib.util
import os
import threading
import types

import numpy as np
import pytest
import torch

from oracle import inversion as OI
from oracle import latent_step as LS
from oracle.kernel_checks import ext_attn_samples
from oracle.oracle_ops import OracleOps
from tokenflow_b200 import ops as tf_ops
from tokenflow_b200 import sd_unet
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.editor import TokenFlowEditor, synthetic_inputs
from tokenflow_b200.ops import blend_weights
from tokenflow_b200.preprocess import LatentInverter, inversion_coef_tables
from tokenflow_b200.scheduler import DDIMScheduler

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ops():
    tfu._install_ops_for_testing(None)
    return tf_ops.CudaOps()


def _schedule(steps):
    sch = DDIMScheduler()
    sch.set_timesteps(steps)
    return sch


def _edit_coefs(sch):
    """The editor's device coefficient table for the schedule, built by the editor's own method."""
    stub = types.SimpleNamespace(scheduler=sch, _t_host=[int(t) for t in sch.timesteps], device=torch.device("cuda"))
    return TokenFlowEditor._make_coef_table(stub)


def _int_view(t):
    return t.view({2: torch.int16, 4: torch.int32}[t.element_size()]) if t.is_floating_point() else t


def _mismatches(got, want):
    """Device count of elements whose bits differ, NaN counting as equal to NaN."""
    bad = _int_view(got) != _int_view(want)
    if got.is_floating_point():
        bad &= ~(torch.isnan(got) & torch.isnan(want))
    return bad.sum()


def _edges(tag, out):
    a = out.float().abs()
    sub = ((a > 0) & (a < 2.0 ** -14)).sum().item()
    print(f"{tag}: {out.numel()} outputs, {torch.isinf(out).sum().item()} inf, {torch.isnan(out).sum().item()} NaN, "
          f"{sub} subnormal, {(out == 0).sum().item()} zero")
    return sub


def _numpy_agrees(fn, operands, got, coef, *extra, n=1 << 20, seed=0):
    """The numpy restatement on `n` elements drawn from the whole sweep."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    idx = torch.randint(0, got.numel(), (n,), device="cuda", generator=g)
    host = [t.reshape(-1)[idx].cpu().numpy() for t in operands]
    want = fn(*host, coef.cpu().numpy(), *extra)
    ok = LS.same_bits(got.reshape(-1)[idx].cpu().numpy(), want)
    assert ok.all(), f"{int((~ok).sum())} of {n} sampled outputs differ from the numpy restatement"


# ------------------------------------------------------------------------------------------------
# a. tf_cfg_ddim over every fp16 input
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cfg_sweep():
    """(all, structured, x): element (ix * m + ic) * 65536 + bits pairs fp16 pattern `bits` with structured value ic
    and latent ix — 57 * 57 * 65536 = 213 M elements."""
    s = torch.from_numpy(LS.structured_fp16()).cuda()
    m = len(s)
    allv = torch.from_numpy(LS.ALL_FP16.view(np.int16).copy()).cuda().view(torch.float16)
    return allv.repeat(m * m), s.repeat_interleave(1 << 16).repeat(m), s.repeat_interleave(m << 16)


NUMPY_ROWS = (0, 7, 14, 21, 28, 35, 42, 49)


@pytest.mark.parametrize("g", [7.5, 1.0, 0.0, 30.0, 3.3])
@pytest.mark.parametrize("roles", ["u_all", "c_all"])
def test_cfg_ddim_every_fp16_input(ops, cfg_sweep, g, roles):
    allv, struct, x = cfg_sweep
    u, c = (allv, struct) if roles == "u_all" else (struct, allv)
    sch = _schedule(50)
    coef = _edit_coefs(sch)
    out = torch.empty_like(x)
    bad = torch.zeros(50, dtype=torch.int64, device="cuda")
    for row, t in enumerate(int(t) for t in sch.timesteps):
        ops.cfg_ddim(u, c, x, coef[row], g, out=out)
        want = sch.step(u + g * (c - u), t, x)["prev_sample"]
        bad[row] = _mismatches(out, want)
        del want
        if row in NUMPY_ROWS:
            _numpy_agrees(LS.cfg_ddim, (u, c, x), out, coef[row], g, seed=row)
        if row == 49:
            _edges(f"cfg_ddim g={g} {roles} step {row}", out)
    assert bad.sum().item() == 0, {r: v for r, v in enumerate(bad.tolist()) if v}


# ------------------------------------------------------------------------------------------------
# b. tf_ddim over every fp16 input, both 500-step tables, out of place and in place
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ddim_sweep():
    s = torch.from_numpy(LS.structured_fp16()).cuda()
    m = len(s)
    allv = torch.from_numpy(LS.ALL_FP16.view(np.int16).copy()).cuda().view(torch.float16)
    eps = torch.cat([allv.repeat(m), s.repeat_interleave(1 << 16)])
    x = torch.cat([s.repeat_interleave(1 << 16), allv.repeat(m)])
    return eps, x


@pytest.mark.parametrize("direction", ["inversion", "reconstruction"])
def test_ddim_every_fp16_input(ops, ddim_sweep, direction):
    eps, x = ddim_sweep
    sch = _schedule(500)
    inv, rec = inversion_coef_tables(sch)
    table = (inv if direction == "inversion" else rec).cuda()
    out, xi = torch.empty_like(x), torch.empty_like(x)
    bad = torch.zeros(500, 2, dtype=torch.int64, device="cuda")
    subnormal = 0
    for i in range(500):
        want = OI.ddim_expression(x, eps, direction, OI.step_alphas(sch, direction, i))
        ops.ddim(eps, x, table[i], out=out)
        bad[i, 0] = _mismatches(out, want)
        xi.copy_(x)
        assert ops.ddim(eps, xi, table[i], out=xi).data_ptr() == xi.data_ptr()
        bad[i, 1] = _mismatches(xi, want)
        if i in (0, 1, 97, 250, 498, 499):
            _numpy_agrees(LS.ddim, (eps, x), out, table[i], seed=i)
            subnormal += _edges(f"ddim {direction} step {i}", out)
    assert bad.sum().item() == 0, {i: v for i, v in enumerate(bad.tolist()) if any(v)}
    assert subnormal > 0


# ------------------------------------------------------------------------------------------------
# c. every length, outputs between guard bands
# ------------------------------------------------------------------------------------------------
GUARD = 64                                  # elements: keeps the output 16-byte aligned
SENTINEL = 0x7E5A                           # an fp16 NaN payload the kernels never produce
LENGTHS = list(range(1, 41)) + [8 * k + r for k in (255, 256, 257, 1023, 2049) for r in range(8)]


def _guarded(n):
    buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.int16, device="cuda")
    return buf, buf[GUARD:GUARD + n].view(torch.float16)


def _guards_intact(buf):
    return bool((buf[:GUARD] == SENTINEL).all()) and bool((buf[-GUARD:] == SENTINEL).all())


def test_step_ops_write_exactly_n_outputs(ops):
    sch = _schedule(50)
    coef = _edit_coefs(sch)
    inv, _ = inversion_coef_tables(_schedule(500))
    inv = inv.cuda()
    alphas = OI.step_alphas(_schedule(500), "inversion", 300)
    g = torch.Generator(device="cuda").manual_seed(4)
    for n in LENGTHS:
        u, c, x, e = (torch.randn(n, device="cuda", generator=g).half() for _ in range(4))
        buf, out = _guarded(n)
        assert ops.cfg_ddim(u, c, x, coef[17], 7.5, out=out).data_ptr() == out.data_ptr()
        want = sch.step(u + 7.5 * (c - u), int(sch.timesteps[17]), x)["prev_sample"]
        assert _mismatches(out, want).item() == 0 and _guards_intact(buf), n
        want = OI.ddim_expression(x, e, "inversion", alphas)
        buf, out = _guarded(n)
        ops.ddim(e, x, inv[300], out=out)
        assert _mismatches(out, want).item() == 0 and _guards_intact(buf), n
        buf, xi = _guarded(n)
        xi.copy_(x)
        ops.ddim(e, xi, inv[300], out=xi)
        assert _mismatches(xi, want).item() == 0 and _guards_intact(buf), n


# ------------------------------------------------------------------------------------------------
# d. the step ops with every operand 0 ... 7 elements into a larger buffer
# ------------------------------------------------------------------------------------------------
def _at(t, off, channels_last=False):
    """A copy of `t` starting `off` elements into a fresh buffer (whose start is 16-byte aligned)."""
    buf = torch.empty(t.numel() + 16, dtype=t.dtype, device=t.device)
    flat = buf[off:off + t.numel()]
    if channels_last:
        n, c, h, w = t.shape
        view = flat.view(n, h, w, c).permute(0, 3, 1, 2)
    else:
        view = flat.view(t.shape)
    view.copy_(t)
    return view


def test_cfg_ddim_at_every_operand_offset(ops):
    torch.manual_seed(8)
    shape = (3, 4, 13, 21)
    u, c, x = (torch.randn(shape, device="cuda").half() for _ in range(3))
    coef = _edit_coefs(_schedule(50))[23]
    want = ops.cfg_ddim(u, c, x, coef, 7.5)
    us, cs, xs, outs = ([_at(t, o) for o in range(8)] for t in (u, c, x, torch.zeros_like(u)))
    bad = torch.zeros((), dtype=torch.int64, device="cuda")
    for iu in range(8):
        for ic in range(8):
            for ix in range(8):
                for io in range(8):
                    got = ops.cfg_ddim(us[iu], cs[ic], xs[ix], coef, 7.5, out=outs[io])
                    assert got.data_ptr() == outs[io].data_ptr()
                    bad += _mismatches(got, want)
    assert bad.item() == 0


@pytest.mark.parametrize("eps_layout", ["contiguous", "channels_last"])
def test_ddim_at_every_operand_offset(ops, eps_layout):
    torch.manual_seed(9)
    shape = (3, 4, 13, 21)
    eps, x = torch.randn(shape, device="cuda").half(), (2 * torch.randn(shape, device="cuda")).half()
    coef = inversion_coef_tables(_schedule(500))[1][200].cuda()
    want = ops.ddim(eps, x, coef)
    es = [_at(eps, o, channels_last=eps_layout == "channels_last") for o in range(8)]
    xs, outs = [_at(x, o) for o in range(8)], [_at(torch.zeros_like(x), o) for o in range(8)]
    bad = torch.zeros((), dtype=torch.int64, device="cuda")
    for ie in range(8):
        for ix in range(8):
            for io in range(8):
                got = ops.ddim(es[ie], xs[ix], coef, out=outs[io])
                assert got.data_ptr() == outs[io].data_ptr()
                bad += _mismatches(got, want)
            assert torch.equal(xs[ix], x)                                  # out of place: x is only read
            xi = _at(x, ix)
            got = ops.ddim(es[ie], xi, coef, out=xi)
            assert got.data_ptr() == xi.data_ptr()                         # in place stays in place
            bad += _mismatches(xi, want)
    assert bad.item() == 0


# ------------------------------------------------------------------------------------------------
# e. every other op with each tensor operand 1 ... 7 fp16 elements in
# ------------------------------------------------------------------------------------------------
def _norm_ln(dim):
    norm = torch.nn.LayerNorm(dim).cuda().half()
    with torch.no_grad():
        norm.weight.uniform_(0.5, 1.5)
        norm.bias.uniform_(-0.3, 0.3)
    return norm


def _cases():
    """name -> (operands, call(ops, **operands) -> tensor or tuple, channels_last operand names)."""
    torch.manual_seed(12)
    r = lambda *s: torch.randn(*s, device="cuda")
    u8 = lambda *s: torch.randint(0, 256, s, dtype=torch.uint8, device="cuda")
    ln = _norm_ln(64)
    gn = torch.nn.GroupNorm(8, 64).cuda().half()
    with torch.no_grad():
        gn.weight.uniform_(0.5, 1.5)
        gn.bias.uniform_(-0.3, 0.3)
    piv = torch.nn.functional.normalize(r(2, 64, 64), dim=-1)
    xu = torch.nn.functional.normalize(piv[1][torch.randperm(64, device="cuda")] + 0.3 * r(4, 64, 64), dim=-1)
    kf_a, kf_b, w = [1] * 4, [0] * 4, blend_weights(4)
    idx_a = torch.randint(0, 64, (4, 64), dtype=torch.int32, device="cuda")
    idx_b = torch.randint(0, 64, (4, 64), dtype=torch.int32, device="cuda")
    q, k, v = (r(6, 64, 80).half() for _ in range(3))
    cl = lambda t: t.contiguous(memory_format=torch.channels_last)
    return {
        "unit_rows_f16": (dict(x=r(6, 40, 64).half()), lambda o, x: o.unit_rows(x), ()),
        "unit_rows_f32": (dict(x=r(6, 40, 64)), lambda o, x: o.unit_rows(x), ()),
        "layernorm_unit_rows": (dict(x=r(6, 40, 64).half()), lambda o, x: o.layernorm_unit_rows(x, ln), ()),
        "layernorm_rows": (dict(x=r(6, 40, 64).half(), y_out=torch.zeros(6, 40, 64, device="cuda").half(),
                                unit_out=torch.zeros(2, 40, 64, device="cuda").half()),
                           lambda o, x, y_out, unit_out: o.layernorm_rows(x, ln, 2, y_out=y_out, unit_out=unit_out), ()),
        "nn_field": (dict(x_unit=xu.half(), piv_unit=piv.half()),
                     lambda o, x_unit, piv_unit: o.nn_field(x_unit, piv_unit, kf_a, kf_b), ()),
        "propagate": (dict(A=r(3, 2, 64, 64).half(), idx_a=idx_a, idx_b=idx_b, residual=r(12, 64, 64).half()),
                      lambda o, A, idx_a, idx_b, residual: o.propagate(A, idx_a, idx_b, kf_a, kf_b, w, residual), ()),
        "ext_attn": (dict(q=q, k=k, v=v), lambda o, q, k, v: o.ext_attn(q, k, v, 2, 40 ** -0.5, True), ()),
        "ext_attn_table": (dict(q=q, k=k, v=v), lambda o, q, k, v: o.ext_attn_table(
            q, k, v, ext_attn_samples(2, False), 2, 40 ** -0.5), ()),
        "group_norm_nhwc": (dict(x=cl(r(2, 64, 8, 12).half()), bias=r(2, 64).half()),
                            lambda o, x, bias: o.group_norm_nhwc(x, gn, bias, True), ("x",)),
        "geglu": (dict(xh=r(5, 77, 40).half(), gate=r(5, 77, 40).half()), lambda o, xh, gate: o.geglu(xh, gate), ()),
        "frames_to_nhwc": (dict(frames=u8(2, 9, 13, 3)), lambda o, frames: o.frames_to_nhwc(frames), ()),
        "nhwc_to_frames": (dict(x=cl((1.2 * r(2, 3, 9, 13)).half())), lambda o, x: o.nhwc_to_frames(x), ("x",)),
        "resize_frames": (dict(frames=u8(2, 9, 13, 3), tmp=torch.zeros(2, 9, 10, 3, dtype=torch.uint8, device="cuda"),
                               out=torch.zeros(2, 7, 10, 3, dtype=torch.uint8, device="cuda")),
                          lambda o, frames, tmp, out: o.resize_frames(frames, (7, 10), tmp=tmp, out=out), ()),
        "canny": (dict(frames=u8(2, 16, 20, 3), out_edges=torch.zeros(2, 16, 20, dtype=torch.uint8, device="cuda"),
                       out_cond=cl(torch.zeros(2, 3, 16, 20, device="cuda").half())),
                  lambda o, frames, out_edges, out_cond: o.canny(frames, out_edges=out_edges, out_cond=out_cond),
                  ("out_cond",)),
    }


def _outputs(res):
    return [t for t in (res if isinstance(res, tuple) else (res,)) if t is not None]


OP_CASES = ["unit_rows_f16", "unit_rows_f32", "layernorm_unit_rows", "layernorm_rows", "nn_field", "propagate",
            "ext_attn", "ext_attn_table", "group_norm_nhwc", "geglu", "frames_to_nhwc", "nhwc_to_frames", "resize_frames",
            "canny"]


def _is_output(arg):
    return arg.endswith("out") or arg == "tmp"


@pytest.mark.parametrize("name", OP_CASES)
def test_every_op_at_every_operand_offset(ops, name):
    """Each operand alone moved 1 ... 7 fp16 (1 ... 3 fp32 / int32, 1 ... 15 uint8) elements off a 16-byte boundary:
    the outputs hold the aligned call's bytes, and an output given to the op is the one written."""
    operands, call, channels_last = _cases()[name]
    fresh = lambda d: {k: v.clone() if _is_output(k) else v for k, v in d.items()}
    want = [t.clone() for t in _outputs(call(ops, **fresh(operands)))]
    for arg, t in operands.items():
        for off in range(1, {1: 15, 2: 7, 4: 3}[t.element_size()] + 1):
            moved = fresh(operands)
            moved[arg] = _at(t, off, channels_last=arg in channels_last)
            got = _outputs(call(ops, **moved))
            assert len(got) == len(want)
            for gt, wt in zip(got, want):
                assert _mismatches(gt, wt).item() == 0, (name, arg, off)
            if _is_output(arg) and arg != "tmp":
                assert any(gt.data_ptr() == moved[arg].data_ptr() for gt in got), (name, arg, off)


# ------------------------------------------------------------------------------------------------
# f. odd latent sizes end to end
# ------------------------------------------------------------------------------------------------
ODD = (13, 21)


def _tiny_edit(mode, steps, fused=True, graph=False, world=1, rank=0, comm=None, unet=None):
    if unet is None:
        unet = sd_unet.build_unet("tiny", seed=1, device="cuda", dtype=torch.float16)
    cfg = {"n_frames": 6, "batch_size": 2, "n_timesteps": steps, "guidance_scale": 7.5, "mode": mode,
           "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "start": 0.9, "fused_pass": fused, "cuda_graph": graph, "keyframe_seed": 1}
    x, text, pnp, src = synthetic_inputs(6, ODD, unet.config.cross_attention_dim, steps, seed=1, device="cuda",
                                         dtype=torch.float16, ctx_len=7)
    ed = TokenFlowEditor(unet, DDIMScheduler(), tfu, cfg, text, pnp, source_latents=lambda t: src[t],
                         world_size=world, rank=rank)
    if comm is not None:
        ed.attach_communicator(comm)
    ed.init_method()
    return ed.sample_loop(x), ed.keyframe_log


@pytest.mark.parametrize("mode,steps", [("pnp", 5), ("sdedit", 10)])
def test_tiny_unet_edit_at_13x21(mode, steps):
    """6 frames, batch 2: the fused step's frame slice starts 9 + 6 samples into the UNet output."""
    tfu._install_ops_for_testing(None)
    eager, kf_e = _tiny_edit(mode, steps)
    graphed, kf_g = _tiny_edit(mode, steps, graph=True)
    assert kf_g == kf_e and torch.equal(graphed, eager)
    tfu._install_ops_for_testing(OracleOps())                 # the reference's arithmetic and schedule
    want, kf_w = _tiny_edit(mode, steps, fused=False)
    tfu._install_ops_for_testing(None)
    assert kf_w == kf_e and eager.shape == (6, 4) + ODD and torch.isfinite(eager).all()
    rel = (eager.float() - want.float()).norm() / want.float().norm()
    assert rel.item() < 2e-2, rel.item()


def _thread_world():
    spec = importlib.util.spec_from_file_location("_tf_gpu_round2", os.path.join(REPO, "tests", "test_gpu_round2.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod._ThreadWorld


def test_two_rank_threads_at_13x21():
    """Rank 1 denoises frames 3 ... 5: its latents start 3 * 4 * 273 elements (8 bytes past a 16-byte boundary)
    into x."""
    tfu._install_ops_for_testing(None)
    tfu._ops()
    unets = [sd_unet.build_unet("tiny", seed=1, device="cuda", dtype=torch.float16) for _ in range(3)]
    want, kf_want = _tiny_edit("pnp", 5, unet=unets[2])
    tw = _thread_world()(2)
    res = {}

    def run(r):
        try:
            res[r] = _tiny_edit("pnp", 5, world=2, rank=r, comm=tw.rank(r), unet=unets[r])
        except BaseException as ex:  # noqa: BLE001
            res[r] = ex
            tw.barrier.abort()

    threads = [threading.Thread(target=run, args=(r,)) for r in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=600)
    errors = [res.get(r) for r in range(2) if not isinstance(res.get(r), tuple)]
    errors.sort(key=lambda e: isinstance(e, threading.BrokenBarrierError))      # the cause first
    assert not errors, errors
    for r in range(2):
        got, kf = res[r]
        assert kf == kf_want and torch.isfinite(got).all()
        rel = (got.float() - want.float()).norm() / want.float().norm()
        assert rel.item() < 2e-2, (r, rel.item())
    assert torch.equal(res[0][0], res[1][0])


@pytest.fixture(scope="module")
def sd15():
    unet = sd_unet.build_unet("sd15", seed=1, device="cuda", dtype=torch.float16, init_on_device=True)
    return unet.to(memory_format=torch.channels_last)


def test_sd15_channels_last_edit_at_45x75():
    """360 x 600 frames: 45 x 75 latents, 3 PnP steps, graphed == eager."""
    outs = []
    tfu._install_ops_for_testing(None)
    for graph in (False, True):
        sd15 = sd_unet.build_unet("sd15", seed=1, device="cuda", dtype=torch.float16,
                                  init_on_device=True).to(memory_format=torch.channels_last)
        cfg = {"n_frames": 6, "batch_size": 2, "n_timesteps": 3, "guidance_scale": 7.5, "mode": "pnp",
               "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "fused_pass": True, "cuda_graph": graph, "keyframe_seed": 1}
        x, text, pnp, src = synthetic_inputs(6, (45, 75), sd15.config.cross_attention_dim, 3, seed=1, device="cuda",
                                             dtype=torch.float16, ctx_len=7)
        ed = TokenFlowEditor(sd15, DDIMScheduler(), tfu, cfg, text, pnp, source_latents=lambda t: src[t])
        ed.init_method()
        outs.append((ed.sample_loop(x), ed.keyframe_log))
        del ed, sd15
    assert outs[0][1] == outs[1][1]
    assert outs[0][0].shape == (6, 4, 45, 75) and torch.isfinite(outs[0][0]).all()
    assert torch.equal(outs[1][0], outs[0][0])


def test_sd15_channels_last_inversion_at_45x75(sd15):
    g = torch.Generator().manual_seed(3)
    x0 = torch.randn(3, 4, 45, 75, generator=g).half().cuda()
    cond = torch.randn(1, 77, sd15.config.cross_attention_dim, generator=g).half().cuda()
    res = {}
    for graphed in (True, False):
        inv = LatentInverter(sd15, DDIMScheduler(), 3)
        inv._use_graph = graphed
        xT = inv.ddim_inversion(cond, x0, None, batch_size=2)
        res[graphed] = (xT, inv.ddim_sample(xT, cond, batch_size=2), inv.scheduler)
    assert torch.equal(res[True][0], res[False][0]) and torch.equal(res[True][1], res[False][1])
    want_T, _ = OI.ddim_inversion(sd15, res[True][2], cond, x0.clone(), 2)
    want_rec = OI.ddim_sample(sd15, res[True][2], want_T.clone(), cond, 2)
    assert torch.isfinite(want_rec).all()
    assert torch.equal(res[True][0], want_T) and torch.equal(res[True][1], want_rec)
