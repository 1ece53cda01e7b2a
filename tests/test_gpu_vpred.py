"""GPU tier (-m gpu): the v-prediction latent updates and the stages that use them.

* Every fp16 input.  tf_cfg_ddim_v with u over all 65 536 fp16 bit patterns against the structured values of c and x
  (oracle/latent_step.py `structured_fp16`), then with the roles of u and c swapped, at every step of a 50-step
  schedule and five guidances; tf_ddim_v with v over all patterns against structured x and the other way round, at
  every step of both 500-step inversion tables, out of place and in place.  References: the v scheduler's eager fp16
  step (and oracle/inversion_v.py's v form of the reference's inversion expression) on the same GPU, bit for bit with
  NaN equal to NaN, and the numpy restatement (oracle/latent_step_v.py) on a sample of every sweep.
* Lengths 1 ... 40 and 8k + r between guard bands; every operand 0 ... 7 elements into a larger buffer.
* End to end with a v scheduler: the tiny UNet at 13 x 21 latents (PnP, SDEdit, PnP with a `from_unet` ControlNet:
  graphed edit == eager edit; two rank threads == one rank; graphed inversion == oracle/inversion_v.py's loop), and
  SD2.1 channels_last at C4's 96 x 96 latents (a graphed SDEdit step == eager, a short-grid inversion == the oracle).
"""
import importlib.util
import os
import threading
import types

import numpy as np
import pytest
import torch

from oracle import gen_canny_golden as gg
from oracle import inversion as OI
from oracle import inversion_v as OIV
from oracle import latent_step as LS
from oracle import latent_step_v as LSV
from tokenflow_b200 import ops as tf_ops
from tokenflow_b200 import preprocess, sd_unet
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.controlnet import ControlNetModel
from tokenflow_b200.editor import TokenFlowEditor, synthetic_inputs
from tokenflow_b200.preprocess import LatentInverter, inversion_coef_tables
from tokenflow_b200.scheduler import DDIMScheduler

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V = "v_prediction"


@pytest.fixture(scope="module")
def ops():
    tfu._install_ops_for_testing(None)
    return tf_ops.CudaOps()


def _schedule(steps):
    sch = DDIMScheduler(prediction_type=V)
    sch.set_timesteps(steps)
    return sch


def _edit_coefs(sch):
    stub = types.SimpleNamespace(scheduler=sch, _t_host=[int(t) for t in sch.timesteps], device=torch.device("cuda"))
    return TokenFlowEditor._make_coef_table(stub)


def _int_view(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t


def _mismatches(got, want):
    bad = _int_view(got) != _int_view(want)
    bad &= ~(torch.isnan(got) & torch.isnan(want))
    return bad.sum()


def _edges(tag, out):
    a = out.float().abs()
    sub = ((a > 0) & (a < 2.0 ** -14)).sum().item()
    print(f"{tag}: {out.numel()} outputs, {torch.isinf(out).sum().item()} inf, {torch.isnan(out).sum().item()} NaN, "
          f"{sub} subnormal, {(out == 0).sum().item()} zero")
    return sub


def _numpy_agrees(fn, operands, got, coef, *extra, n=1 << 20, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    idx = torch.randint(0, got.numel(), (n,), device="cuda", generator=g)
    host = [t.reshape(-1)[idx].cpu().numpy() for t in operands]
    want = fn(*host, coef.cpu().numpy(), *extra)
    ok = LS.same_bits(got.reshape(-1)[idx].cpu().numpy(), want)
    assert ok.all(), f"{int((~ok).sum())} of {n} sampled outputs differ from the numpy restatement"


# ------------------------------------------------------------------------------------------------
# a. tf_cfg_ddim_v over every fp16 input
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cfg_sweep():
    s = torch.from_numpy(LS.structured_fp16()).cuda()
    m = len(s)
    allv = torch.from_numpy(LS.ALL_FP16.view(np.int16).copy()).cuda().view(torch.float16)
    return allv.repeat(m * m), s.repeat_interleave(1 << 16).repeat(m), s.repeat_interleave(m << 16)


NUMPY_ROWS = (0, 7, 14, 20, 21, 35, 42, 49)


@pytest.mark.parametrize("g", [7.5, 1.0, 0.0, 30.0, 3.3])
@pytest.mark.parametrize("roles", ["u_all", "c_all"])
def test_cfg_ddim_v_every_fp16_input(ops, cfg_sweep, g, roles):
    allv, struct, x = cfg_sweep
    u, c = (allv, struct) if roles == "u_all" else (struct, allv)
    sch = _schedule(50)
    coef = _edit_coefs(sch)
    out = torch.empty_like(x)
    bad = torch.zeros(50, dtype=torch.int64, device="cuda")
    for row, t in enumerate(int(t) for t in sch.timesteps):
        ops.cfg_ddim_v(u, c, x, coef[row], g, out=out)
        want = sch.step(u + g * (c - u), t, x)["prev_sample"]
        bad[row] = _mismatches(out, want)
        del want
        if row in NUMPY_ROWS:
            _numpy_agrees(LSV.cfg_ddim_v, (u, c, x), out, coef[row], g, seed=row)
        if row == 49:
            _edges(f"cfg_ddim_v g={g} {roles} step {row}", out)
    assert bad.sum().item() == 0, {r: v for r, v in enumerate(bad.tolist()) if v}


# ------------------------------------------------------------------------------------------------
# b. tf_ddim_v over every fp16 input, both 500-step tables, out of place and in place
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ddim_sweep():
    s = torch.from_numpy(LS.structured_fp16()).cuda()
    m = len(s)
    allv = torch.from_numpy(LS.ALL_FP16.view(np.int16).copy()).cuda().view(torch.float16)
    v = torch.cat([allv.repeat(m), s.repeat_interleave(1 << 16)])
    x = torch.cat([s.repeat_interleave(1 << 16), allv.repeat(m)])
    return v, x


@pytest.mark.parametrize("direction", ["inversion", "reconstruction"])
def test_ddim_v_every_fp16_input(ops, ddim_sweep, direction):
    v, x = ddim_sweep
    sch = _schedule(500)
    inv, rec = inversion_coef_tables(sch)
    table = (inv if direction == "inversion" else rec).cuda()
    out, xi = torch.empty_like(x), torch.empty_like(x)
    bad = torch.zeros(500, 2, dtype=torch.int64, device="cuda")
    subnormal = 0
    for i in range(500):
        want = OIV.v_expression(x, v, direction, OI.step_alphas(sch, direction, i))
        ops.ddim_v(v, x, table[i], out=out)
        bad[i, 0] = _mismatches(out, want)
        xi.copy_(x)
        assert ops.ddim_v(v, xi, table[i], out=xi).data_ptr() == xi.data_ptr()
        bad[i, 1] = _mismatches(xi, want)
        if i in (0, 1, 97, 250, 498, 499):
            _numpy_agrees(LSV.ddim_v, (v, x), out, table[i], seed=i)
            subnormal += _edges(f"ddim_v {direction} step {i}", out)
    assert bad.sum().item() == 0, {i: b for i, b in enumerate(bad.tolist()) if any(b)}
    assert subnormal > 0


# ------------------------------------------------------------------------------------------------
# c. every length, outputs between guard bands; every operand offset
# ------------------------------------------------------------------------------------------------
GUARD = 64
SENTINEL = 0x7E5A                           # an fp16 NaN payload the kernels never produce
LENGTHS = list(range(1, 41)) + [8 * k + r for k in (255, 256, 257, 1023, 2049) for r in range(8)]


def _guarded(n):
    buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.int16, device="cuda")
    return buf, buf[GUARD:GUARD + n].view(torch.float16)


def _guards_intact(buf):
    return bool((buf[:GUARD] == SENTINEL).all()) and bool((buf[-GUARD:] == SENTINEL).all())


def test_v_step_ops_write_exactly_n_outputs(ops):
    sch = _schedule(50)
    coef = _edit_coefs(sch)
    sch500 = _schedule(500)
    inv = inversion_coef_tables(sch500)[0].cuda()
    alphas = OI.step_alphas(sch500, "inversion", 300)
    g = torch.Generator(device="cuda").manual_seed(4)
    for n in LENGTHS:
        u, c, x, e = (torch.randn(n, device="cuda", generator=g).half() for _ in range(4))
        buf, out = _guarded(n)
        assert ops.cfg_ddim_v(u, c, x, coef[17], 7.5, out=out).data_ptr() == out.data_ptr()
        want = sch.step(u + 7.5 * (c - u), int(sch.timesteps[17]), x)["prev_sample"]
        assert _mismatches(out, want).item() == 0 and _guards_intact(buf), n
        want = OIV.v_expression(x, e, "inversion", alphas)
        buf, out = _guarded(n)
        ops.ddim_v(e, x, inv[300], out=out)
        assert _mismatches(out, want).item() == 0 and _guards_intact(buf), n
        buf, xi = _guarded(n)
        xi.copy_(x)
        ops.ddim_v(e, xi, inv[300], out=xi)
        assert _mismatches(xi, want).item() == 0 and _guards_intact(buf), n


def _at(t, off, channels_last=False):
    buf = torch.empty(t.numel() + 16, dtype=t.dtype, device=t.device)
    flat = buf[off:off + t.numel()]
    if channels_last:
        n, c, h, w = t.shape
        view = flat.view(n, h, w, c).permute(0, 3, 1, 2)
    else:
        view = flat.view(t.shape)
    view.copy_(t)
    return view


def test_cfg_ddim_v_at_every_operand_offset(ops):
    torch.manual_seed(8)
    shape = (3, 4, 13, 21)
    u, c, x = (torch.randn(shape, device="cuda").half() for _ in range(3))
    coef = _edit_coefs(_schedule(50))[23]
    want = ops.cfg_ddim_v(u, c, x, coef, 7.5)
    us, cs, xs, outs = ([_at(t, o) for o in range(8)] for t in (u, c, x, torch.zeros_like(u)))
    bad = torch.zeros((), dtype=torch.int64, device="cuda")
    for iu in range(8):
        for ic in range(8):
            for ix in range(8):
                for io in range(8):
                    got = ops.cfg_ddim_v(us[iu], cs[ic], xs[ix], coef, 7.5, out=outs[io])
                    assert got.data_ptr() == outs[io].data_ptr()
                    bad += _mismatches(got, want)
    assert bad.item() == 0


@pytest.mark.parametrize("v_layout", ["contiguous", "channels_last"])
def test_ddim_v_at_every_operand_offset(ops, v_layout):
    torch.manual_seed(9)
    shape = (3, 4, 13, 21)
    v, x = torch.randn(shape, device="cuda").half(), (2 * torch.randn(shape, device="cuda")).half()
    coef = inversion_coef_tables(_schedule(500))[1][200].cuda()
    want = ops.ddim_v(v, x, coef)
    vs = [_at(v, o, channels_last=v_layout == "channels_last") for o in range(8)]
    xs, outs = [_at(x, o) for o in range(8)], [_at(torch.zeros_like(x), o) for o in range(8)]
    bad = torch.zeros((), dtype=torch.int64, device="cuda")
    for iv in range(8):
        for ix in range(8):
            for io in range(8):
                got = ops.ddim_v(vs[iv], xs[ix], coef, out=outs[io])
                assert got.data_ptr() == outs[io].data_ptr()
                bad += _mismatches(got, want)
            assert torch.equal(xs[ix], x)
            xi = _at(x, ix)
            got = ops.ddim_v(vs[iv], xi, coef, out=xi)
            assert got.data_ptr() == xi.data_ptr()
            bad += _mismatches(xi, want)
    assert bad.item() == 0


# ------------------------------------------------------------------------------------------------
# d. the tiny UNet at 13 x 21 latents with a v scheduler
# ------------------------------------------------------------------------------------------------
ODD = (13, 21)


def _canny(n, h, w, seed=5):
    rng = np.random.default_rng(seed)
    frames = torch.from_numpy(np.stack([gg.make_frame("smooth", h, w, rng) for _ in range(n)])).cuda()
    return preprocess.canny_cond(frames)


def _tiny_edit(mode, steps, graph=False, world=1, rank=0, comm=None, unet=None, controlnet=False, kind=V):
    if unet is None:
        unet = sd_unet.build_unet("tiny", seed=1, device="cuda", dtype=torch.float16)
    cfg = {"n_frames": 6, "batch_size": 2, "n_timesteps": steps, "guidance_scale": 7.5, "mode": mode,
           "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "start": 0.9, "fused_pass": True, "cuda_graph": graph, "keyframe_seed": 1}
    x, text, pnp, src = synthetic_inputs(6, ODD, unet.config.cross_attention_dim, steps, seed=1, device="cuda",
                                         dtype=torch.float16, ctx_len=7)
    kw = {}
    if controlnet:
        kw = dict(controlnet=ControlNetModel.from_unet(unet), controlnet_cond=_canny(6, 8 * ODD[0], 8 * ODD[1]))
    ed = TokenFlowEditor(unet, DDIMScheduler(prediction_type=kind), tfu, cfg, text, pnp,
                         source_latents=lambda t: src[t], world_size=world, rank=rank, **kw)
    if comm is not None:
        ed.attach_communicator(comm)
    ed.init_method()
    return ed.sample_loop(x), ed.keyframe_log, ed


@pytest.mark.parametrize("mode,steps,controlnet", [("pnp", 5, False), ("sdedit", 10, False), ("pnp", 5, True)],
                         ids=["pnp", "sdedit", "pnp-controlnet"])
def test_tiny_unet_v_edit_graphed_equals_eager_at_13x21(mode, steps, controlnet):
    tfu._install_ops_for_testing(None)
    eager, kf_e, _ = _tiny_edit(mode, steps, controlnet=controlnet)
    graphed, kf_g, ed = _tiny_edit(mode, steps, graph=True, controlnet=controlnet)
    assert all(e["replays"] >= 1 for e in ed._graphs.values())
    assert kf_g == kf_e and torch.isfinite(eager).all() and eager.shape == (6, 4) + ODD
    assert torch.equal(graphed, eager), (graphed.float() - eager.float()).abs().max().item()
    eps, _, _ = _tiny_edit(mode, steps, controlnet=controlnet, kind="epsilon")
    assert not torch.equal(eps, eager)


def _thread_world():
    spec = importlib.util.spec_from_file_location("_tf_gpu_round2", os.path.join(REPO, "tests", "test_gpu_round2.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod._ThreadWorld


def test_two_rank_threads_v_edit_at_13x21():
    tfu._install_ops_for_testing(None)
    tfu._ops()
    unets = [sd_unet.build_unet("tiny", seed=1, device="cuda", dtype=torch.float16) for _ in range(3)]
    want, kf_want, _ = _tiny_edit("pnp", 5, unet=unets[2])
    tw = _thread_world()(2)
    res = {}

    def run(r):
        try:
            res[r] = _tiny_edit("pnp", 5, world=2, rank=r, comm=tw.rank(r), unet=unets[r])[:2]
        except BaseException as ex:  # noqa: BLE001
            res[r] = ex
            tw.barrier.abort()

    threads = [threading.Thread(target=run, args=(r,)) for r in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=600)
    errors = [res.get(r) for r in range(2) if not isinstance(res.get(r), tuple)]
    errors.sort(key=lambda e: isinstance(e, threading.BrokenBarrierError))
    assert not errors, errors
    for r in range(2):
        got, kf = res[r]
        assert kf == kf_want and torch.isfinite(got).all()
        rel = (got.float() - want.float()).norm() / want.float().norm()
        assert rel.item() < 2e-2, (r, rel.item())
    assert torch.equal(res[0][0], res[1][0])


def _inversion_equals_the_oracle(unet, x0, cond, steps, batch_size):
    res = {}
    for graphed in (True, False):
        inv = LatentInverter(unet, DDIMScheduler(prediction_type=V), steps)
        inv._use_graph = graphed
        xT = inv.ddim_inversion(cond, x0, None, batch_size=batch_size)
        res[graphed] = (xT, inv.ddim_sample(xT, cond, batch_size=batch_size), inv.saved_latents(), inv.scheduler)
    assert torch.equal(res[True][0], res[False][0]) and torch.equal(res[True][1], res[False][1])
    for t in res[True][2]:
        assert torch.equal(res[True][2][t], res[False][2][t]), t
    sch = res[True][3]
    want_T, want_saved = OIV.ddim_inversion_v(unet, sch, cond, x0.clone(), batch_size)
    want_rec = OIV.ddim_sample_v(unet, sch, want_T.clone(), cond, batch_size)
    assert torch.isfinite(want_rec).all()
    assert torch.equal(res[True][0], want_T), (res[True][0].float() - want_T.float()).abs().max().item()
    assert torch.equal(res[True][1], want_rec), (res[True][1].float() - want_rec.float()).abs().max().item()
    assert sorted(res[True][2]) == sorted(want_saved)
    for t, lat in want_saved.items():
        assert torch.equal(res[True][2][t], lat), t
    eps_T, _ = OI.ddim_inversion(unet, sch, cond, x0.clone(), batch_size)
    assert not torch.equal(eps_T, want_T)


def test_tiny_unet_v_inversion_equals_the_oracle_loop_at_13x21():
    tfu._install_ops_for_testing(None)
    unet = sd_unet.build_unet("tiny", seed=1, device="cuda", dtype=torch.float16)
    g = torch.Generator().manual_seed(3)
    x0 = torch.randn(5, 4, *ODD, generator=g).half().cuda()
    cond = torch.randn(1, 7, unet.config.cross_attention_dim, generator=g).half().cuda()
    _inversion_equals_the_oracle(unet, x0, cond, 8, 2)


# ------------------------------------------------------------------------------------------------
# e. SD2.1 channels_last at C4's 96 x 96 latents
# ------------------------------------------------------------------------------------------------
def _sd21():
    unet = sd_unet.build_unet("sd21", seed=1, device="cuda", dtype=torch.float16, init_on_device=True)
    return unet.to(memory_format=torch.channels_last)


def test_sd21_channels_last_v_edit_at_96x96():
    """8 frames, B = 4, SDEdit with 3 steps (start 0.9: the last one runs): graphed == eager."""
    tfu._install_ops_for_testing(None)
    outs = []
    for graph in (False, True):
        unet = _sd21()
        cfg = {"n_frames": 8, "batch_size": 4, "n_timesteps": 3, "guidance_scale": 7.5, "mode": "sdedit",
               "start": 0.9, "fused_pass": True, "cuda_graph": graph, "keyframe_seed": 1}
        x, text, pnp, src = synthetic_inputs(8, 96, unet.config.cross_attention_dim, 3, seed=1, device="cuda",
                                             dtype=torch.float16, ctx_len=7)
        ed = TokenFlowEditor(unet, DDIMScheduler(prediction_type=V), tfu, cfg, text, pnp,
                             source_latents=lambda t: src[t])
        ed.init_method()
        outs.append((ed.sample_loop(x), ed.keyframe_log))
        del ed, unet
        torch.cuda.empty_cache()
    assert outs[0][1] == outs[1][1]
    assert outs[0][0].shape == (8, 4, 96, 96) and torch.isfinite(outs[0][0]).all()
    assert torch.equal(outs[1][0], outs[0][0])


def test_sd21_channels_last_v_inversion_at_96x96():
    tfu._install_ops_for_testing(None)
    unet = _sd21()
    g = torch.Generator().manual_seed(3)
    x0 = torch.randn(4, 4, 96, 96, generator=g).half().cuda()
    cond = torch.randn(1, 77, unet.config.cross_attention_dim, generator=g).half().cuda()
    _inversion_equals_the_oracle(unet, x0, cond, 3, 2)
