"""GPU tier (-m gpu): videos of any length on the H100.

* The graphed step in frame chunks == the same step eager, bit for bit: the tiny UNet at 13 x 21 latents with N = 13,
  B = 4 (a short last keyframe group), PnP over all three graph variants, SDEdit, PnP with a ControlNet, an eps and a v
  scheduler; SD1.5 channels_last at 64 x 64 with N = 20, B = 8 and chunks of 6 frames.
* Chunked == unchunked on SD1.5 channels_last, and 3 rank threads with uneven shares == one rank, within the relative
  L2 bound the sharded path is held to.
* The kernels at the new shapes: the NN field and propagation of a pass whose frames include a short last group, and
  extended attention over 3 ceil(N / B) samples, against oracle/kernel_checks.py.
* Without `frames_per_pass` a replay of the captured step launches the library kernels of one fused call, in order;
  with chunks the graphed step's peak memory is lower.
"""
import importlib.util
import os
import threading

import pytest
import torch

from oracle import kernel_checks as KC
from tokenflow_b200 import ops as tf_ops
from tokenflow_b200 import sd_unet
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.editor import TokenFlowEditor, synthetic_inputs
from tokenflow_b200.scheduler import DDIMScheduler

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ODD = (13, 21)


def _editor(kind="tiny", mode="pnp", steps=5, n_frames=13, batch=4, latent=ODD, chunk=None, graph=False,
            prediction="epsilon", controlnet=False, world=1, rank=0, comm=None, unet=None):
    if unet is None:
        unet = sd_unet.build_unet(kind, seed=1, device="cuda", dtype=torch.float16, init_on_device=kind != "tiny")
        if kind != "tiny":
            unet = unet.to(memory_format=torch.channels_last)
    cfg = {"n_frames": n_frames, "batch_size": batch, "n_timesteps": steps, "guidance_scale": 7.5, "mode": mode,
           "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "start": 0.9, "fused_pass": True, "cuda_graph": graph, "keyframe_seed": 1}
    if chunk is not None:
        cfg["frames_per_pass"] = chunk
    x, text, pnp, src = synthetic_inputs(n_frames, latent, unet.config.cross_attention_dim, steps, seed=1,
                                         device="cuda", dtype=torch.float16, ctx_len=7)
    kw = {}
    if controlnet:
        from tokenflow_b200.controlnet import build_controlnet
        h, w = (latent, latent) if isinstance(latent, int) else latent
        g = torch.Generator().manual_seed(5)
        kw = dict(controlnet=build_controlnet(kind, seed=3, device="cuda", dtype=torch.float16),
                  controlnet_cond=torch.rand(n_frames, 3, 8 * h, 8 * w, generator=g).cuda())
    ed = TokenFlowEditor(unet, DDIMScheduler(prediction_type=prediction), tfu, cfg, text, pnp,
                         source_latents=lambda t: src[t], world_size=world, rank=rank, **kw)
    if comm is not None:
        ed.attach_communicator(comm)
    ed.init_method()
    return ed, x


@pytest.mark.parametrize("chunk", [3, 13])
@pytest.mark.parametrize("mode,steps,prediction,controlnet", [
    pytest.param("pnp", 5, "epsilon", False, id="pnp"),
    pytest.param("sdedit", 10, "epsilon", False, id="sdedit"),
    pytest.param("pnp", 5, "epsilon", True, id="pnp-controlnet"),
    pytest.param("pnp", 5, "v_prediction", False, id="pnp-v")])
def test_tiny_graphed_chunks_equal_eager(mode, steps, prediction, controlnet, chunk):
    tfu._install_ops_for_testing(None)
    kw = dict(mode=mode, steps=steps, prediction=prediction, controlnet=controlnet, chunk=chunk)
    ed_e, x = _editor(**kw)
    want = ed_e.sample_loop(x.clone())
    ed_g, x = _editor(graph=True, **kw)
    got = ed_g.sample_loop(x.clone())
    assert ed_g.keyframe_log == ed_e.keyframe_log
    assert all(len(kf) == 4 and kf[-1] == 12 for kf in ed_g.keyframe_log)          # the short last group: frame 12
    if mode == "pnp":
        assert len(ed_g._graphs) == 3                      # q/k + conv injection, conv injection only, none
    assert all(e["replays"] >= 1 for e in ed_g._graphs.values())
    assert got.shape == (13, 4) + ODD and torch.isfinite(got).all()
    assert torch.equal(got, want), (got.float() - want.float()).abs().max().item()


def test_sd15_graphed_chunks_equal_eager_and_unchunked():
    """N = 20, B = 8 (groups of 8, 8, 4), chunks of 6: graphed == eager bit for bit; against the unchunked step the
    criterion of the sharded path (relative L2 < 2e-2 after 4 steps, the same keyframes)."""
    tfu._install_ops_for_testing(None)
    kw = dict(kind="sd15", steps=4, n_frames=20, batch=8, latent=64)
    outs = {}
    for name, extra in (("eager", dict(chunk=6)), ("graph", dict(chunk=6, graph=True)), ("whole", dict(graph=True))):
        ed, x = _editor(**kw, **extra)
        outs[name] = (ed.sample_loop(x.clone()), ed.keyframe_log)
        del ed
        torch.cuda.empty_cache()
    assert outs["graph"][1] == outs["eager"][1] == outs["whole"][1]
    assert torch.isfinite(outs["graph"][0]).all()
    assert torch.equal(outs["graph"][0], outs["eager"][0])
    want = outs["whole"][0].float()
    rel = ((outs["graph"][0].float() - want).norm() / want.norm()).item()
    assert rel < 2e-2, rel


def _thread_world():
    spec = importlib.util.spec_from_file_location("_tf_gpu_round2", os.path.join(REPO, "tests", "test_gpu_round2.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod._ThreadWorld


@pytest.mark.parametrize("n_frames,chunk", [(10, None), (40, None), (40, 5)])
def test_three_uneven_rank_threads_equal_one_rank(n_frames, chunk):
    """3 ranks: 10 frames in shares 4, 4, 2 and 40 in 14, 14, 12, B = 4 (40 frames: also in chunks of 5)."""
    world, steps = 3, 4
    tfu._install_ops_for_testing(None)
    tfu._ops()                                              # one op object for all threads
    unets = [sd_unet.build_unet("tiny", seed=1, device="cuda", dtype=torch.float16) for _ in range(world + 1)]

    def run(world_size, rank, comm, out, unet):
        try:
            ed, x = _editor(steps=steps, n_frames=n_frames, latent=16, chunk=chunk, world=world_size, rank=rank,
                            comm=comm, unet=unet)
            per_step = []
            out[rank] = (ed.sample_loop(x, on_step=lambda i, t, z: per_step.append(z.float())), ed.keyframe_log,
                         per_step)
        except BaseException as ex:  # noqa: BLE001
            out[rank] = ex
            if comm is not None:
                comm.parent.barrier.abort()

    ref = {}
    run(1, 0, None, ref, unets[world])
    assert not isinstance(ref[0], BaseException), ref[0]
    want, kf_want, _ = ref[0]
    tw = _thread_world()(world)
    res = {}
    threads = [threading.Thread(target=run, args=(world, r, tw.rank(r), res, unets[r])) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=600)
    errors = [res.get(r) for r in range(world) if not isinstance(res.get(r), tuple)]
    errors.sort(key=lambda e: isinstance(e, threading.BrokenBarrierError))      # the cause first
    assert not errors, errors
    for r in range(world):
        got, kf, _ = res[r]
        assert kf == kf_want and torch.isfinite(got).all()
        rel = ((got.float() - want.float()).norm() / want.float().norm()).item()
        assert rel < 2e-2, (r, rel)
    for i in range(steps):                                  # every rank ends every step with the same latents
        for r in range(1, world):
            assert torch.equal(res[r][2][i], res[0][2][i]), (i, r)


def test_kernels_at_a_short_last_group():
    """N = 13, B = 4: K = 4 keyframes, the last of a group of one frame.  The NN field and propagation of all 13
    frames in one pass (frame 12's kf_a is the short group), and extended attention over the 3K = 12 samples."""
    tfu._install_ops_for_testing(None)
    ops = tf_ops.CudaOps()
    N, B, S, dim, heads = 13, 4, 256, 320, 5
    K = -(-N // B)
    ed = TokenFlowEditor.__new__(TokenFlowEditor)
    ed.config = {"batch_size": B}
    kf_a, kf_b, w = ed.frame_table(list(range(N)))
    assert kf_a[-1] == K - 1 and kf_b[-1] == K - 2
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.randn(N, S, dim, device="cuda", generator=g).half()
    piv = torch.randn(K, S, dim, device="cuda", generator=g).half()
    x_unit, piv_unit = ops.unit_rows(x), ops.unit_rows(piv)
    idx_a, idx_b = ops.nn_field(x_unit, piv_unit, kf_a, kf_b)
    KC.check_nn_field(idx_a, idx_b, x_unit, piv_unit, kf_a, kf_b, tag="N=13,B=4")
    A = torch.randn(3, K, S, dim, device="cuda", generator=g).half()
    residual = torch.randn(3 * N, S, dim, device="cuda", generator=g).half()
    for out_dtype in (torch.float16, torch.float32):
        got = ops.propagate(A, idx_a, idx_b, kf_a, kf_b, w, residual=residual, out_dtype=out_dtype)
        want = KC.propagate_exact(A, idx_a, idx_b, kf_a, kf_b, w, residual, out_dtype)
        assert torch.equal(got.cpu(), want), out_dtype
    q, k, v = (torch.randn(3 * K, S, dim, device="cuda", generator=g).half() for _ in range(3))
    scale = (dim // heads) ** -0.5
    for inject in (False, True):
        table = KC.ext_attn_samples(K, inject)
        assert len(table) == 3 * K
        got = ops.ext_attn(q, k, v, heads, scale, inject)
        KC.check_ext_attn(got, q, k, v, table, heads, scale)


def test_default_step_launches_one_fused_call():
    """Without frames_per_pass (and with it at the rank's frame count) one replay of the captured step launches the
    library kernels of one eager fused call, in the same order."""
    tfu._install_ops_for_testing(None)
    ops = tfu._ops()
    calls = []
    launch = ops._launch

    def recording(timer, work, fn, *args):
        calls.append((fn, torch.cuda.is_current_stream_capturing()))
        return launch(timer, work, fn, *args)

    ops._launch = recording
    try:
        ed, x = _editor(n_frames=13)
        n0 = ops.launch_count()
        ed.step_index(x.clone(), 0)
        eager, eager_kernels = [fn for fn, _ in calls], ops.launch_count() - n0
        for chunk in (None, 13):
            calls.clear()
            ed_g, x = _editor(n_frames=13, graph=True, chunk=chunk)
            ed_g.step_index(x.clone(), 0)
            captured = [fn for fn, cap in calls if cap]
            assert captured == eager, chunk
            assert ed_g.graph_launches_per_step() == eager_kernels
        calls.clear()
        ed_c, x = _editor(n_frames=13, graph=True, chunk=3)
        ed_c.step_index(x.clone(), 0)
        chunked = [fn for fn, cap in calls if cap]
        assert chunked != eager and chunked.count("tf_nn_field") > eager.count("tf_nn_field")
    finally:
        del ops._launch


def test_chunks_lower_the_peak_memory():
    """SD1.5 channels_last at 64 x 64, 40 frames, B = 8: the graphed step's peak allocation, capture included, is
    lower in chunks of 8 frames than in one call."""
    tfu._install_ops_for_testing(None)
    peaks = {}
    for chunk in (None, 8):
        # a UNet per arm: its blocks keep the last keyframe caches, which would hold on to the other arm's graph pool
        ed, x = _editor(kind="sd15", steps=2, n_frames=40, batch=8, latent=64, graph=True, chunk=chunk)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        ed.step_index(x, 0)
        ed.step_index(x, 1)
        torch.cuda.synchronize()
        peaks[chunk] = torch.cuda.max_memory_allocated()
        del ed, x
        torch.cuda.empty_cache()
    print({k: round(v / 2 ** 30, 2) for k, v in peaks.items()})
    assert peaks[8] < peaks[None], peaks
