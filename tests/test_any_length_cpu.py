"""CPU tier: videos of any length through the editor, on the oracle ops.

* Keyframes: a last keyframe group of r = N mod B frames gets one more draw; when B divides N the draws are the ones the
  editor always made, from the global RNG and from `keyframe_seed`.
* The frame table of a short last group keeps the stride B: its weights are `closed_form.blend_weight(g % B, B)`, and a
  TokenFlow block's output for the tail frames is `closed_form.propagate` of the group.
* The fused step in frame chunks == the unchunked fused step == the non-fused schedule, at N = K B + r.
* Uneven frame shards on gloo ranks == one rank, with and without chunks; a split that leaves a rank without frames is
  refused.
"""
import os
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import closed_form
from oracle.oracle_ops import OracleOps
from tokenflow_b200 import sd_unet
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.editor import TokenFlowEditor, synthetic_inputs
from tokenflow_b200.ops import frame_share
from tokenflow_b200.scheduler import DDIMScheduler

B = 4


def _keyframe_editor(batch, **cfg):
    ed = TokenFlowEditor.__new__(TokenFlowEditor)
    ed.config = dict(cfg, batch_size=batch)
    ed.world_size, ed.rank = 1, 0
    ed._kf_gen = torch.Generator().manual_seed(cfg["keyframe_seed"]) if "keyframe_seed" in cfg else None
    return ed


def _draws_before(n, batch, gen=None):
    """The editor's draws for n a multiple of the batch: randint(B, (n // B,)) + arange(0, n, B)."""
    kw = {} if gen is None else {"generator": gen}
    return torch.randint(batch, (n // batch,), **kw) + torch.arange(0, n, batch)


@pytest.mark.parametrize("seeded", [False, True])
@pytest.mark.parametrize("n,batch", [(8, 2), (40, 8), (192, 16), (4, 4)])
def test_keyframes_unchanged_when_the_batch_divides_the_frames(n, batch, seeded):
    cfg = {"keyframe_seed": 3} if seeded else {}
    ed = _keyframe_editor(batch, **cfg)
    torch.manual_seed(5)
    got = [ed.draw_keyframes(n) for _ in range(3)]
    gen = torch.Generator().manual_seed(3) if seeded else None
    torch.manual_seed(5)
    want = [_draws_before(n, batch, gen) for _ in range(3)]
    for g, w in zip(got, want):
        assert torch.equal(g, w)


@pytest.mark.parametrize("seeded", [False, True])
@pytest.mark.parametrize("n,batch", [(9, 4), (11, 4), (3, 4), (1, 8), (200, 16), (13, 4)])
def test_short_last_group_gets_its_own_keyframe(n, batch, seeded):
    cfg = {"keyframe_seed": 7} if seeded else {}
    full, r = divmod(n, batch)
    for trial in range(20):
        ed = _keyframe_editor(batch, **cfg)
        torch.manual_seed(trial)
        idx = ed.draw_keyframes(n)
        assert idx.shape == (full + 1,)
        assert n - r <= int(idx[-1]) < n
        # the full groups are drawn first, exactly as before; the last draw is randint(r) from the same generator
        gen = torch.Generator().manual_seed(7) if seeded else None
        torch.manual_seed(trial)
        want = _draws_before(full * batch, batch, gen)
        last = torch.randint(r, (1,), **({} if gen is None else {"generator": gen})) + full * batch
        assert torch.equal(idx, torch.cat([want, last]))
    for k, f in enumerate(idx.tolist()):
        assert k * batch <= f < min(n, (k + 1) * batch)


@pytest.mark.parametrize("n,batch", [(9, 4), (11, 4), (23, 8), (200, 16), (3, 4)])
def test_frame_table_of_tail_frames_keeps_the_stride(n, batch):
    ed = _keyframe_editor(batch)
    frames = list(range(n - n % batch, n))
    kf_a, kf_b, w = ed.frame_table(frames)
    for g, a, b, wg in zip(frames, kf_a, kf_b, w):
        assert a == g // batch and b == (g // batch - 1 if g >= batch else -1)
        assert abs(wg - closed_form.blend_weight(g % batch, batch)) < 1e-6


@pytest.mark.parametrize("r", [1, B - 1])
def test_tail_frames_propagate_from_the_short_group(r):
    """One TokenFlow block: pivotal pass over K = 3 keyframes, then the frame pass of the r tail frames with the
    editor's frame table; the propagated rows equal `closed_form.propagate` of the last group (its first r frames of a
    nominal group of B)."""
    tfu._install_ops_for_testing(OracleOps())
    torch.manual_seed(0)
    dim, heads, S, K = 32, 2, 16, 3
    N = (K - 1) * B + r
    block = sd_unet.BasicTransformerBlock(dim, heads, dim // heads, 24).eval()
    model = torch.nn.Module()
    model.unet = torch.nn.Module()
    model.unet.block = block
    tfu.register_extended_attention(model)
    tfu.set_tokenflow(model.unet)
    ed = _keyframe_editor(B)
    with torch.no_grad():
        block._tf_pivotal(torch.randn(3 * K, S, dim), None, {})
        hidden = torch.randn(3 * r, S, dim)
        tfu.register_frame_table(model, *ed.frame_table(list(range(N - r, N))))
        out = block._tf_frames(hidden)
    idx_a, idx_b = block._tf_nn_idx
    assert idx_b is not None
    pad = lambda idx: np.concatenate([idx.numpy(), np.zeros((B - r, S), dtype=np.int64)])
    want = closed_form.propagate(block.kf_attn_output.view(3, K, S, dim).numpy(), pad(idx_a), pad(idx_b), K - 1, B)
    want = want.reshape(3, B, S, dim)[:, :r].reshape(3 * r, S, dim)
    assert np.allclose((out - hidden).numpy(), want, atol=1e-5, rtol=1e-5)


def _edit(mode, n_frames, world=1, rank=0, fused=True, chunk=None, steps=None, batch=B):
    tfu._install_ops_for_testing(OracleOps())
    unet = sd_unet.build_unet("tiny", seed=1)
    steps = steps or (2 if mode == "pnp" else 4)
    cfg = {"n_frames": n_frames, "batch_size": batch, "n_timesteps": steps, "guidance_scale": 7.5, "mode": mode,
           "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "start": 0.9, "fused_pass": fused, "keyframe_seed": 1}
    if chunk is not None:
        cfg["frames_per_pass"] = chunk
    x, text, pnp, src = synthetic_inputs(n_frames, 16, unet.config.cross_attention_dim, steps, seed=1, ctx_len=7)
    ed = TokenFlowEditor(unet, DDIMScheduler(), tfu, cfg, text, pnp, source_latents=lambda t: src[t],
                         world_size=world, rank=rank)
    ed.init_method()
    steps_out = []
    out = ed.sample_loop(x, on_step=lambda i, t, z: steps_out.append(z.clone()))
    return out, ed.keyframe_log, steps_out


@pytest.mark.parametrize("mode", ["pnp", "sdedit"])
@pytest.mark.parametrize("r", [1, B - 1])
def test_fused_step_in_chunks_equals_the_reference_schedule(mode, r):
    n = 2 * B + r
    want, kf_want, steps_want = _edit(mode, n, fused=False)
    assert all(len(kf) == 3 and n - r <= kf[-1] < n for kf in kf_want)
    for chunk in (None, 1, B - 1, B, 5):
        got, kf, steps_got = _edit(mode, n, chunk=chunk)
        assert kf == kf_want, chunk
        for g, w in zip(steps_got, steps_want):
            assert torch.allclose(g, w, atol=2e-4, rtol=1e-4), chunk
        assert torch.allclose(got, want, atol=2e-4, rtol=1e-4), chunk


def _init_file():
    fd, path = tempfile.mkstemp(prefix="tf_b200_rdzv_")
    os.close(fd)
    os.unlink(path)
    return path


def _worker(rank, world, rdzv, n_frames, chunk, q):
    torch.set_num_threads(1)
    dist.init_process_group("gloo", init_method=f"file://{rdzv}", rank=rank, world_size=world)
    try:
        out, kf, _ = _edit("pnp", n_frames, world=world, rank=rank, chunk=chunk)
        q.put((rank, out.numpy().tolist(), kf))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,n_frames,chunk", [(3, 10, None), (2, 13, None), (2, 13, 3)])
def test_uneven_shards_equal_one_rank(world, n_frames, chunk):
    """3 ranks x 10 frames (shares 4, 4, 2) and 2 ranks x 13 frames (7, 6), both with a short last keyframe group;
    the chunked case gives the ranks different numbers of UNet calls."""
    want, kf_want, _ = _edit("pnp", n_frames)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    rdzv = _init_file()
    procs = [ctx.Process(target=_worker, args=(r, world, rdzv, n_frames, chunk, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, out, kf in results:
        assert kf == kf_want
        assert torch.allclose(torch.tensor(out), want, atol=2e-4, rtol=1e-4), f"rank {rank}"


@pytest.mark.parametrize("n,world", [(9, 4), (5, 4), (1, 2), (10, 6)])
def test_split_without_frames_for_a_rank_is_refused(n, world):
    assert frame_share(n, world, world - 1)[1] <= frame_share(n, world, world - 1)[0]
    tfu._install_ops_for_testing(OracleOps())
    unet = sd_unet.build_unet("tiny", seed=1)
    cfg = {"n_frames": n, "batch_size": B, "n_timesteps": 2, "guidance_scale": 7.5, "mode": "pnp",
           "fused_pass": True, "keyframe_seed": 1}
    x, text, pnp, src = synthetic_inputs(n, 16, unet.config.cross_attention_dim, 2, seed=1, ctx_len=7)
    ed = TokenFlowEditor(unet, DDIMScheduler(), tfu, cfg, text, pnp, source_latents=lambda t: src[t],
                         world_size=world, rank=0)
    ed.init_method()
    with pytest.raises(ValueError, match="without frames"):
        ed.step_index(x, 0)
    assert ed.keyframe_log == []                           # refused before any keyframe is drawn


def test_frames_per_pass_below_one_is_refused():
    tfu._install_ops_for_testing(OracleOps())
    with pytest.raises(ValueError, match="frames_per_pass"):
        _edit("sdedit", 5, chunk=0)
