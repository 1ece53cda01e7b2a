"""CPU tier: the multi-GPU path (the fused step: frames sharded, keyframe tensors all-gathered) on 2 gloo
ranks with the oracle ops == the single-process loop of the reference's schedule.  Covers the shard plan, the
all-gather ordering and routing, the per-frame keyframe/weight tables and the sharded attention table."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tokenflow_b200 import tokenflow_utils as tfu


def _init_file(tmp_path_factory=None):
    """file:// rendezvous: no port to race for (ADVICE r1)."""
    import tempfile
    fd, path = tempfile.mkstemp(prefix="tf_b200_rdzv_")
    os.close(fd)
    os.unlink(path)
    return path


def _edit(world, rank, mode, steps, fused=False):
    from oracle.oracle_ops import OracleOps
    from tokenflow_b200 import sd_unet
    from tokenflow_b200.editor import TokenFlowEditor, synthetic_inputs
    from tokenflow_b200.scheduler import DDIMScheduler
    tfu._install_ops_for_testing(OracleOps())
    unet = sd_unet.build_unet("tiny", seed=1)
    cfg = {"n_frames": 8, "batch_size": 2, "n_timesteps": steps, "guidance_scale": 7.5, "mode": mode,
           "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "start": 0.9, "fused_pass": fused}
    x, text, pnp, src = synthetic_inputs(8, 16, unet.config.cross_attention_dim, steps, seed=1, ctx_len=7)
    ed = TokenFlowEditor(unet, DDIMScheduler(), tfu, cfg, text, pnp, source_latents=lambda t: src[t],
                         world_size=world, rank=rank)
    ed.init_method()
    torch.manual_seed(1)
    return ed.sample_loop(x), ed.keyframe_log


def _worker(rank, world, rdzv, mode, steps, q):
    torch.set_num_threads(2)
    dist.init_process_group("gloo", init_method=f"file://{rdzv}", rank=rank, world_size=world)
    try:
        out, kf = _edit(world, rank, mode, steps, fused=True)
        # plain Python data on the queue: a torch tensor would travel by file-descriptor passing, which needs
        # the sender alive until the parent has rebuilt it (the worker exits right after the put)
        q.put((rank, out.numpy().tolist(), kf))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("mode,steps", [("pnp", 2), ("sdedit", 10)])
def test_two_rank_edit_equals_single_process(mode, steps):
    want, kf_want = _edit(1, 0, mode, steps)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    rdzv = _init_file()
    procs = [ctx.Process(target=_worker, args=(r, 2, rdzv, mode, steps, q)) for r in range(2)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, out, kf in results:
        assert kf == kf_want
        assert torch.allclose(torch.tensor(out), want, atol=2e-4, rtol=1e-4), f"rank {rank}"


def test_shard_plan_and_global_attention_table():
    K = 5
    for G in (2, 4, 8):
        m = -(-15 // G)
        seen = []
        for r in range(G):
            sh = tfu.PivotalShard(G, r, K)
            assert len(sh.slots) == m
            seen += sh.slots
            tab = sh.global_attention_table(False)
            tab_inj = sh.global_attention_table(True)
            assert len(tab) == len(tab_inj) == 15
            for i in range(15):
                for qs, k0, v0, nkv in (tab[i], tab_inj[i]):       # inside the G*m gathered slabs
                    assert 0 <= qs < G * m and 0 <= k0 and k0 + nkv <= G * m and 0 <= v0 and v0 + nkv <= G * m
                s, f = divmod(i, K)
                if s == 0:
                    assert tab[i] == tab_inj[i] == (i, i, i, 1)
                else:
                    assert tab[i] == (i, s * K, s * K, K)
                    assert tab_inj[i] == (f, 0, s * K, K)       # q and k of the source stream, own v
        assert seen == list(range(G * m))                       # every slot once; the first 15 are the samples


def test_all_gather_routes(monkeypatch):
    """`ops.all_gather`: one rank returns its input; a CPU tensor never reaches an attached communicator (tf_allgather
    would read it as device memory) but goes through torch.distributed, contiguous; the communicator itself refuses
    anything that is not on the current CUDA device."""
    from tokenflow_b200 import ops
    t = torch.arange(12.0).view(3, 4)
    assert ops.all_gather(t, 1, comm=object()) is t

    class RecordingComm:
        calls = 0

        def all_gather(self, t):
            RecordingComm.calls += 1
            return t

    recorded = []

    def all_gather_into_tensor(out, t, group=None):
        recorded.append((tuple(out.shape), t.is_contiguous(), group))
        out.copy_(torch.cat([t, t + 100]))

    monkeypatch.setattr(dist, "all_gather_into_tensor", all_gather_into_tensor)
    got = ops.all_gather(t.t(), 2, group="g", comm=RecordingComm())     # a strided view
    assert RecordingComm.calls == 0
    assert recorded == [((8, 3), True, "g")]
    assert torch.equal(got, torch.cat([t.t(), t.t() + 100]))
    with pytest.raises(ops.TokenflowB200Error):
        ops.Communicator.__new__(ops.Communicator).all_gather(t)


def test_frame_table_matches_batch_idx_arithmetic():
    from oracle import tokenflow_oracle as O
    from tokenflow_b200.editor import TokenFlowEditor
    ed = TokenFlowEditor.__new__(TokenFlowEditor)
    ed.config = {"batch_size": 8}
    kf_a, kf_b, w = TokenFlowEditor.frame_table(ed, list(range(5, 10)))     # rank 1 of 8 at N=40: spans batches 0,1
    assert kf_a == [0, 0, 0, 1, 1] and kf_b == [-1, -1, -1, 0, 0]
    ref = O.blend_weights(1, 8)
    assert abs(w[3] - float(ref[0])) < 1e-7 and abs(w[4] - float(ref[1])) < 1e-7
