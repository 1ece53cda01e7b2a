"""CPU tier: host-side logic added in round 2 — the query-row split of the sharded attention, the sample tables, the
DDIM coefficient table of the fused CFG+DDIM kernel, the injection variants that key the step graphs, bench configs."""
import os
import sys

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from oracle.oracle_ops import OracleOps  # noqa: E402
from tokenflow_b200 import sd_unet, tokenflow_utils as tfu  # noqa: E402
from tokenflow_b200.editor import TokenFlowEditor, synthetic_inputs  # noqa: E402
from tokenflow_b200.scheduler import DDIMScheduler  # noqa: E402


@pytest.mark.parametrize("S", [64, 256, 576, 1024, 4096, 9216])
@pytest.mark.parametrize("G", [2, 4, 8])
def test_row_split_tiles_cover_all_tokens_once(S, G):
    covered = []
    nrows_all = set()
    for r in range(G):
        row0, nrows = tfu.PivotalShard(G, r, 5).row_split(S)
        assert row0 % 128 == 0 and nrows % 128 == 0 and nrows > 0
        nrows_all.add(nrows)
        covered += list(range(row0, min(S, row0 + nrows)))
    assert len(nrows_all) == 1                       # equal buffers on every rank (all-gather)
    assert covered == list(range(S))                 # every token exactly once, in order
    assert G * nrows_all.pop() >= S


def test_global_attention_table_matches_the_reference_batch():
    K = 5
    sh = tfu.PivotalShard(8, 3, K)
    plain, inj = sh.global_attention_table(False), sh.global_attention_table(True)
    assert len(plain) == len(inj) == 3 * K
    for i in range(3 * K):
        s, f = divmod(i, K)
        if s == 0:                                   # source stream: own frame only (reference :173,:177)
            assert plain[i] == inj[i] == (i, i, i, 1)
        else:                                        # uncond / cond: all K frames; injection reads the source q, k (:124-130)
            assert plain[i] == (i, s * K, s * K, K)
            assert inj[i] == (f, 0, s * K, K)
    # the uncond and cond sample of a keyframe share q and k when injected -> the C ABI pairs them
    for f in range(K):
        assert inj[K + f][:2] == inj[2 * K + f][:2] and inj[K + f][2] != inj[2 * K + f][2]
    assert sh.local_index("cpu").tolist() == [min(i, 3 * K - 1) for i in sh.slots]
    assert sh.source_index("cpu").tolist() == [i % K if i < 3 * K else i for i in sh.slots]


def test_row_range_attention_of_the_oracle_tiles_the_full_result():
    torch.manual_seed(0)
    n, S, heads, d = 2, 300, 2, 8
    q, k, v = (torch.randn(3 * n, S, heads * d) for _ in range(3))
    sh = tfu.PivotalShard(4, 0, n)
    table = sh.global_attention_table(True)
    ops = OracleOps()
    full = ops.ext_attn_table(q, k, v, table, heads, d ** -0.5)
    parts = []
    for r in range(4):
        row0, nrows = tfu.PivotalShard(4, r, n).row_split(S)
        parts.append(ops.ext_attn_table(q, k, v, table, heads, d ** -0.5, row0=row0, nrows=nrows))
    nrows = parts[0].shape[1]
    got = torch.stack(parts).permute(1, 0, 2, 3).reshape(3 * n, 4 * nrows, heads * d)[:, :S]
    assert torch.allclose(got, full, atol=1e-6)


def _toy_editor(mode="pnp", steps=10):
    unet = sd_unet.build_unet("tiny", seed=1)
    cfg = {"n_frames": 4, "batch_size": 2, "n_timesteps": steps, "guidance_scale": 7.5, "mode": mode,
           "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "start": 0.9}
    x, text, pnp, src = synthetic_inputs(4, 16, unet.config.cross_attention_dim, steps, seed=1, ctx_len=7)
    tfu._install_ops_for_testing(OracleOps())
    ed = TokenFlowEditor(unet, DDIMScheduler(), tfu, cfg, text, pnp, source_latents=lambda t: src[t])
    ed.init_method()
    return ed, x


def test_ddim_coefficient_table_reproduces_scheduler_step():
    """tf_cfg_ddim reads sqrt(1-a_t), 1/sqrt(a_t), sqrt(a_prev), sqrt(1-a_prev) from this table: in fp32 the
    coefficient form must equal DDIMScheduler.step (run_tokenflow_pnp.py:217) for every timestep."""
    ed, x = _toy_editor()
    sch = ed.scheduler
    torch.manual_seed(3)
    eps = torch.randn(4, 4, 16, 16)
    assert ed._coef_table.shape == (len(ed._t_host), 4)
    for i, t in enumerate(ed._t_host):
        s1, inv_s2, s3, s4 = (float(v) for v in ed._coef_table[i])
        want = sch.step(eps, t, x)["prev_sample"]
        got = s3 * ((x - s1 * eps) * inv_s2) + s4 * eps
        assert torch.allclose(got, want, atol=2e-5, rtol=1e-5), t
    assert ed._t_index[ed._t_host[3]] == 3


def test_injection_variants_follow_the_pnp_thresholds():
    ed, _ = _toy_editor("pnp", steps=10)             # q/k injection for the first 5 steps, conv injection for the first 8
    got = [ed._variant(t) for t in ed._t_host]
    assert got == [(True, True)] * 5 + [(False, True)] * 3 + [(False, False)] * 2
    assert ed._variant(1000) == (True, True)         # reference: `t == 1000` always injects (:86, :124)
    ed2, _ = _toy_editor("sdedit", steps=10)
    assert {ed2._variant(t) for t in ed2._t_host} == {(False, False)}


def test_keyframe_generator_is_rank_independent_and_checked():
    """ADVICE r1: ranks must draw identical keyframes whatever else consumed their global RNG."""
    eds = []
    for r in range(2):
        unet = sd_unet.build_unet("tiny", seed=1)
        cfg = {"n_frames": 8, "batch_size": 2, "n_timesteps": 4, "guidance_scale": 7.5, "mode": "pnp", "fused_pass": True}
        x, text, pnp, src = synthetic_inputs(8, 16, unet.config.cross_attention_dim, 4, seed=1, ctx_len=7)
        eds.append(TokenFlowEditor(unet, DDIMScheduler(), tfu, cfg, text, pnp, source_latents=lambda t: src[t],
                                   world_size=2, rank=r))
        torch.manual_seed(100 + r)                   # a per-rank global seed must not matter
        torch.rand(r + 1)
    draws = [[ed.draw_keyframes(8).tolist() for _ in range(3)] for ed in eds]
    assert draws[0] == draws[1]
    for d in draws[0]:
        assert all(2 * i <= k < 2 * i + 2 for i, k in enumerate(d))      # one frame inside every batch


def test_constructor_refuses_schedules_that_do_not_exist():
    """A step runs one way: no dual-stream schedule, and several ranks only with the fused step.  Asking for anything
    else fails in the constructor instead of running another schedule under its name."""
    unet = sd_unet.build_unet("tiny", seed=1)
    x, text, pnp, src = synthetic_inputs(8, 16, unet.config.cross_attention_dim, 4, seed=1, ctx_len=7)
    base = {"n_frames": 8, "batch_size": 2, "n_timesteps": 4, "guidance_scale": 7.5, "mode": "pnp"}

    def make(cfg, world):
        return TokenFlowEditor(unet, DDIMScheduler(), tfu, dict(base, **cfg), text, pnp,
                               source_latents=lambda t: src[t], world_size=world, rank=0)
    for world in (1, 2):
        with pytest.raises(ValueError, match="dual_stream"):
            make({"dual_stream": True, "fused_pass": True}, world)
    for cfg in ({}, {"fused_pass": False}, {"fused_pass": False, "dual_stream": None}):
        with pytest.raises(ValueError, match="fused_pass"):
            make(cfg, 2)
    tfu._install_ops_for_testing(OracleOps())
    for dual in (None, False):
        ed = make({"dual_stream": dual, "fused_pass": True}, 2)
        ed.init_method()
        assert ed.world_size == 2 and ed.config["fused_pass"]
        assert make({"dual_stream": dual, "fused_pass": False}, 1).world_size == 1


def test_register_fused_and_shard_reach_the_conv_site_from_the_unet_itself():
    """ADVICE r1: the helpers are called with the wrapper (`.unet`) or with the UNet itself."""
    unet = sd_unet.build_unet("tiny", seed=1)

    class W(torch.nn.Module):
        def __init__(self, u):
            super().__init__()
            self.unet = u
    w = W(unet)
    tfu.register_conv_injection(w, [981])
    tfu.set_tokenflow(unet)
    site = unet.up_blocks[1].resnets[1]
    for root in (w, unet):
        tfu.register_fused(root, 7)
        assert site._tf_fused == 7
        sh = tfu.PivotalShard(2, 0, 2)
        tfu.register_shard(root, sh)
        assert site._tf_shard is sh
        tfu.register_fused(root, 0)
        tfu.register_shard(root, None)
        assert site._tf_fused == 0 and site._tf_shard is None


def test_bench_configs_match_baseline_json():
    import bench
    assert bench.metric_name("C2") == "frames/sec for 40-frame 512x512 SD1.5 50-step edit"
    c = bench.CONFIGS
    assert (c["C2"]["n_frames"], c["C2"]["batch"], c["C2"]["latent"], c["C2"]["mode"]) == (40, 8, 64, "pnp")
    assert (c["C3"]["n_frames"], c["C3"]["batch"]) == (80, 8)
    assert (c["C4"]["kind"], c["C4"]["latent"], c["C4"]["mode"], c["C4"]["n_steps"]) == ("sd21", 96, "sdedit", 44)
    assert [c[k]["n_frames"] // c[k]["batch"] for k in ("C5s4", "C5s8", "C5s16")] == [50, 25, 12]
    assert bench.unet_levels("sd15", 64) == ((4096, 320, 8, 5), (1024, 640, 8, 5), (256, 1280, 8, 5), (64, 1280, 8, 1))
    assert bench.unet_levels("sd21", 96)[0] == (9216, 320, 5, 5)
    threads, probe = bench.pick_cpu_threads(3)
    assert threads == 3 and probe == {}


def test_graph_event_aggregation_weights_variants_by_their_replays():
    class Ev:
        def __init__(self, t):
            self.t = t

        def elapsed_time(self, other):
            return other.t - self.t
    a = {"replays": 5, "mark": 2, "events": [("tf_ext_attn", 10.0, Ev(0.0), Ev(2.0)), ("tf_nn_field", 4.0, Ev(2.0), Ev(2.5))]}
    b = {"replays": 1, "events": [("tf_ext_attn", 10.0, Ev(0.0), Ev(1.0))]}
    c = {"replays": 3, "mark": 3, "events": [("tf_ext_attn", 10.0, Ev(0.0), Ev(9.0))]}      # not replayed since the mark
    d = {"replays": 2, "events": None}                                                         # captured without timing
    agg, steps = TokenFlowEditor.aggregate_graph_events([a, b, c, d], since_mark=True)
    assert steps == 4
    assert agg["tf_ext_attn"] == {"launches": 4, "ms": 3 * 2.0 + 1.0, "work": 40.0}
    assert agg["tf_nn_field"] == {"launches": 3, "ms": 1.5, "work": 12.0}
    agg_all, steps_all = TokenFlowEditor.aggregate_graph_events([a, b, c, d])
    assert steps_all == 9 and agg_all["tf_ext_attn"]["launches"] == 9
