"""GPU tier (-m gpu): the inversion stage on the H100 — tf_ddim against the reference's expression, the graphed path
against its eager form and against the reference's loop (oracle/inversion.py), the in-memory hand-off to the editor,
and two ranks against one."""
import os
import socket
import subprocess
import sys

import pytest
import torch

from oracle import inversion as OI
from tokenflow_b200 import sd_unet
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.editor import TokenFlowEditor
from tokenflow_b200.preprocess import LatentInverter, inversion_coef_tables
from tokenflow_b200.scheduler import DDIMScheduler

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ops():
    from tokenflow_b200.ops import CudaOps
    tfu._install_ops_for_testing(None)
    return CudaOps()


@pytest.fixture(scope="module")
def sd15():
    unet = sd_unet.build_unet("sd15", seed=1, device="cuda", dtype=torch.float16, init_on_device=True)
    return unet.to(memory_format=torch.channels_last)


def _inputs(n, latent, ctx, seed=3):
    g = torch.Generator().manual_seed(seed)
    x0 = torch.randn(n, 4, latent, latent, generator=g).half().cuda()
    cond = torch.randn(1, 77, ctx, generator=g).half().cuda()
    return x0, cond


# ------------------------------------------------------------------------------------------------
# 1. tf_ddim == the reference's eager expression with 0-dim fp32 CPU alphas (preprocess.py:224-225, :259-260)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("direction", ["inversion", "reconstruction"])
@pytest.mark.parametrize("case", ["out_of_place", "in_place", "tail"])
def test_ddim_equals_the_reference_expression(ops, direction, case):
    sch = DDIMScheduler()
    sch.set_timesteps(500)
    inv, rec = inversion_coef_tables(sch)
    table = (inv if direction == "inversion" else rec).cuda()
    shape = (3, 4, 7, 5) if case == "tail" else (5, 4, 64, 64)          # 420 elements: n % 8 == 4
    g = torch.Generator().manual_seed(len(case) * 7 + len(direction))
    for i in (0, 1, 97, 250, 498, 499):
        x = (torch.randn(shape, generator=g) * 2).half().cuda()
        eps = torch.randn(shape, generator=g).half().cuda()
        if case == "out_of_place":
            eps = eps.contiguous(memory_format=torch.channels_last)
        want = OI.ddim_expression(x, eps, direction, OI.step_alphas(sch, direction, i))
        x_before = x.clone()
        if case == "in_place":
            got = ops.ddim(eps, x, table[i], out=x)
            assert got.data_ptr() == x.data_ptr()
        else:
            got = ops.ddim(eps, x, table[i])
            assert torch.equal(x, x_before)
        assert got.dtype == torch.float16 and got.shape == x.shape
        assert torch.equal(got, want), (i, (got.float() - want.float()).abs().max().item())


# ------------------------------------------------------------------------------------------------
# 2. graph replay == the same device path run eagerly
# ------------------------------------------------------------------------------------------------
def test_graph_replay_equals_eager(ops, sd15):
    x0, cond = _inputs(4, 64, sd15.config.cross_attention_dim)
    res = {}
    for graphed in (True, False):
        inv = LatentInverter(sd15, DDIMScheduler(), 10)
        inv._use_graph = graphed
        xT = inv.ddim_inversion(cond, x0, None, batch_size=2)
        rec = inv.ddim_sample(xT, cond, batch_size=2)
        res[graphed] = (xT, rec, inv.saved_latents())
    assert torch.isfinite(res[True][1]).all()
    assert torch.equal(res[True][0], res[False][0]) and torch.equal(res[True][1], res[False][1])
    assert sorted(res[True][2]) == sorted(res[False][2])
    for t in res[True][2]:
        assert torch.equal(res[True][2][t], res[False][2][t]), t


# ------------------------------------------------------------------------------------------------
# 3. the whole inversion against the reference's loop
# ------------------------------------------------------------------------------------------------
def test_sdpa_route_equals_the_reference_loop(ops, sd15):
    x0, cond = _inputs(4, 64, sd15.config.cross_attention_dim)
    inv = LatentInverter(sd15, DDIMScheduler(), 10)
    ts_up = [int(t) for t in reversed(inv.scheduler.timesteps.tolist())]
    keep = ts_up[2::3]
    xT = inv.ddim_inversion(cond, x0, None, batch_size=2, timesteps_to_save=keep)
    rec = inv.ddim_sample(xT, cond, batch_size=2)
    want_T, want_saved = OI.ddim_inversion(sd15, inv.scheduler, cond, x0.clone(), 2, keep)
    want_rec = OI.ddim_sample(sd15, inv.scheduler, want_T.clone(), cond, 2)
    assert sorted(inv.saved_latents()) == sorted(want_saved)
    for t, v in want_saved.items():
        assert torch.equal(inv.saved_latents()[t], v), t
    assert torch.equal(xT, want_T)
    assert torch.equal(rec, want_rec), (rec.float() - want_rec.float()).abs().max().item()


# ------------------------------------------------------------------------------------------------
# 4. hand-off: files and saved_latents() feed the same edit
# ------------------------------------------------------------------------------------------------
def test_in_memory_hand_off_equals_the_files(ops, tmp_path):
    steps, n = 4, 4
    unet = sd_unet.build_unet("tiny", seed=1, device="cuda", dtype=torch.float16).to(memory_format=torch.channels_last)
    ctx = unet.config.cross_attention_dim
    g = torch.Generator().manual_seed(11)
    x0 = torch.randn(n, 4, 16, 16, generator=g).half().cuda()
    pnp = torch.randn(1, 7, ctx, generator=g).half().cuda()
    text = torch.randn(2, 7, ctx, generator=g).half().cuda()
    inv = LatentInverter(unet, DDIMScheduler(), steps)
    noisy = inv.ddim_inversion(pnp, x0, str(tmp_path), batch_size=2)
    saved = inv.saved_latents()
    lat = str(tmp_path / "latents")
    assert sorted(os.listdir(lat)) == sorted(f"noisy_latents_{t}.pt" for t in saved)
    for t, v in saved.items():
        assert torch.equal(tfu.load_source_latents_t(t, lat), v)
    cfg = {"n_frames": n, "batch_size": 2, "n_timesteps": steps, "guidance_scale": 7.5, "mode": "pnp",
           "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "fused_pass": True, "cuda_graph": True, "keyframe_seed": 1,
           "latents_path": lat}
    outs = []
    for source in (None, saved.__getitem__):
        edit_unet = sd_unet.build_unet("tiny", seed=1, device="cuda", dtype=torch.float16)
        ed = TokenFlowEditor(edit_unet.to(memory_format=torch.channels_last), DDIMScheduler(), tfu, cfg, text, pnp,
                             source_latents=source)
        ed.init_method()
        outs.append((ed.sample_loop(noisy.clone()), ed.keyframe_log))
    assert outs[0][1] == outs[1][1]
    assert torch.isfinite(outs[0][0]).all() and torch.equal(outs[0][0], outs[1][0])


# ------------------------------------------------------------------------------------------------
# 5. two ranks over tf_allgather == one rank  (skipped with fewer than two GPUs)
# ------------------------------------------------------------------------------------------------
_WORKER = r"""
import os, sys, json, torch
sys.path.insert(0, {repo!r})
import torch.distributed as dist
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
from tokenflow_b200 import sd_unet
from tokenflow_b200.preprocess import LatentInverter
from tokenflow_b200.scheduler import DDIMScheduler
from tokenflow_b200.ops import Communicator
unet = sd_unet.build_unet("tiny", seed=1, device="cuda", dtype=torch.float16).to(memory_format=torch.channels_last)
g = torch.Generator().manual_seed(2)
x0 = torch.randn(5, 4, 16, 16, generator=g).half().cuda()
cond = torch.randn(1, 7, unet.config.cross_attention_dim, generator=g).half().cuda()
def run(world, rank, comm):
    inv = LatentInverter(unet, DDIMScheduler(), 6, world_size=world, rank=rank)
    if comm is not None:
        inv.attach_communicator(comm)
    xT = inv.ddim_inversion(cond, x0, None, batch_size=2)
    return xT.float(), inv.ddim_sample(xT, cond, batch_size=2).float(), {{t: v.float() for t, v in inv.saved_latents().items()}}
want = run(1, 0, None)
comm = Communicator(world, rank)
res = {{}}
for name, c in (("capi", comm), ("torch", None)):
    xT, rec, saved = run(world, rank, c)
    rel = lambda a, b: float((a - b).norm() / b.norm())
    res[name] = dict(xT=rel(xT, want[0]), rec=rel(rec, want[1]), saved=max(rel(saved[t], want[2][t]) for t in want[2]),
                     same_keys=sorted(saved) == sorted(want[2]), finite=bool(torch.isfinite(rec).all()))
comm.destroy()
if rank == 0:
    print("RESULT " + json.dumps(res), flush=True)
dist.destroy_process_group()
"""


def test_two_rank_inversion_equals_one_rank(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    script = tmp_path / "worker.py"
    script.write_text(_WORKER.format(repo=REPO))
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), str(script)],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    import json
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1]
    res = json.loads(line[len("RESULT "):])
    for name, v in res.items():
        assert v["same_keys"] and v["finite"], (name, v)
        for key in ("xT", "rec", "saved"):
            assert v[key] < 2e-2, (name, key, v)                   # the tolerance of the two-rank edit test
