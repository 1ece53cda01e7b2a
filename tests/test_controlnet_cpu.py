"""CPU tier: the ControlNet (tokenflow_b200/controlnet.py), the UNet's residual inputs, and the ControlNet through the
inversion stage and the editor.

* state-dict names and shapes are diffusers' ControlNetModel at the sd-controlnet-canny configuration;
* `from_unet`: the features before the zero convolutions are the UNet's own skips bit for bit, the residuals are zero,
  and the UNet with them equals the UNet without;
* non-zero residuals land where diffusers adds them (a restatement of its forward);
* the TokenFlow hooks leave the ControlNet's attention alone;
* `LatentInverter` with a ControlNet equals the reference's `controlnet_pred` loop (oracle/controlnet_inversion.py), and rank
  shares read their own frames' conditioning;
* the editor: a `from_unet` ControlNet changes nothing, the fused step equals the reference's per-batch schedule with
  per-frame conditioning, and two gloo ranks equal one.
"""
import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

from oracle import canny as oc
from oracle import gen_canny_golden as gg
from oracle import controlnet_inversion as CI
from oracle import inversion as OI
from tokenflow_b200 import preprocess
from tokenflow_b200 import sd_unet
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.controlnet import ControlNetModel, build_controlnet
from tokenflow_b200.scheduler import DDIMScheduler


def edge_cond(n, h, w, seed=5):
    """[n, 3, h, w] fp32 0/1 conditioning from the Canny edges of seeded frames."""
    rng = np.random.default_rng(seed)
    frames = np.stack([gg.make_frame("smooth", h, w, rng) for _ in range(n)])
    return oc.canny_cond(oc.canny_frames(frames, 100, 200)).float().contiguous()


def randomise(net: ControlNetModel, seed=7, scale=0.05):
    """Non-zero zero convolutions, as trained weights have."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in [net.controlnet_cond_embedding.conv_out, *net.controlnet_down_blocks, net.controlnet_mid_block]:
            for p in m.parameters():
                p.copy_(torch.randn(p.shape, generator=g) * scale)
    return net


# ----------------------------------------------------------------------------------------------------------------
# the model
# ----------------------------------------------------------------------------------------------------------------
def test_state_dict_names_and_shapes_are_diffusers():
    unet = sd_unet.build_unet("sd15")
    cn = ControlNetModel.from_unet(unet)
    sd, usd = cn.state_dict(), unet.state_dict()
    shared = ("conv_in.", "time_embedding.", "down_blocks.", "mid_block.")
    for k, v in sd.items():
        if k.startswith(shared):
            assert k in usd and usd[k].shape == v.shape, k
    assert {k for k in usd if k.startswith(shared)} == {k for k in sd if k.startswith(shared)}
    emb = {"conv_in": (16, 3), "blocks.0": (16, 16), "blocks.1": (32, 16), "blocks.2": (32, 32), "blocks.3": (96, 32),
           "blocks.4": (96, 96), "blocks.5": (256, 96), "conv_out": (320, 256)}
    for name, (co, ci) in emb.items():
        assert sd[f"controlnet_cond_embedding.{name}.weight"].shape == (co, ci, 3, 3)
        assert sd[f"controlnet_cond_embedding.{name}.bias"].shape == (co,)
    assert [cn.controlnet_cond_embedding.blocks[i].stride for i in range(6)] == [(1, 1), (2, 2)] * 3
    widths = [320] * 4 + [640] * 3 + [1280] * 5
    for i, c in enumerate(widths):
        assert sd[f"controlnet_down_blocks.{i}.weight"].shape == (c, c, 1, 1)
        assert sd[f"controlnet_down_blocks.{i}.bias"].shape == (c,)
    assert f"controlnet_down_blocks.{len(widths)}.weight" not in sd
    assert sd["controlnet_mid_block.weight"].shape == (1280, 1280, 1, 1)
    other = [k for k in sd if not k.startswith(shared + ("controlnet_cond_embedding.", "controlnet_down_blocks.",
                                                         "controlnet_mid_block."))]
    assert other == []
    fresh = ControlNetModel()
    fresh.load_state_dict(sd, strict=True)


def _unet_skips(unet, x, t, ctx):
    """The UNet's skips and mid-block output, restated from its forward."""
    t = t.reshape(-1).expand(x.shape[0])
    emb = unet.time_embedding(sd_unet.sinusoidal_timestep_embedding(t, unet.config.block_out_channels[0]))
    h = unet.conv_in(x)
    skips = [h]
    for blk in unet.down_blocks:
        h, outs = blk(h, emb, ctx)
        skips.extend(outs)
    return skips, unet.mid_block(h, emb, ctx), emb


@torch.no_grad()
def test_from_unet_copies_the_encoder_and_gives_zero_residuals():
    unet = sd_unet.build_unet("tiny", seed=1)
    cn = ControlNetModel.from_unet(unet)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(3, 4, 16, 16, generator=g)
    ctx = torch.randn(3, 7, unet.config.cross_attention_dim, generator=g)
    t = torch.tensor(401)
    feats = []
    hooks = [m.register_forward_pre_hook(lambda m, a: feats.append(a[0].clone()))
             for m in [*cn.controlnet_down_blocks, cn.controlnet_mid_block]]
    down, mid = cn(x, t, encoder_hidden_states=ctx, controlnet_cond=edge_cond(3, 128, 128))
    for h in hooks:
        h.remove()
    skips, mid_feat, _ = _unet_skips(unet, x, t, ctx)
    assert len(down) == len(skips) == 12 and len(feats) == 13
    for a, b in zip(feats, skips + [mid_feat]):
        assert torch.equal(a, b)
    assert all(not d.any() for d in down) and not mid.any()
    plain = unet(x, t, encoder_hidden_states=ctx)["sample"]
    with_res = unet(x, t, encoder_hidden_states=ctx, down_block_additional_residuals=down,
                    mid_block_additional_residual=mid)["sample"]
    assert torch.equal(plain, with_res)


def _restated_unet(unet, x, t, ctx, down_res, mid_res):
    """diffusers' UNet2DConditionModel.forward with ControlNet residuals: each skip plus its residual, the mid-block
    output plus the mid residual (unet_2d_condition.py, `is_controlnet`)."""
    skips, h, emb = _unet_skips(unet, x, t, ctx)
    skips = [s + r for s, r in zip(skips, down_res)]
    h = h + mid_res
    for blk in unet.up_blocks:
        h = blk(h, skips, emb, ctx)
    return unet.conv_out(F.silu(unet.conv_norm_out(h)))


@torch.no_grad()
@pytest.mark.parametrize("scale", [1.0, 0.6])
def test_residuals_are_added_where_diffusers_adds_them(scale):
    unet = sd_unet.build_unet("tiny", seed=1)
    cn = build_controlnet("tiny", seed=3)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 4, 16, 16, generator=g)
    ctx = torch.randn(2, 7, unet.config.cross_attention_dim, generator=g)
    t = torch.tensor(601)
    down, mid = cn(x, t, encoder_hidden_states=ctx, controlnet_cond=edge_cond(2, 128, 128), conditioning_scale=scale)
    assert all(d.abs().max() > 0 for d in down) and mid.abs().max() > 0
    if scale != 1.0:
        d1, m1 = cn(x, t, encoder_hidden_states=ctx, controlnet_cond=edge_cond(2, 128, 128))
        assert all(torch.equal(a, b * scale) for a, b in zip(down, d1)) and torch.equal(mid, m1 * scale)
    got = unet(x, t, encoder_hidden_states=ctx, down_block_additional_residuals=down,
               mid_block_additional_residual=mid, cross_attention_kwargs={}, return_dict=False)[0]
    want = _restated_unet(unet, x, t, ctx, down, mid)
    assert torch.equal(got, want)
    assert not torch.equal(got, unet(x, t, encoder_hidden_states=ctx)["sample"])
    only_mid = unet(x, t, encoder_hidden_states=ctx, mid_block_additional_residual=mid)["sample"]
    assert torch.equal(only_mid, _restated_unet(unet, x, t, ctx, [0] * 12, mid))
    with pytest.raises(ValueError, match="residuals"):
        unet(x, t, encoder_hidden_states=ctx, down_block_additional_residuals=down[:-1])


# ----------------------------------------------------------------------------------------------------------------
# inversion
# ----------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def test_inversion_with_controlnet_equals_the_reference_loop():
    unet = sd_unet.build_unet("tiny", seed=1)
    cn = build_controlnet("tiny", seed=3)
    g = torch.Generator().manual_seed(6)
    n = 5
    x0 = torch.randn(n, 4, 16, 16, generator=g)
    cond = torch.randn(1, 7, unet.config.cross_attention_dim, generator=g)
    ccond = edge_cond(n, 128, 128)
    inv = preprocess.LatentInverter(unet, DDIMScheduler(), 6, controlnet=cn, controlnet_cond=ccond)
    xT = inv.ddim_inversion(cond, x0.clone(), None, batch_size=2)
    rec = inv.ddim_sample(xT.clone(), cond, batch_size=2)
    want_T, _ = CI.ddim_inversion(unet, cn, inv.scheduler, cond, ccond, x0.clone(), 2)
    want_rec = CI.ddim_sample(unet, cn, inv.scheduler, want_T.clone(), cond, ccond, 2)
    assert torch.equal(xT, want_T) and torch.equal(rec, want_rec)
    plain_T, _ = OI.ddim_inversion(unet, inv.scheduler, cond, x0.clone(), 2)
    assert not torch.equal(xT, plain_T)
    # each rank inverts its share (frames 0-2, 3-4) with its own frames' conditioning
    for rank, (lo, hi) in enumerate([(0, 3), (3, 5)]):
        inv_r = preprocess.LatentInverter(unet, DDIMScheduler(), 6, world_size=2, rank=rank, controlnet=cn,
                                          controlnet_cond=ccond)
        inv_r._gathered = lambda x_local, n_: x_local
        got = inv_r.ddim_inversion(cond, x0.clone(), None, batch_size=2, save_latents=False)
        want, _ = CI.ddim_inversion(unet, cn, inv.scheduler, cond, ccond[lo:hi], x0[lo:hi].clone(), 2)
        assert torch.equal(got, want), rank
    with pytest.raises(ValueError):
        preprocess.LatentInverter(unet, DDIMScheduler(), 6, controlnet=cn)


# ----------------------------------------------------------------------------------------------------------------
# editor
# ----------------------------------------------------------------------------------------------------------------
def _edit(world, rank, mode, steps, fused, controlnet="random", scale=1.0, return_editor=False):
    from oracle.oracle_ops import OracleOps
    from tokenflow_b200.editor import TokenFlowEditor, synthetic_inputs
    tfu._install_ops_for_testing(OracleOps())
    unet = sd_unet.build_unet("tiny", seed=1)
    cn = None
    if controlnet == "random":
        cn = randomise(build_controlnet("tiny", seed=3))
    elif controlnet == "from_unet":
        cn = ControlNetModel.from_unet(unet)
    cfg = {"n_frames": 8, "batch_size": 2, "n_timesteps": steps, "guidance_scale": 7.5, "mode": mode,
           "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "start": 0.9, "fused_pass": fused,
           "controlnet_conditioning_scale": scale}
    x, text, pnp, src = synthetic_inputs(8, 16, unet.config.cross_attention_dim, steps, seed=1, ctx_len=7)
    ed = TokenFlowEditor(unet, DDIMScheduler(), tfu, cfg, text, pnp, source_latents=lambda t: src[t],
                         world_size=world, rank=rank, controlnet=cn,
                         controlnet_cond=edge_cond(8, 128, 128) if cn is not None else None)
    ed.init_method()
    torch.manual_seed(1)
    out = ed.sample_loop(x)
    return (out, ed.keyframe_log, ed) if return_editor else (out, ed.keyframe_log)


@pytest.mark.parametrize("mode,steps", [("pnp", 2), ("sdedit", 10)])
@pytest.mark.parametrize("fused", [False, True])
def test_from_unet_controlnet_changes_nothing(mode, steps, fused):
    plain, kf_plain = _edit(1, 0, mode, steps, fused, controlnet=None)
    got, kf = _edit(1, 0, mode, steps, fused, controlnet="from_unet")
    assert kf == kf_plain and torch.equal(got, plain)


@pytest.mark.parametrize("mode,steps", [("pnp", 2), ("sdedit", 10)])
def test_fused_equals_the_reference_schedule(mode, steps):
    ref, kf_ref = _edit(1, 0, mode, steps, fused=False)
    got, kf = _edit(1, 0, mode, steps, fused=True)
    plain, _ = _edit(1, 0, mode, steps, fused=True, controlnet=None)
    assert kf == kf_ref
    assert torch.allclose(got, ref, atol=2e-4, rtol=1e-4), (got - ref).abs().max().item()
    assert (got - plain).abs().max() > 1e-2                     # the conditioning does act
    scaled, _ = _edit(1, 0, mode, steps, fused=True, scale=0.0)
    assert torch.allclose(scaled, plain, atol=2e-4, rtol=1e-4)  # scale 0: no residuals


def test_hooks_leave_the_controlnet_unpatched():
    _, _, ed = _edit(1, 0, "pnp", 2, fused=True, return_editor=True)
    cn = ed.controlnet
    assert "controlnet" not in dict(ed.named_children())
    blocks = [m for m in cn.modules() if type(m).__name__.startswith("BasicTransformerBlock")]
    assert blocks and all(type(m) is sd_unet.BasicTransformerBlock for m in blocks)
    for m in cn.modules():
        assert "forward" not in m.__dict__, type(m).__name__
        assert not [a for a in m.__dict__ if a.startswith("_tf_") or a in ("pivotal_pass", "batch_idx", "t",
                                                                             "injection_schedule")], type(m).__name__
    unet_blocks = [m for m in ed.unet.modules() if type(m).__name__.startswith("BasicTransformerBlock")]
    assert all(type(m) is not sd_unet.BasicTransformerBlock for m in unet_blocks)    # the UNet's are patched


def _worker(rank, world, rdzv, mode, steps, q):
    torch.set_num_threads(2)
    dist.init_process_group("gloo", init_method=f"file://{rdzv}", rank=rank, world_size=world)
    try:
        out, kf = _edit(world, rank, mode, steps, fused=True)
        q.put((rank, out.numpy().tolist(), kf))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("mode,steps", [("pnp", 2), ("sdedit", 10)])
def test_two_rank_edit_equals_single_process(mode, steps):
    import os
    import tempfile
    want, kf_want = _edit(1, 0, mode, steps, fused=False)
    fd, rdzv = tempfile.mkstemp(prefix="tf_b200_cn_rdzv_")
    os.close(fd)
    os.unlink(rdzv)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
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
