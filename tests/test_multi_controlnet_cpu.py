"""CPU tier: several ControlNets at once and conditioning sources other than Canny.

* `MultiControlNetModel`'s residuals, and the UNet output they give, equal diffusers' summation restated in
  oracle/multi_controlnet.py, for 2 and 3 nets, a float scale and a list of scales;
* a second net made by `from_unet` (zero convolutions) changes neither the inversion nor the edit (PnP and SDEdit,
  fused and unfused); a list of one ControlNet is today's single-net path;
* `LatentInverter` with two nets equals the reference's ControlNet loops with the summed residuals;
* `control_cond`: "frames" and maps take every byte value to `np.float32(v) / 255` in fp16; maps are resized to the
  frames' size, also for non-square frames and maps of another aspect;
* refusals: too few maps, control or scale counts that do not match the nets, conditioning_channels != 3;
* the command line: `--controlnet_dir` / `--control` pairing, the counts refused before a model loads, and the
  `controlnets` record of `edit`'s config.yaml;
* a two-rank gloo edit with two nets equals the single-process edit (to the CPU kernels' rounding of other batch
  shapes).
"""
import os
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import yaml

from oracle import multi_controlnet as MC
from oracle.oracle_ops import OracleOps
from tokenflow_b200 import pipeline, preprocess, run, sd_unet
from tokenflow_b200 import synthetic_checkpoint as fx
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.controlnet import (ControlNetConfig, ControlNetModel, MultiControlNetModel, build_controlnet,
                                       conditioning_scale_for)
from tokenflow_b200.editor import TokenFlowEditor, synthetic_inputs
from tokenflow_b200.scheduler import DDIMScheduler

from test_controlnet_cpu import edge_cond, randomise


def _nets(k):
    return [randomise(build_controlnet("tiny", seed=3 + i), seed=7 + i) for i in range(k)]


def _conds(k, n, h=128, w=128):
    return torch.cat([edge_cond(n, h, w, seed=5 + i) for i in range(k)], dim=1)


# ----------------------------------------------------------------------------------------------------------------
# the sum
# ----------------------------------------------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize("k,scale", [(2, 1.0), (2, 0.7), (2, [0.6, 1.3]), (3, 0.8), (3, [1.0, 0.5, 0.25])])
def test_residuals_equal_diffusers_summation(k, scale):
    unet = sd_unet.build_unet("tiny", seed=1)
    nets = _nets(k)
    multi = MultiControlNetModel(nets)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 4, 16, 16, generator=g)
    ctx = torch.randn(2, 7, unet.config.cross_attention_dim, generator=g)
    t = torch.tensor(601)
    cond = _conds(k, 2)
    down, mid = multi(x, t, ctx, cond, scale)
    scales = scale if isinstance(scale, list) else [scale] * k
    want_down, want_mid = MC.MultiControlNet(nets, scales)(x, t, encoder_hidden_states=ctx, controlnet_cond=cond)
    assert len(down) == len(want_down) == 12
    assert all(torch.equal(a, b) for a, b in zip(down, want_down)) and torch.equal(mid, want_mid)
    one, _ = nets[0](x, t, ctx, cond[:, :3], scales[0])
    assert not torch.equal(down[0], one[0])                    # the other nets do act
    got = unet(x, t, encoder_hidden_states=ctx, down_block_additional_residuals=down,
               mid_block_additional_residual=mid)["sample"]
    want = MC.controlnet_pred(nets, scales, unet, x, t, ctx, cond)
    assert torch.equal(got, want)


@torch.no_grad()
def test_fp16_sums_round_each_add_in_net_order():
    nets = [n.half() for n in _nets(3)]
    g = torch.Generator().manual_seed(4)
    x = torch.randn(1, 4, 16, 16, generator=g).half()
    ctx = torch.randn(1, 7, 32, generator=g).half()
    cond = _conds(3, 1).half()
    t = torch.tensor(401)
    try:
        down, mid = MultiControlNetModel(nets)(x, t, ctx, cond, [0.5, 1.0, 2.0])
    except RuntimeError as e:                                  # no fp16 convolution on this CPU build
        pytest.skip(str(e))
    parts = [net(x, t, ctx, cond[:, 3 * i:3 * i + 3], s) for i, (net, s) in enumerate(zip(nets, [0.5, 1.0, 2.0]))]
    assert down[0].dtype == torch.float16
    assert torch.equal(mid, (parts[0][1] + parts[1][1]) + parts[2][1])


def test_a_list_of_one_is_the_single_net_path():
    net = _nets(1)[0]
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 4, 16, 16, generator=g)
    ctx = torch.randn(2, 7, 32, generator=g)
    cond = _conds(1, 2)
    with torch.no_grad():
        d1, m1 = net(x, torch.tensor(1), ctx, cond, 0.8)
        d2, m2 = MultiControlNetModel([net])(x, torch.tensor(1), ctx, cond, [0.8])
    assert all(torch.equal(a, b) for a, b in zip(d1, d2)) and torch.equal(m1, m2)
    assert conditioning_scale_for(net, [0.8]) == 0.8 and conditioning_scale_for(net, 2) == 2.0
    assert conditioning_scale_for(MultiControlNetModel(_nets(2)), 0.5) == [0.5, 0.5]
    a, _ = _edit("pnp", 2, True, nets="one", scale=0.8)
    b, _ = _edit("pnp", 2, True, nets="one", scale=[0.8])
    assert torch.equal(a, b)


# ----------------------------------------------------------------------------------------------------------------
# inversion and editor
# ----------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def test_inversion_with_two_nets_equals_the_reference_loop_and_a_zero_net_changes_nothing():
    unet = sd_unet.build_unet("tiny", seed=1)
    nets = _nets(2)
    g = torch.Generator().manual_seed(6)
    n = 5
    x0 = torch.randn(n, 4, 16, 16, generator=g)
    cond = torch.randn(1, 7, unet.config.cross_attention_dim, generator=g)
    ccond = _conds(2, n)
    inv = preprocess.LatentInverter(unet, DDIMScheduler(), 6, controlnet=MultiControlNetModel(nets),
                                    controlnet_cond=ccond, controlnet_conditioning_scale=[0.7, 1.2])
    xT = inv.ddim_inversion(cond, x0.clone(), None, batch_size=2)
    rec = inv.ddim_sample(xT.clone(), cond, batch_size=2)
    want_T, _ = MC.ddim_inversion(unet, nets, [0.7, 1.2], inv.scheduler, cond, ccond, x0.clone(), 2)
    want_rec = MC.ddim_sample(unet, nets, [0.7, 1.2], inv.scheduler, want_T.clone(), cond, ccond, 2)
    assert torch.equal(xT, want_T) and torch.equal(rec, want_rec)
    # a from_unet second net: the single-net inversion, bit for bit
    single = preprocess.LatentInverter(unet, DDIMScheduler(), 6, controlnet=nets[0], controlnet_cond=ccond[:, :3],
                                       controlnet_conditioning_scale=0.7)
    zero = preprocess.LatentInverter(unet, DDIMScheduler(), 6,
                                     controlnet=MultiControlNetModel([nets[0], ControlNetModel.from_unet(unet)]),
                                     controlnet_cond=ccond, controlnet_conditioning_scale=[0.7, 1.2])
    assert torch.equal(single.ddim_inversion(cond, x0.clone(), None, batch_size=2),
                       zero.ddim_inversion(cond, x0.clone(), None, batch_size=2))
    with pytest.raises(ValueError, match="3 ControlNet conditioning scales for 2 ControlNets"):
        preprocess.LatentInverter(unet, DDIMScheduler(), 6, controlnet=MultiControlNetModel(nets),
                                  controlnet_cond=ccond, controlnet_conditioning_scale=[1, 1, 1])


def _edit(mode, steps, fused, nets="two", scale=1.0, world=1, rank=0):
    tfu._install_ops_for_testing(OracleOps())
    unet = sd_unet.build_unet("tiny", seed=1)
    first = randomise(build_controlnet("tiny", seed=3))
    cn = {"one": first, "two": MultiControlNetModel([first, randomise(build_controlnet("tiny", seed=4), seed=8)]),
          "zero": MultiControlNetModel([first, ControlNetModel.from_unet(unet)])}[nets]
    cfg = {"n_frames": 8, "batch_size": 2, "n_timesteps": steps, "guidance_scale": 7.5, "mode": mode,
           "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "start": 0.9, "fused_pass": fused,
           "controlnet_conditioning_scale": scale}
    x, text, pnp, src = synthetic_inputs(8, 16, unet.config.cross_attention_dim, steps, seed=1, ctx_len=7)
    ccond = _conds(1 if nets == "one" else 2, 8)
    ed = TokenFlowEditor(unet, DDIMScheduler(), tfu, cfg, text, pnp, source_latents=lambda t: src[t],
                         world_size=world, rank=rank, controlnet=cn, controlnet_cond=ccond)
    ed.init_method()
    torch.manual_seed(1)
    return ed.sample_loop(x), ed.keyframe_log


@pytest.mark.parametrize("mode,steps", [("pnp", 2), ("sdedit", 10)])
@pytest.mark.parametrize("fused", [False, True])
def test_a_zero_second_net_changes_nothing(mode, steps, fused):
    one, kf_one = _edit(mode, steps, fused, nets="one", scale=0.8)
    zero, kf = _edit(mode, steps, fused, nets="zero", scale=[0.8, 1.5])
    assert kf == kf_one and torch.equal(zero, one)
    two, _ = _edit(mode, steps, fused, nets="two", scale=[0.8, 1.5])
    assert (two - one).abs().max() > 1e-3


def _worker(rank, world, rdzv, q):
    torch.set_num_threads(2)
    dist.init_process_group("gloo", init_method=f"file://{rdzv}", rank=rank, world_size=world)
    try:
        out, kf = _edit("pnp", 2, True, scale=[0.8, 1.5], world=world, rank=rank)
        q.put((rank, out.numpy().tolist(), kf))
    finally:
        dist.destroy_process_group()


def test_two_rank_edit_with_two_nets_equals_single_process():
    want, kf_want = _edit("pnp", 2, True, scale=[0.8, 1.5])
    fd, rdzv = tempfile.mkstemp(prefix="tf_b200_mcn_rdzv_")
    os.close(fd)
    os.unlink(rdzv)
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, rdzv, q)) for r in range(2)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, out, kf in results:
        assert kf == kf_want
        # a rank's UNet calls have other batch shapes, so the CPU kernels may round differently (as in
        # test_controlnet_cpu.py's two-rank test)
        assert torch.allclose(torch.tensor(out), want, atol=2e-4, rtol=1e-4), f"rank {rank}"


# ----------------------------------------------------------------------------------------------------------------
# conditioning sources
# ----------------------------------------------------------------------------------------------------------------
def test_frames_and_maps_take_every_byte_to_float32_over_255():
    v = np.arange(256, dtype=np.uint8)
    frames = torch.from_numpy(np.stack([np.roll(v, 3 * i) for i in range(3)], -1).reshape(1, 16, 16, 3))
    want = torch.from_numpy(np.float32(frames.numpy()) / 255).half().permute(0, 3, 1, 2)
    got = preprocess.control_cond(frames, ["frames", frames.clone()])
    assert got.dtype == torch.float16 and got.shape == (1, 6, 16, 16)
    assert torch.equal(got[:, :3], want) and torch.equal(got[:, 3:], want)
    assert torch.equal(preprocess.control_cond(frames, ["canny"]), preprocess.canny_cond(frames))


@pytest.mark.parametrize("frames_hw,maps_hw", [((64, 64), (64, 64)), ((48, 80), (96, 160)), ((48, 80), (100, 60)),
                                               ((72, 40), (30, 30))])
def test_maps_are_resized_to_the_frames_size(frames_hw, maps_hw):
    g = torch.Generator().manual_seed(0)
    frames = torch.randint(0, 256, (3, *frames_hw, 3), generator=g, dtype=torch.uint8)
    maps = torch.randint(0, 256, (5, *maps_hw, 3), generator=g, dtype=torch.uint8)
    got = preprocess.control_cond(frames, ["canny", maps])
    resized = preprocess.resize_frames(maps[:3], frames_hw)
    want = torch.from_numpy(np.float32(resized.numpy()) / 255).half().permute(0, 3, 1, 2)
    assert got.shape == (3, 6, *frames_hw)
    assert torch.equal(got[:, 3:], want) and torch.equal(got[:, :3], preprocess.canny_cond(frames))


def test_refusals_name_the_counts():
    frames = torch.zeros(4, 16, 16, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="3 control maps for 4 frames"):
        preprocess.control_cond(frames, [torch.zeros(3, 16, 16, 3, dtype=torch.uint8)])
    with pytest.raises(ValueError, match="'depth'"):
        preprocess.control_cond(frames, ["depth"])
    unet = sd_unet.build_unet("tiny", seed=1)
    nets = MultiControlNetModel(_nets(2))
    parts = pipeline.Parts(unet=unet, vae=None, scheduler=None, tokenizer=None, text_encoder=None, controlnet=nets)
    with pytest.raises(ValueError, match="1 controls for 2 ControlNets"):
        pipeline.conditioning(parts, frames, ["frames"])
    with pytest.raises(ValueError, match="3 ControlNet conditioning scales for 2 ControlNets"):
        nets(torch.zeros(1, 4, 2, 2), torch.tensor(1), None, torch.zeros(1, 6, 16, 16), [1.0, 1.0, 1.0])
    with pytest.raises(ValueError, match="1 ControlNet conditioning scales for 2 ControlNets"):
        TokenFlowEditor(unet, DDIMScheduler(), tfu, {"n_timesteps": 2, "controlnet_conditioning_scale": [1.0]},
                        torch.zeros(2, 7, 32), torch.zeros(1, 7, 32), controlnet=nets,
                        controlnet_cond=torch.zeros(4, 6, 16, 16))
    depth = ControlNetModel(ControlNetConfig(unet.config, conditioning_channels=1,
                                             conditioning_embedding_out_channels=(8, 8, 16, 16)))
    parts.controlnet = MultiControlNetModel([nets.nets[0], depth])
    with pytest.raises(ValueError, match="ControlNet 1 takes 1 conditioning channels"):
        pipeline.conditioning(parts, frames)
    parts.controlnet = None
    assert pipeline.conditioning(parts, frames) is None


# ----------------------------------------------------------------------------------------------------------------
# command line
# ----------------------------------------------------------------------------------------------------------------
def test_cli_refuses_counts_before_a_model_loads(tmp_path):
    missing = str(tmp_path / "no-model")
    base = ["preprocess", "--model_dir", missing, "--device", "cpu", "--data_path", str(tmp_path)]
    with pytest.raises(ValueError, match="1 --control for 2 --controlnet_dir"):
        run.main(base + ["--controlnet_dir", "a", "--controlnet_dir", "b", "--control", "frames"])
    with pytest.raises(ValueError, match="1 --control for 0 --controlnet_dir"):
        run.main(base + ["--control", "frames"])
    with pytest.raises(ValueError, match="3 controlnet_conditioning_scale values for 2 --controlnet_dir"):
        run.main(base + ["--controlnet_dir", "a", "--controlnet_dir", "b", "--controlnet_conditioning_scale", "1",
                         "2", "3"])
    cfg = tmp_path / "config.yaml"
    cfg.write_text(yaml.dump({"controlnet_conditioning_scale": [1.0, 0.5, 0.2]}))
    with pytest.raises(ValueError, match="3 controlnet_conditioning_scale values for 1 --controlnet_dir"):
        run.main(["edit", "--model_dir", missing, "--device", "cpu", "--config_path", str(cfg), "--controlnet_dir",
                  "a"])


def test_read_control_sources(tmp_path):
    assert run.read_control("canny", 4) == "canny" and run.read_control("frames", 4) == "frames"
    maps = torch.randint(0, 256, (3, 16, 24, 3), generator=torch.Generator().manual_seed(0), dtype=torch.uint8)
    run.write_frames(maps, str(tmp_path / "maps"))
    assert torch.equal(run.read_control(str(tmp_path / "maps"), 2), maps[:2])
    assert torch.equal(run.read_control(str(tmp_path / "maps"), 5), maps)        # control_cond refuses 3 for 5
    with pytest.raises(ValueError, match="not canny, frames"):
        run.read_control(str(tmp_path / "nothing"), 2)


N, H, W = 8, 64, 96
PNP = {"prompt": "a marble sculpture of a woman", "negative_prompt": "ugly blurry", "guidance_scale": 7.5,
       "n_timesteps": 5, "batch_size": 4, "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "seed": 1}


def test_cli_two_controlnets_record_and_equal_the_pipeline(tmp_path, monkeypatch):
    from tokenflow_b200.util import save_video
    tfu._install_ops_for_testing(OracleOps())
    model_dir, cn_dir = fx.write_checkpoint(str(tmp_path / "ckpt"), "tiny", controlnet=True)
    monkeypatch.chdir(tmp_path)
    g = torch.Generator().manual_seed(0)
    frames = (torch.nn.functional.interpolate(torch.rand(N, 3, H // 8, W // 8, generator=g), size=(H, W),
                                              mode="bilinear") * 255).round().to(torch.uint8)
    frames = frames.permute(0, 2, 3, 1).contiguous()
    run.write_frames(frames, "data/clip")
    maps = frames.flip(2).contiguous()[:, :40]                # another aspect than the frames
    run.write_frames(maps, "maps")
    argv = ["--model_dir", model_dir, "--device", "cpu", "--controlnet_dir", cn_dir, "--controlnet_dir", cn_dir,
            "--control", "frames", "--control", "maps"]
    run.main(["preprocess", *argv, "--data_path", "data/clip", "--H", str(H), "--W", str(W), "--save_dir", "latents",
              "--sd_version", "1.5", "--steps", "10", "--batch_size", "4", "--save_steps", "5", "--n_frames", str(N),
              "--controlnet_conditioning_scale", "0.7", "1.2"])
    cfg = {**PNP, "data_path": "data/clip", "latents_path": "latents", "sd_version": "1.5", "n_inversion_steps": 10,
           "n_frames": N, "output_path": "out", "controlnet_conditioning_scale": [0.7, 1.2]}
    with open("config.yaml", "w") as f:
        yaml.dump(cfg, f)
    run.main(["edit", *argv, "--config_path", "config.yaml"])
    record = yaml.safe_load(open("out/config.yaml"))
    assert record["controlnets"] == [{"path": cn_dir, "control": "frames", "scale": 0.7},
                                     {"path": cn_dir, "control": "maps", "scale": 1.2}]
    # the same calls in Python
    parts = pipeline.load_parts(model_dir, "cpu", torch.float32, [cn_dir, cn_dir])
    assert isinstance(parts.controlnet, MultiControlNetModel) and len(parts.controlnet.nets) == 2
    opt = {"H": H, "W": W, "steps": 10, "batch_size": 4, "save_steps": 5, "inversion_prompt": "a woman running",
           "controlnet_conditioning_scale": [0.7, 1.2]}
    torch.manual_seed(1)
    saved, _ = pipeline.preprocess(parts, frames, opt, controls=["frames", maps])
    got = run.read_latents(os.path.join("latents", "sd_1.5", "clip", "steps_10", f"nframes_{N}"))
    assert sorted(got) == sorted(saved) and all(torch.equal(got[t], saved[t]) for t in saved)
    torch.manual_seed(1)
    out = pipeline.edit(parts, frames, {**cfg, "inversion_prompt": "a woman running"}, saved,
                        controls=["frames", maps])
    assert torch.equal(run.read_frames("out/img_ode", N), out)
    # one --controlnet_dir stays a plain ControlNetModel
    assert type(pipeline.load_parts(model_dir, "cpu", torch.float32, [cn_dir]).controlnet) is ControlNetModel
