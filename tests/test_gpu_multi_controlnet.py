"""GPU tier (-m gpu): two ControlNets at once on the H100.

* editor: the CUDA-graphed fused step with a `MultiControlNetModel` of two nets against the eager fused step, bit for
  bit, in PnP (its three injection variants) and SDEdit, with and without `frames_per_pass` chunks, on the tiny UNet
  and on SD1.5 channels_last;
* inversion: the graphed step with two nets against the same device path run eagerly and against the reference's
  loop with diffusers' summed residuals (oracle/multi_controlnet.py);
* `control_cond` on CUDA frames equals the CPU path: maps from a device tensor, "frames", and "canny" beside them;
* the command line: a synthetic SD1.5 checkpoint, a ControlNet folder and a cldm `.pth`, `preprocess` and `edit` with
  `--control frames --control maps.mp4`, give the frames `pipeline.edit` gives for the same tensors.
"""
import os

import numpy as np
import pytest
import torch
import yaml

from oracle import gen_canny_golden as gg
from oracle import ldm_layout
from oracle import multi_controlnet as MC
from tokenflow_b200 import pipeline, preprocess, run, sd_unet
from tokenflow_b200 import synthetic_checkpoint as fx
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.controlnet import MultiControlNetModel, build_controlnet
from tokenflow_b200.editor import TokenFlowEditor, synthetic_inputs
from tokenflow_b200.preprocess import LatentInverter
from tokenflow_b200.scheduler import DDIMScheduler
from tokenflow_b200.util import save_video
from tokenflow_b200.video import read_video

pytestmark = pytest.mark.gpu

SCALES = [0.8, 0.5]


def _frames(n, h, w, seed=5):
    rng = np.random.default_rng(seed)
    return torch.from_numpy(np.stack([gg.make_frame("smooth", h, w, rng) for _ in range(n)])).cuda()


def _cond(n, h, w):
    """Canny for the first net, the frames of another seed as maps for the second."""
    return preprocess.control_cond(_frames(n, h, w), ["canny", _frames(n, h, w, seed=6)])


def _models(kind):
    tfu._install_ops_for_testing(None)
    unet = sd_unet.build_unet(kind, seed=1, device="cuda", dtype=torch.float16, init_on_device=kind != "tiny")
    nets = [build_controlnet(kind, seed=s, device="cuda", dtype=torch.float16) for s in (3, 4)]
    if kind != "tiny":
        unet = unet.to(memory_format=torch.channels_last)
        nets = [n.to(memory_format=torch.channels_last) for n in nets]
    return unet, nets


def test_inversion_graph_replay_equals_eager_and_the_reference_loop():
    unet, nets = _models("sd15")
    g = torch.Generator().manual_seed(3)
    n = 4
    x0 = torch.randn(n, 4, 64, 64, generator=g).half().cuda()
    cond = torch.randn(1, 77, 768, generator=g).half().cuda()
    ccond = _cond(n, 512, 512)
    res = {}
    for graphed in (True, False):
        inv = LatentInverter(unet, DDIMScheduler(), 6, controlnet=MultiControlNetModel(nets), controlnet_cond=ccond,
                             controlnet_conditioning_scale=SCALES)
        inv._use_graph = graphed
        xT = inv.ddim_inversion(cond, x0, None, batch_size=2)
        rec = inv.ddim_sample(xT, cond, batch_size=2)
        res[graphed] = (xT, rec, inv.saved_latents(), inv.scheduler)
    assert torch.isfinite(res[True][1]).all()
    assert torch.equal(res[True][0], res[False][0]) and torch.equal(res[True][1], res[False][1])
    for t in res[True][2]:
        assert torch.equal(res[True][2][t], res[False][2][t]), t
    sch = res[True][3]
    want_T, _ = MC.ddim_inversion(unet, nets, SCALES, sch, cond, ccond, x0.clone(), 2)
    want_rec = MC.ddim_sample(unet, nets, SCALES, sch, want_T.clone(), cond, ccond, 2)
    assert torch.equal(res[True][0], want_T), (res[True][0].float() - want_T.float()).abs().max().item()
    assert torch.equal(res[True][1], want_rec), (res[True][1].float() - want_rec.float()).abs().max().item()
    one = LatentInverter(unet, DDIMScheduler(), 6, controlnet=nets[0], controlnet_cond=ccond[:, :3],
                         controlnet_conditioning_scale=SCALES[0])
    assert not torch.equal(one.ddim_inversion(cond, x0, None, batch_size=2), res[True][0])


def _editor(kind, mode, steps, graph, n_frames=8, batch=2, latent=16, frames_per_pass=None):
    unet, nets = _models(kind)
    cfg = {"n_frames": n_frames, "batch_size": batch, "n_timesteps": steps, "guidance_scale": 7.5, "mode": mode,
           "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "start": 0.9, "fused_pass": True, "cuda_graph": graph,
           "keyframe_seed": 1, "controlnet_conditioning_scale": SCALES}
    if frames_per_pass:
        cfg["frames_per_pass"] = frames_per_pass
    x, text, pnp, src = synthetic_inputs(n_frames, latent, unet.config.cross_attention_dim, steps, seed=1,
                                         device="cuda", dtype=torch.float16, ctx_len=7)
    ed = TokenFlowEditor(unet, DDIMScheduler(), tfu, cfg, text, pnp, source_latents=lambda t: src[t],
                         controlnet=MultiControlNetModel(nets), controlnet_cond=_cond(n_frames, 8 * latent, 8 * latent))
    ed.init_method()
    return ed, x


@pytest.mark.parametrize("kind,mode,steps,fpp", [pytest.param("tiny", "pnp", 5, None, id="tiny-pnp-5"),
                                                 pytest.param("tiny", "pnp", 5, 3, id="tiny-pnp-5-chunks"),
                                                 pytest.param("tiny", "sdedit", 10, None, id="tiny-sdedit-10"),
                                                 pytest.param("tiny", "sdedit", 10, 3, id="tiny-sdedit-10-chunks"),
                                                 pytest.param("sd15", "pnp", 5, None, id="sd15-pnp-5"),
                                                 pytest.param("sd15", "pnp", 5, 4, id="sd15-pnp-5-chunks"),
                                                 pytest.param("sd15", "sdedit", 10, None, id="sd15-sdedit-10")])
def test_cuda_graph_step_identical_to_eager(kind, mode, steps, fpp):
    kw = {} if kind == "tiny" else dict(latent=64, batch=4)
    ed_e, x = _editor(kind, mode, steps, graph=False, frames_per_pass=fpp, **kw)
    want = ed_e.sample_loop(x.clone())
    ed_g, x = _editor(kind, mode, steps, graph=True, frames_per_pass=fpp, **kw)
    got = ed_g.sample_loop(x.clone())
    assert ed_g.keyframe_log == ed_e.keyframe_log
    assert len(ed_g._graphs) == (3 if mode == "pnp" else 1)       # every PnP injection variant was captured
    assert all(e["replays"] >= 1 for e in ed_g._graphs.values())
    assert torch.isfinite(got).all()
    assert torch.equal(got, want), (got.float() - want.float()).abs().max().item()


def test_control_cond_on_cuda_equals_the_cpu_path():
    frames = _frames(5, 96, 160)
    maps = _frames(7, 120, 90, seed=9)
    got = preprocess.control_cond(frames, [maps, "frames", "canny"])
    want = preprocess.control_cond(frames.cpu(), [maps.cpu(), "frames", "canny"])
    assert got.is_cuda and got.shape == (5, 9, 96, 160)
    assert torch.equal(got.cpu(), want)
    v = torch.arange(256, dtype=torch.uint8).reshape(1, 16, 16, 1).expand(1, 16, 16, 3).contiguous().cuda()
    unit = preprocess.control_cond(v, ["frames"]).cpu()
    assert torch.equal(unit, torch.from_numpy(np.float32(v.cpu().numpy()) / 255).half().permute(0, 3, 1, 2))


N, H, W = 8, 256, 384
PNP = {"prompt": "a marble sculpture of a woman", "negative_prompt": "ugly blurry", "guidance_scale": 7.5,
       "n_timesteps": 5, "batch_size": 4, "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "seed": 1}


@torch.no_grad()
def test_cli_with_a_folder_and_a_pth_controlnet_equals_the_pipeline(tmp_path, monkeypatch):
    tfu._install_ops_for_testing(None)
    root = str(tmp_path)
    model_dir, cn_dir = fx.write_checkpoint(root, "sd15", controlnet=True, dtype=torch.float16, init_device="cuda")
    pth = os.path.join(root, "control_v11f1p_sd15_depth.pth")
    ldm_layout.save(pth, ldm_layout.ldm_controlnet(build_controlnet("sd15", seed=4)), torch.float16)
    monkeypatch.chdir(tmp_path)
    frames = _frames(N, H, W).cpu()
    run.write_frames(frames, "data/clip")
    save_video(_frames(N + 1, 240, 320, seed=7).cpu(), "maps.mp4", fps=10)
    argv = ["--model_dir", model_dir, "--controlnet_dir", cn_dir, "--controlnet_dir", pth,
            "--control", "frames", "--control", "maps.mp4"]
    run.main(["preprocess", *argv, "--data_path", "data/clip", "--H", str(H), "--W", str(W), "--save_dir", "latents",
              "--sd_version", "1.5", "--steps", "10", "--batch_size", "8", "--save_steps", "5", "--n_frames", str(N),
              "--controlnet_conditioning_scale", *map(str, SCALES)])
    cfg = {**PNP, "data_path": "data/clip", "latents_path": "latents", "sd_version": "1.5", "n_inversion_steps": 10,
           "n_frames": N, "output_path": "out", "controlnet_conditioning_scale": SCALES}
    with open("config.yaml", "w") as f:
        yaml.dump(cfg, f)
    run.main(["edit", *argv, "--config_path", "config.yaml"])
    assert yaml.safe_load(open("out/config.yaml"))["controlnets"] == [
        {"path": cn_dir, "control": "frames", "scale": SCALES[0]}, {"path": pth, "control": "maps.mp4",
                                                                     "scale": SCALES[1]}]
    got = run.read_frames("out/img_ode", N)
    assert got.shape == (N, H, W, 3) and os.path.isfile("out/tokenflow_PnP_fps_10.mp4")

    parts = pipeline.load_parts(model_dir, "cuda", torch.float16, [cn_dir, pth])
    maps = read_video("maps.mp4")[0]
    saved = run.read_latents(os.path.join("latents", "sd_1.5", "clip", "steps_10", f"nframes_{N}"))
    want_saved, _ = pipeline.preprocess(parts, frames, {"H": H, "W": W, "steps": 10, "batch_size": 8,
                                                        "save_steps": 5, "inversion_prompt": "a woman running",
                                                        "controlnet_conditioning_scale": SCALES},
                                        controls=["frames", maps])
    assert sorted(saved) == sorted(want_saved) and all(torch.equal(saved[t], want_saved[t].cpu()) for t in saved)
    torch.manual_seed(1)
    want = pipeline.edit(parts, frames, {**cfg, "inversion_prompt": "a woman running"}, saved,
                         controls=["frames", maps])
    assert torch.equal(got, want.cpu())
    assert 0 < got.float().std()
