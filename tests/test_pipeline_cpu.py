"""CPU tier: `pipeline.preprocess` + `pipeline.edit` and the `python -m tokenflow_b200.run` command line, on synthetic
checkpoint folders, with the oracle ops under the hooks.

* the two stages equal, bit for bit (fp32, torch.equal), the INTEGRATION.md §6 chain written out by hand from the same
  folders: PnP, SDEdit with and without DDIM noise, with a Canny ControlNet, and with a v-prediction scheduler;
* the hand chain encodes its prompts with direct CLIPTextModel calls in the reference's order;
* the command line reads a PNG frame directory, writes the reference's latents directory (read back by
  `load_source_latents_t`), and writes %05d.png frames equal to what `edit` returns;
* under torchrun's environment, two gloo ranks per stage write the latents one process computes, and edited frames
  within 1 of its edit with the same keyframe generator.
"""
import os

import numpy as np
import pytest
import torch
import yaml

from tokenflow_b200 import synthetic_checkpoint as fx

from oracle.oracle_ops import OracleOps
from tokenflow_b200 import checkpoint, pipeline, run
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.editor import TokenFlowEditor
from tokenflow_b200.preprocess import (LatentInverter, canny_cond, ddim_eps, decode_latents, encode_imgs,
                                       resize_frames)

N, H, W = 8, 64, 96
OPT = {"H": H, "W": W, "steps": 10, "batch_size": 4, "save_steps": 5, "inversion_prompt": "a woman running"}
PNP = {"prompt": "a marble sculpture of a woman", "negative_prompt": "ugly blurry", "guidance_scale": 7.5,
       "n_timesteps": 5, "batch_size": 4, "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "seed": 1}
SDEDIT = {"prompt": "a shiny silver robotic wolf", "negative_prompt": "ugly blurry", "guidance_scale": 7.5,
          "n_timesteps": 5, "batch_size": 4, "start": 0.9, "use_ddim_noise": True, "seed": 1}


def frames(n=N, h=48, w=80, seed=0):
    """Smooth random uint8 frames [n, h, w, 3] with edges for Canny."""
    g = torch.Generator().manual_seed(seed)
    base = torch.nn.functional.interpolate(torch.rand(n, 3, h // 8, w // 8, generator=g), size=(h, w),
                                           mode="bilinear", align_corners=False)
    return (base * 255).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def _direct_embeds(tok, enc, prompt, negative):
    """The reference's get_text_embeds written out: CLIPTextModel on the tokenizer's ids, uncond then cond."""
    with torch.no_grad():
        cond = enc(tok(prompt, padding="max_length", max_length=tok.model_max_length, truncation=True,
                       return_tensors="pt").input_ids)[0]
        uncond = enc(tok(negative, padding="max_length", max_length=tok.model_max_length,
                         return_tensors="pt").input_ids)[0]
    return torch.cat([uncond, cond])


@torch.no_grad()
def hand_chain(model_dir, cn_dir, frames_u8, opt, config):
    """INTEGRATION.md §6 stage by stage, from freshly loaded models."""
    from tokenflow_b200.scheduler import DDIMScheduler
    import json
    unet = checkpoint.load_unet(model_dir)
    vae = checkpoint.load_vae(model_dir)
    cn = checkpoint.load_controlnet(cn_dir) if cn_dir else None
    tok, enc = checkpoint.load_text_encoder(model_dir)
    with open(os.path.join(model_dir, "scheduler", "scheduler_config.json")) as f:
        sched = json.load(f)
    # preprocess
    fr = resize_frames(frames_u8, (opt["H"], opt["W"]))
    latents = encode_imgs(vae, fr)
    edges = canny_cond(fr) if cn is not None else None
    toy = DDIMScheduler.from_config(sched)
    toy.set_timesteps(opt["save_steps"])
    inv = LatentInverter(unet, DDIMScheduler.from_config(sched), opt["steps"], controlnet=cn, controlnet_cond=edges)
    cond = _direct_embeds(tok, enc, opt["inversion_prompt"], "")[1:]
    x_T = inv.ddim_inversion(cond, latents, None, batch_size=opt["batch_size"],
                             timesteps_to_save=toy.timesteps.tolist())
    recon = decode_latents(vae, inv.ddim_sample(x_T, cond, batch_size=opt["batch_size"]))
    saved = inv.saved_latents()
    # edit
    torch.manual_seed(config["seed"])
    text = _direct_embeds(tok, enc, config["prompt"], config["negative_prompt"])
    pnp = _direct_embeds(tok, enc, opt["inversion_prompt"], opt["inversion_prompt"]).chunk(2)[0]
    mode = "pnp" if "pnp_attn_t" in config else "sdedit"
    cfg = {**config, "mode": mode, "fused_pass": True}
    editor = TokenFlowEditor(unet, DDIMScheduler.from_config(sched), tfu, cfg, text, pnp,
                             source_latents=saved.__getitem__, controlnet=cn, controlnet_cond=edges)
    eps = ddim_eps(latents, saved, editor.scheduler)
    if mode == "sdedit" and not config["use_ddim_noise"]:
        eps = torch.randn_like(eps[[0]]).repeat(len(eps), 1, 1, 1)
    x = editor.scheduler.add_noise(latents, eps, editor.scheduler.timesteps[0])
    editor.init_method()
    return saved, recon, decode_latents(vae, editor.sample_loop(x))


def run_pipeline(model_dir, cn_dir, frames_u8, opt, config):
    parts = pipeline.load_parts(model_dir, "cpu", torch.float32, cn_dir)
    saved, recon = pipeline.preprocess(parts, frames_u8, opt)
    torch.manual_seed(config["seed"])
    out = pipeline.edit(parts, frames_u8, {**config, "inversion_prompt": opt["inversion_prompt"]}, saved)
    return saved, recon, out


CASES = {
    "pnp": (PNP, fx.SD15_SCHEDULER, False),
    "sdedit": (SDEDIT, fx.SD15_SCHEDULER, False),
    "sdedit-random-noise": ({**SDEDIT, "use_ddim_noise": False}, fx.SD15_SCHEDULER, False),
    "pnp-controlnet": (PNP, fx.SD15_SCHEDULER, True),
    "sdedit-controlnet": (SDEDIT, fx.SD15_SCHEDULER, True),
    "pnp-v": (PNP, fx.SD21_V_SCHEDULER, False),
}


@pytest.mark.parametrize("case", list(CASES))
def test_pipeline_equals_the_hand_chain(tmp_path, case):
    config, sched, with_cn = CASES[case]
    tfu._install_ops_for_testing(OracleOps())
    model_dir, cn_dir = fx.write_checkpoint(str(tmp_path), "tiny", scheduler=sched, controlnet=with_cn)
    fr = frames()
    saved, recon, out = run_pipeline(model_dir, cn_dir, fr, OPT, config)
    want_saved, want_recon, want_out = hand_chain(model_dir, cn_dir, fr, OPT, config)
    assert sorted(saved) == sorted(want_saved) == [1, 201, 401, 601, 801, 901]
    for t in saved:
        assert saved[t].dtype == torch.float32 and torch.equal(saved[t], want_saved[t]), t
    assert recon.shape == (N, H, W, 3) and recon.dtype == torch.uint8 and torch.equal(recon, want_recon)
    assert out.shape == (N, H, W, 3) and out.dtype == torch.uint8 and torch.equal(out, want_out)


def test_square_frames_are_edited_at_512(tmp_path):
    """The reference turns square frames into 512², whatever H and W say; the edit resizes to the latents' size."""
    tfu._install_ops_for_testing(OracleOps())
    model_dir, _ = fx.write_checkpoint(str(tmp_path), "tiny")
    parts = pipeline.load_parts(model_dir, "cpu", torch.float32)
    fr = frames(n=2, h=40, w=40)
    opt = {**OPT, "steps": 2, "save_steps": 1, "batch_size": 2}
    saved, recon = pipeline.preprocess(parts, fr, opt)
    assert recon.shape == (2, 512, 512, 3) and all(v.shape == (2, 4, 64, 64) for v in saved.values())


def _write_pngs(folder, frames_u8):
    from PIL import Image
    os.makedirs(folder, exist_ok=True)
    for i, f in enumerate(frames_u8.numpy()):
        Image.fromarray(f).save(os.path.join(folder, f"{i:05d}.png"))


@pytest.mark.parametrize("config", [PNP, SDEDIT], ids=["pnp", "sdedit"])
def test_cli_writes_the_reference_layout_and_the_edit(tmp_path, monkeypatch, config):
    tfu._install_ops_for_testing(OracleOps())
    model_dir, _ = fx.write_checkpoint(str(tmp_path), "tiny")
    fr = frames()
    data = tmp_path / "data" / "clip"
    _write_pngs(str(data), fr)
    monkeypatch.chdir(tmp_path)
    run.main(["preprocess", "--model_dir", model_dir, "--device", "cpu", "--data_path", str(data), "--H", str(H),
              "--W", str(W), "--save_dir", "latents", "--sd_version", "1.5", "--steps", "10", "--batch_size", "4",
              "--save_steps", "5", "--n_frames", str(N), "--inversion_prompt", OPT["inversion_prompt"]])
    lat = tmp_path / "latents" / "sd_1.5" / "clip" / "steps_10" / f"nframes_{N}"
    assert (lat / "inversion_prompt.txt").read_text() == OPT["inversion_prompt"]
    assert yaml.safe_load((tmp_path / "latents" / "inversion_prompts.yaml").read_text()) == {
        "clip": OPT["inversion_prompt"]}
    assert sorted(os.listdir(lat / "frames")) == [f"{i:05d}.png" for i in range(N)]
    # what the stages compute in one process, the files hold
    parts = pipeline.load_parts(model_dir, "cpu", torch.float32)
    saved, _ = pipeline.preprocess(parts, fr, OPT)
    for t, v in saved.items():
        assert torch.equal(tfu.load_source_latents_t(t, str(lat / "latents")), v), t
    cfg = {**config, "data_path": str(data), "latents_path": "latents", "sd_version": "1.5", "n_inversion_steps": 10,
           "n_frames": N, "output_path": str(tmp_path / "out")}
    with open(tmp_path / "config.yaml", "w") as f:
        yaml.dump(cfg, f)
    run.main(["edit", "--model_dir", model_dir, "--device", "cpu", "--config_path", str(tmp_path / "config.yaml")])
    written = run.read_frames(str(tmp_path / "out" / "img_ode"), N)
    torch.manual_seed(config["seed"])
    parts = pipeline.load_parts(model_dir, "cpu", torch.float32)
    want = pipeline.edit(parts, fr, {**config, "inversion_prompt": OPT["inversion_prompt"]}, saved)
    assert torch.equal(written, want)
    assert yaml.safe_load((tmp_path / "out" / "config.yaml").read_text())["inversion_prompt"] == OPT["inversion_prompt"]
    assert np.asarray(written).std() > 0


def _cli_rank(rank, world, port, argv, q):
    os.environ.update({"WORLD_SIZE": str(world), "RANK": str(rank), "LOCAL_RANK": str(rank),
                       "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port)})
    torch.set_num_threads(2)
    tfu._install_ops_for_testing(OracleOps())
    try:
        run.main(argv)
        q.put((rank, None))
    except Exception as e:  # noqa: BLE001  — reported to the parent
        q.put((rank, repr(e)))


def _torchrun(argv, world=2):
    """`argv` in `world` fresh processes with torchrun's environment, as one stage of a torchrun job."""
    import socket
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_cli_rank, args=(r, world, port, argv, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        results = dict(q.get(timeout=300) for _ in procs)
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join()
    assert results == {r: None for r in range(world)}
    assert all(p.exitcode == 0 for p in procs)


def test_cli_on_two_gloo_ranks_equals_one_process(tmp_path):
    """`torchrun --nproc_per_node 2 -m tokenflow_b200.run ... --device cpu`: each rank inverts and edits its share of
    the frames; rank 0 writes what one process computes with the same keyframe generator."""
    tfu._install_ops_for_testing(OracleOps())
    model_dir, _ = fx.write_checkpoint(str(tmp_path), "tiny")
    fr = frames()
    data = tmp_path / "data" / "clip"
    _write_pngs(str(data), fr)
    cfg = {**PNP, "data_path": str(data), "latents_path": str(tmp_path / "latents"), "sd_version": "1.5",
           "n_inversion_steps": 10, "n_frames": N, "output_path": str(tmp_path / "out")}
    with open(tmp_path / "config.yaml", "w") as f:
        yaml.dump(cfg, f)
    common = ["--model_dir", model_dir, "--device", "cpu"]
    argvs = [["preprocess", *common, "--data_path", str(data), "--H", str(H), "--W", str(W), "--save_dir",
              str(tmp_path / "latents"), "--sd_version", "1.5", "--steps", "10", "--batch_size", "4",
              "--save_steps", "5", "--n_frames", str(N), "--inversion_prompt", OPT["inversion_prompt"]],
             ["edit", *common, "--config_path", str(tmp_path / "config.yaml")]]
    for argv in argvs:                                   # each stage is its own job
        _torchrun(argv)
    parts = pipeline.load_parts(model_dir, "cpu", torch.float32)
    saved, _ = pipeline.preprocess(parts, fr, OPT)
    lat = tmp_path / "latents" / "sd_1.5" / "clip" / "steps_10" / f"nframes_{N}" / "latents"
    for t, v in saved.items():
        assert torch.equal(torch.load(lat / f"noisy_latents_{t}.pt"), v), t
    want = pipeline.edit(parts, fr, {**PNP, "keyframe_seed": 1, "inversion_prompt": OPT["inversion_prompt"]}, saved)
    got = run.read_frames(str(tmp_path / "out" / "img_ode"), N)
    assert (got.int() - want.int()).abs().max() <= 1
