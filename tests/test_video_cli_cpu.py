"""CPU tier: `python -m tokenflow_b200.run` from a video file to the reference's output videos, on a synthetic tiny
checkpoint with the oracle ops under the hooks.

* `preprocess --data_path clip.mp4` writes data/clip/%05d.png, the decoded and resized frames, and latents equal bit
  for bit to those of `preprocess --data_path data/clip` on that folder, plus inverted.mp4 of the reconstruction;
* `edit` then writes img_ode/, and the reference's videos: tokenflow_PnP_fps_{10,20,30}.mp4 with vae_recon/ and
  vae_recon_{10,20,30}.mp4 for PnP, tokenflow_SDEdit_fps_{10,20,30}.mp4 for SDEdit, each with the frames' count and
  size at its fps; vae_recon/ is `decode_latents(encode_imgs(frames))`;
* two gloo ranks from the video write the data folder and latents one process writes.
"""
import os

import pytest
import torch
import yaml

from tokenflow_b200 import synthetic_checkpoint as fx

from oracle.oracle_ops import OracleOps
from tokenflow_b200 import pipeline, run
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.preprocess import decode_latents, encode_imgs
from tokenflow_b200.util import save_video
from tokenflow_b200.video import read_video

N, H, W = 8, 64, 96
PNP = {"prompt": "a marble sculpture of a woman", "negative_prompt": "ugly blurry", "guidance_scale": 7.5,
       "n_timesteps": 5, "batch_size": 4, "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "seed": 1}
SDEDIT = {"prompt": "a shiny silver robotic wolf", "negative_prompt": "ugly blurry", "guidance_scale": 7.5,
          "n_timesteps": 5, "batch_size": 4, "start": 0.9, "use_ddim_noise": True, "seed": 1}


def clip_file(path, n=N + 2, h=48, w=80):
    """A video of n smooth random frames at h x w, 10 fps; more frames than are preprocessed."""
    g = torch.Generator().manual_seed(0)
    base = torch.nn.functional.interpolate(torch.rand(n, 3, h // 8, w // 8, generator=g), size=(h, w),
                                           mode="bilinear", align_corners=False)
    save_video((base * 255).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous(), path, fps=10)


def preprocess_argv(model_dir, data_path, save_dir):
    return ["preprocess", "--model_dir", model_dir, "--device", "cpu", "--data_path", data_path, "--H", str(H),
            "--W", str(W), "--save_dir", save_dir, "--sd_version", "1.5", "--steps", "10", "--batch_size", "4",
            "--save_steps", "5", "--n_frames", str(N), "--inversion_prompt", "a woman running"]


def latents_of(save_dir):
    return run.read_latents(os.path.join(save_dir, "sd_1.5", "clip", "steps_10", f"nframes_{N}"))


def assert_video(path, n, fps, h=H, w=W):
    frames, got_fps = read_video(path)
    assert frames.shape == (n, h, w, 3) and got_fps == fps, path


def test_cli_from_a_video_writes_the_references_files(tmp_path, monkeypatch):
    tfu._install_ops_for_testing(OracleOps())
    model_dir, _ = fx.write_checkpoint(str(tmp_path / "ckpt"), "tiny")
    monkeypatch.chdir(tmp_path)
    clip_file("clip.mp4")
    run.main(preprocess_argv(model_dir, "clip.mp4", "latents"))
    decoded, _ = read_video("clip.mp4", (H, W))
    assert decoded.shape[0] == N + 2                        # every frame is extracted, the first N preprocessed
    assert torch.equal(run.read_frames("data/clip", N + 2), decoded)
    lat = os.path.join("latents", "sd_1.5", "clip", "steps_10", f"nframes_{N}")
    assert yaml.safe_load(open("latents/inversion_prompts.yaml")) == {"clip": "a woman running"}
    assert_video(os.path.join(lat, "inverted.mp4"), N, 10.0)
    # the same folder given as frames: the same latents, bit for bit
    run.main(preprocess_argv(model_dir, "data/clip", "from_folder"))
    from_video, from_folder = latents_of("latents"), latents_of("from_folder")
    assert sorted(from_video) == sorted(from_folder) == [1, 201, 401, 601, 801, 901]
    for t in from_video:
        assert torch.equal(from_video[t], from_folder[t]), t
    assert torch.equal(run.read_frames(os.path.join(lat, "frames"), N),
                       run.read_frames(os.path.join("from_folder", "sd_1.5", "clip", "steps_10", f"nframes_{N}",
                                                    "frames"), N))

    for mode, config in (("PnP", PNP), ("SDEdit", SDEDIT)):
        out = tmp_path / mode
        cfg = {**config, "data_path": "data/clip", "latents_path": "latents", "sd_version": "1.5",
               "n_inversion_steps": 10, "n_frames": N, "output_path": str(out)}
        with open("config.yaml", "w") as f:
            yaml.dump(cfg, f)
        run.main(["edit", "--model_dir", model_dir, "--device", "cpu", "--config_path", "config.yaml"])
        videos = [f"tokenflow_{mode}_fps_{fps}.mp4" for fps in (10, 20, 30)]
        folders = ["img_ode"]
        if mode == "PnP":
            videos += [f"vae_recon_{fps}.mp4" for fps in (10, 20, 30)]
            folders.append("vae_recon")
        assert sorted(os.listdir(out)) == sorted(videos + folders + ["config.yaml"])
        for name in videos:
            assert_video(str(out / name), N, float(name[:-4].rsplit("_", 1)[1]))
        assert run.read_frames(str(out / "img_ode"), N).shape == (N, H, W, 3)
    parts = pipeline.load_parts(model_dir, "cpu", torch.float32)
    want = decode_latents(parts.vae, encode_imgs(parts.vae, decoded[:N]))
    assert torch.equal(run.read_frames(str(tmp_path / "PnP" / "vae_recon"), N), want)
    assert sorted(os.listdir(tmp_path / "PnP" / "vae_recon")) == [f"{i:05d}.png" for i in range(N)]


def test_cli_from_a_video_on_two_gloo_ranks_equals_one_process(tmp_path, monkeypatch):
    from test_pipeline_cpu import _torchrun
    tfu._install_ops_for_testing(OracleOps())
    model_dir, _ = fx.write_checkpoint(str(tmp_path / "ckpt"), "tiny")
    monkeypatch.chdir(tmp_path)
    clip_file("clip.mp4")
    _torchrun(preprocess_argv(model_dir, "clip.mp4", "two"))
    two_frames = run.read_frames("data/clip", N + 2)
    run.main(preprocess_argv(model_dir, "clip.mp4", "one"))
    assert torch.equal(two_frames, run.read_frames("data/clip", N + 2))
    two, one = latents_of("two"), latents_of("one")
    assert sorted(two) == sorted(one)
    for t in one:
        assert torch.equal(two[t], one[t]), t
    lat = os.path.join("two", "sd_1.5", "clip", "steps_10", f"nframes_{N}")
    assert_video(os.path.join(lat, "inverted.mp4"), N, 10.0)
    # the edit on two ranks: rank 0 alone decodes and writes the VAE reconstruction
    cfg = {**PNP, "data_path": "data/clip", "latents_path": "two", "sd_version": "1.5", "n_inversion_steps": 10,
           "n_frames": N, "output_path": "out"}
    with open("config.yaml", "w") as f:
        yaml.dump(cfg, f)
    _torchrun(["edit", "--model_dir", model_dir, "--device", "cpu", "--config_path", "config.yaml"])
    parts = pipeline.load_parts(model_dir, "cpu", torch.float32)
    want = decode_latents(parts.vae, encode_imgs(parts.vae, two_frames[:N]))
    assert torch.equal(run.read_frames("out/vae_recon", N), want)
    for name in ("tokenflow_PnP_fps", "vae_recon"):
        for fps in (10, 20, 30):
            assert_video(f"out/{name}_{fps}.mp4", N, float(fps))
