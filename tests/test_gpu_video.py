"""GPU tier (-m gpu, H100): video files through the CUDA resize and the command line.

* frames extracted with `read_video(..., device="cuda")` (decoded by OpenCV, resized by `tf_resize_u8`) equal the CPU
  extraction (PIL's Lanczos) byte for byte: the reference's `wolf.mp4` at 512² and 384 x 672, and a 1920 x 1080 clip
  at 512² and 384 x 672, with chunks that do not divide the frame count;
* `run preprocess --data_path wolf.mp4` then `run edit`, PnP and SDEdit, at 8 frames on a synthetic full-size SD1.5
  checkpoint, write exactly what `pipeline.preprocess` and `pipeline.edit` return in memory: the extracted frames,
  the latents, the reconstruction, the edited frames and the VAE reconstruction, and every mp4 at its frame count.
"""
import os

import pytest
import torch
import yaml

from tokenflow_b200 import synthetic_checkpoint as fx

from tokenflow_b200 import pipeline, run
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.preprocess import decode_latents, encode_imgs
from tokenflow_b200.util import save_video, seed_everything
from tokenflow_b200.video import read_video

pytestmark = pytest.mark.gpu

WOLF = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wolf.mp4")
N = 8
OPT = {"H": 512, "W": 512, "steps": 10, "batch_size": 8, "save_steps": 5, "inversion_prompt": "a wolf"}
PNP = {"prompt": "a marble sculpture of a wolf", "negative_prompt": "ugly blurry", "guidance_scale": 7.5,
       "n_timesteps": 5, "batch_size": 4, "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "seed": 1}
SDEDIT = {"prompt": "a shiny silver robotic wolf", "negative_prompt": "ugly blurry", "guidance_scale": 7.5,
          "n_timesteps": 5, "batch_size": 4, "start": 0.9, "use_ddim_noise": True, "seed": 1}


def hd_clip(path, n=10):
    g = torch.Generator().manual_seed(0)
    base = torch.nn.functional.interpolate(torch.rand(n, 3, 1080 // 40, 1920 // 40, generator=g), size=(1080, 1920),
                                           mode="bilinear", align_corners=False)
    save_video((base * 255).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous(), path, fps=30)


def test_cuda_extraction_equals_pil(tmp_path):
    hd = str(tmp_path / "hd.mp4")
    hd_clip(hd)
    for path, n in ((WOLF, 40), (hd, 10)):
        for size in (512, (384, 672)):
            want, fps = read_video(path, size, "cpu")
            got, got_fps = read_video(path, size, "cuda", chunk=7)
            h, w = (size, size) if isinstance(size, int) else size
            assert got.shape == (n, h, w, 3) and not got.is_cuda and got_fps == fps
            assert torch.equal(got, want), (path, size)


@pytest.fixture(scope="module")
def sd15(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("sd15"))
    model_dir, _ = fx.write_checkpoint(root, "sd15", variant="fp16", dtype=torch.float16, init_device="cuda",
                                       deprecated_vae=True)
    torch.cuda.empty_cache()
    return model_dir


def test_cli_from_the_references_video_writes_the_pipelines_result(sd15, tmp_path, monkeypatch):
    tfu._install_ops_for_testing(None)
    monkeypatch.chdir(tmp_path)
    os.makedirs("data")
    os.symlink(WOLF, "data/wolf.mp4")
    common = ["--model_dir", sd15, "--variant", "fp16"]
    run.main(["preprocess", *common, "--data_path", "data/wolf.mp4", "--sd_version", "1.5", "--steps",
              str(OPT["steps"]), "--batch_size", str(OPT["batch_size"]), "--save_steps", str(OPT["save_steps"]),
              "--n_frames", str(N), "--inversion_prompt", OPT["inversion_prompt"]])
    decoded, _ = read_video(WOLF, 512, "cpu")
    assert torch.equal(run.read_frames("data/wolf", 40), decoded)
    lat = os.path.join("latents", "sd_1.5", "wolf", "steps_10", f"nframes_{N}")

    parts = pipeline.load_parts(sd15, "cuda", torch.float16, variant="fp16")
    saved, recon = pipeline.preprocess(parts, decoded[:N], OPT)
    written = run.read_latents(lat)
    assert sorted(written) == sorted(saved)
    for t in saved:
        assert torch.equal(written[t], saved[t].cpu()), t
    assert torch.equal(run.read_frames(os.path.join(lat, "frames"), N), recon.cpu())
    inverted, fps = read_video(os.path.join(lat, "inverted.mp4"))
    assert inverted.shape == (N, 512, 512, 3) and fps == 10.0

    for mode, config in (("PnP", PNP), ("SDEdit", SDEDIT)):
        out = tmp_path / mode
        cfg = {**config, "data_path": "data/wolf", "latents_path": "latents", "sd_version": "1.5",
               "n_inversion_steps": 10, "n_frames": N, "output_path": str(out)}
        with open("config.yaml", "w") as f:
            yaml.dump(cfg, f)
        run.main(["edit", *common, "--config_path", "config.yaml"])
        del parts                             # each edit on freshly loaded models, as each `run edit` loads its own
        torch.cuda.empty_cache()
        parts = pipeline.load_parts(sd15, "cuda", torch.float16, variant="fp16")
        seed_everything(config["seed"])
        want = pipeline.edit(parts, decoded[:N], {**config, "inversion_prompt": OPT["inversion_prompt"]}, saved)
        assert torch.equal(run.read_frames(str(out / "img_ode"), N), want.cpu()), mode
        names = [f"tokenflow_{mode}_fps_{fps}.mp4" for fps in (10, 20, 30)]
        if mode == "PnP":
            names += [f"vae_recon_{fps}.mp4" for fps in (10, 20, 30)]
            want_recon = decode_latents(parts.vae, encode_imgs(parts.vae, decoded[:N].cuda()))
            assert torch.equal(run.read_frames(str(out / "vae_recon"), N), want_recon.cpu())
        for name in names:
            frames, fps = read_video(str(out / name))
            assert frames.shape == (N, 512, 512, 3) and fps == float(name[:-4].rsplit("_", 1)[1]), name
