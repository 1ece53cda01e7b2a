"""Command line of the two stages: a diffusers checkpoint directory, a video file or frame directory and a config in,
the reference's latents directory, edited frames and videos out.

    python -m tokenflow_b200.run preprocess --model_dir DIR --data_path VIDEO_OR_FRAMES [--H 512 --W 512
        --save_dir latents --sd_version 2.1 --steps 500 --batch_size 40 --save_steps 50 --n_frames 40
        --inversion_prompt "..."]
    python -m tokenflow_b200.run edit --config_path configs/config_pnp.yaml --model_dir DIR [--controlnet_dir DIR]

`preprocess` takes the reference's flags (preprocess.py:336-349).  A `--data_path` that is a file is a video: as
preprocess.py:351-354 does, every frame is decoded (`video.read_video`, OpenCV's FFmpeg) and resized to --W x --H,
rank 0 writes them to data/<stem>/%05d.png under the working directory, and the first `n_frames` of them are
preprocessed as if `--data_path data/<stem>` had been given; a video shorter than `n_frames` is refused before any
model loads.  Every torchrun rank decodes and resizes the video itself: the resize is integer arithmetic, so the
ranks hold the same frames.  A directory is read as %05d.png, else %05d.jpg (util.load_imgs), with PIL.  `preprocess`
writes the reference's latents directory (<save_dir>/sd_<ver>/<name>/steps_<n>/nframes_<n>/latents/
noisy_latents_<t>.pt, inversion_prompt.txt, frames/ and inverted.mp4 at 10 fps with the reconstruction) and
<save_dir>/inversion_prompts.yaml.

`edit` takes the reference's YAML config (config_pnp.yaml or config_sdedit.yaml; PnP when it has pnp_attn_t), finds
the latents directory the way run_tokenflow_pnp.py does, and writes under <output_path>: the edited frames as
img_ode/%05d.png, tokenflow_PnP_fps_{10,20,30}.mp4 or tokenflow_SDEdit_fps_{10,20,30}.mp4 of them, config.yaml,
and for PnP the VAE reconstruction of the source frames as vae_recon/%05d.png and vae_recon_{10,20,30}.mp4
(run_tokenflow_pnp.py:242-261, run_tokenflow_sdedit.py:201-203).  The mp4 files are MPEG-4 Part 2 (`mp4v`,
`util.save_video`), not the reference's H.264.  The config's sd_version, data_path, latents_path and
n_inversion_steps must name the directory preprocess wrote.  It edits min(n_frames, the latents' frame count)
frames; unlike the reference's driver it does not trim that count to a multiple of batch_size, since the editor
takes a short last keyframe group (INTEGRATION.md §6).

`--controlnet_dir` adds a Canny ControlNet to both stages, from a diffusers folder or a single cldm file.
`--weights FILE` takes the UNet, VAE and text encoder weights from a single-file checkpoint in the original LDM
layout; `--model_dir` must then be a diffusers folder of the same family, which gives the architectures, the
tokenizer and the scheduler.  `--lora FILE[:SCALE]` (repeatable, SCALE 1.0 by default) merges a LoRA into the UNet
and the text encoder once they are loaded (`lora.merge`).  It applies to the stage it is given to: to invert with the
base model and edit with the LoRA, give it to `edit` only.  The latents directory's name does not depend on it;
`edit` records the LoRAs in its config.yaml (`loras: [{path, scale}]`).  Under torchrun every process edits on its
local GPU (`LOCAL_RANK`), and reads and merges each LoRA itself: frames are sharded over the ranks and the
all-gathers run through `ops.Communicator`; rank 0 writes the files.  With `--device cpu` the processes run on the
CPU and gather over gloo.
"""
from __future__ import annotations

import argparse
import glob
import os
import re
import sys
from pathlib import Path
from typing import List, Optional, Tuple

import numpy as np
import torch


def read_frames(data_path: str, n_frames: int) -> torch.Tensor:
    """[n, H, W, 3] uint8 from <data_path>/%05d.png, or %05d.jpg when there is no 00000.png."""
    from PIL import Image
    ext = "png" if os.path.exists(os.path.join(data_path, "00000.png")) else "jpg"
    paths = [os.path.join(data_path, f"{i:05d}.{ext}") for i in range(n_frames)]
    return torch.from_numpy(np.stack([np.asarray(Image.open(p).convert("RGB")) for p in paths]))


def write_frames(frames_u8: torch.Tensor, folder: str) -> None:
    from PIL import Image
    os.makedirs(folder, exist_ok=True)
    for i, f in enumerate(frames_u8.cpu().numpy()):
        Image.fromarray(f).save(os.path.join(folder, f"{i:05d}.png"))


def find_latents(config: dict) -> str:
    """The latents directory an edit reads (run_tokenflow_pnp.py:114-125): under
    <latents_path>/sd_<ver>/<name>/steps_<n_inversion_steps>, the nframes_<n> directory with the most frames."""
    root = os.path.join(config["latents_path"], f"sd_{config['sd_version']}", Path(config["data_path"]).stem,
                        f"steps_{config['n_inversion_steps']}")
    found = [d for d in glob.glob(os.path.join(root, "nframes_*")) if os.path.isdir(d)]
    if not found:
        raise FileNotFoundError(f"no nframes_<n> latents directory under {root}: run preprocess first")
    return max(found, key=lambda d: int(d.rsplit("_", 1)[1]))


def read_latents(path: str) -> dict:
    """{t: tensor} of <path>/latents/noisy_latents_<t>.pt."""
    files = glob.glob(os.path.join(path, "latents", "noisy_latents_*.pt"))
    return {int(re.search(r"noisy_latents_(\d+)\.pt$", f).group(1)): torch.load(f, map_location="cpu")
            for f in files}


def parse_lora(arg: str) -> Tuple[str, float]:
    """(path, scale) of a `--lora FILE[:SCALE]` argument: a suffix after the last `:` that parses as a float is the
    scale, else the whole argument is the path and the scale is 1.0."""
    path, sep, tail = arg.rpartition(":")
    if sep:
        try:
            return path, float(tail)
        except ValueError:
            pass
    return arg, 1.0


def _distributed(device: str):
    """(world_size, rank, communicator, device) of this process: under torchrun one GPU per process (`LOCAL_RANK`)
    with the library's NCCL all-gather, or CPU processes over gloo with `--device cpu`; else one process."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world == 1:
        return 1, 0, None, torch.device(device)
    import torch.distributed as dist
    if torch.device(device).type == "cpu":
        dist.init_process_group("gloo")
        return world, dist.get_rank(), None, torch.device("cpu")
    from .ops import Communicator
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl")
    rank = dist.get_rank()
    return world, rank, Communicator(world, rank), torch.device("cuda", local)


def main(argv: Optional[List[str]] = None) -> None:
    ap = argparse.ArgumentParser(prog="python -m tokenflow_b200.run")
    sub = ap.add_subparsers(dest="stage", required=True)
    for name in ("preprocess", "edit"):
        p = sub.add_parser(name)
        p.add_argument("--model_dir", required=True, help="diffusers checkpoint directory (unet/, vae/, scheduler/, "
                                                          "text_encoder/, tokenizer/)")
        p.add_argument("--weights", default=None,
                       help="single-file SD checkpoint in the original LDM layout (.safetensors, .ckpt); its UNet, "
                            "VAE and text encoder weights replace --model_dir's, which still gives the architectures, "
                            "tokenizer and scheduler")
        p.add_argument("--controlnet_dir", default=None,
                       help="diffusers ControlNet directory (Canny), or a single-file ControlNet (.pth, .safetensors) "
                            "built on --model_dir's UNet config")
        p.add_argument("--variant", default=None, help="weights variant of the folders read, e.g. fp16")
        p.add_argument("--lora", action="append", default=[], type=parse_lora, metavar="FILE[:SCALE]",
                       help="LoRA file (kohya, diffusers or PEFT layout) merged into the UNet and text encoder of this "
                            "stage at SCALE (default 1.0); repeatable")
        p.add_argument("--device", default="cuda")
    p = sub.choices["preprocess"]
    p.add_argument("--data_path", type=str, default="data/woman-running")
    p.add_argument("--H", type=int, default=512)
    p.add_argument("--W", type=int, default=512)
    p.add_argument("--save_dir", type=str, default="latents")
    p.add_argument("--sd_version", type=str, default="2.1")
    p.add_argument("--steps", type=int, default=500)
    p.add_argument("--batch_size", type=int, default=40)
    p.add_argument("--save_steps", type=int, default=50)
    p.add_argument("--n_frames", type=int, default=40)
    p.add_argument("--inversion_prompt", type=str, default="a woman running")
    sub.choices["edit"].add_argument("--config_path", type=str, default="configs/config_pnp.yaml")
    args = ap.parse_args(argv)
    world, rank, comm, device = _distributed(args.device)
    try:
        _run(args, world, rank, comm, device)
    finally:
        if world > 1:
            import torch.distributed as dist
            if comm is not None:
                comm.destroy()
            dist.destroy_process_group()


def read_video_input(args, rank: int, device: torch.device) -> torch.Tensor:
    """preprocess.py:351-354 for a video `--data_path`: every frame decoded and resized to (--H, --W) on `device`,
    written by rank 0 to data/<stem>/%05d.png; `args.data_path` becomes that folder.  Returns the first `n_frames`
    frames, or raises ValueError when the video has fewer."""
    from .video import read_video
    video = args.data_path
    frames, _ = read_video(video, (args.H, args.W), device)
    if args.n_frames > frames.shape[0]:
        raise ValueError(f"--n_frames {args.n_frames} but {video!r} has {frames.shape[0]} frames")
    args.data_path = os.path.join("data", Path(video).stem)
    if rank == 0:
        write_frames(frames, args.data_path)
    return frames[:args.n_frames]


def _run(args, world: int, rank: int, comm, device: torch.device) -> None:
    import yaml
    from . import pipeline
    from .util import add_dict_to_yaml_file, save_video, seed_everything
    video_frames = None
    if args.stage == "preprocess" and os.path.isfile(args.data_path):   # decoded first: a bad video fails fast
        video_frames = read_video_input(args, rank, device)
    dtype = torch.float16 if device.type == "cuda" else torch.float32
    parts = pipeline.load_parts(args.model_dir, device, dtype, args.controlnet_dir, args.variant, args.weights,
                                args.lora)
    dist_kw = dict(world_size=world, rank=rank, comm=comm)

    if args.stage == "preprocess":
        seed_everything(1)                                                   # preprocess.py:303
        frames = video_frames if video_frames is not None else read_frames(args.data_path, args.n_frames)
        _, recon = pipeline.preprocess(parts, frames, args, **dist_kw)
        if rank == 0:
            add_dict_to_yaml_file(os.path.join(args.save_dir, "inversion_prompts.yaml"), Path(args.data_path).stem,
                                  args.inversion_prompt)
            path = pipeline.latents_dir(args, frames.shape[0])
            write_frames(recon, os.path.join(path, "frames"))
            save_video(recon, os.path.join(path, "inverted.mp4"), fps=10)        # preprocess.py:329-330
        return

    with open(args.config_path) as f:
        config = yaml.safe_load(f)
    path = find_latents(config)
    with open(os.path.join(path, "inversion_prompt.txt")) as f:
        config["inversion_prompt"] = f.read()
    source = read_latents(path)
    n = min(int(config["n_frames"]), next(iter(source.values())).shape[0])
    seed_everything(int(config.get("seed", 1)))                              # run_tokenflow_pnp.py:277
    frames = read_frames(config["data_path"], n)
    pnp = pipeline.edit_mode(config) == "pnp"
    out = pipeline.edit(parts, frames, config, source, vae_recon=pnp and rank == 0, **dist_kw)
    if rank == 0:
        out_dir = config["output_path"]
        os.makedirs(out_dir, exist_ok=True)
        if args.lora:
            config["loras"] = [{"path": path, "scale": scale} for path, scale in args.lora]
        with open(os.path.join(out_dir, "config.yaml"), "w") as f:
            yaml.dump(config, f)
        videos = {}
        if pnp:                                                  # run_tokenflow_pnp.py:242-249 `save_vae_recon`
            out, videos["vae_recon"] = out
            write_frames(videos["vae_recon"], os.path.join(out_dir, "vae_recon"))
        write_frames(out, os.path.join(out_dir, "img_ode"))
        videos["tokenflow_PnP_fps" if pnp else "tokenflow_SDEdit_fps"] = out
        for name, frames_u8 in videos.items():
            for fps in (10, 20, 30):
                save_video(frames_u8, os.path.join(out_dir, f"{name}_{fps}.mp4"), fps=fps)


if __name__ == "__main__":
    main(sys.argv[1:])
