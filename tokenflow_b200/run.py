"""Command line of the two stages: a diffusers checkpoint directory, a frame directory and a config in, the reference's
latents directory and edited frames out.

    python -m tokenflow_b200.run preprocess --model_dir DIR --data_path FRAMES [--H 512 --W 512 --save_dir latents
        --sd_version 2.1 --steps 500 --batch_size 40 --save_steps 50 --n_frames 40 --inversion_prompt "..."]
    python -m tokenflow_b200.run edit --config_path configs/config_pnp.yaml --model_dir DIR [--controlnet_dir DIR]

`preprocess` takes the reference's flags (preprocess.py:336-349) and writes its latents directory
(<save_dir>/sd_<ver>/<name>/steps_<n>/nframes_<n>/latents/noisy_latents_<t>.pt, inversion_prompt.txt, frames/ with the
reconstruction) and <save_dir>/inversion_prompts.yaml.  `edit` takes the reference's YAML config (config_pnp.yaml or
config_sdedit.yaml; PnP when it has pnp_attn_t), finds the latents directory the way run_tokenflow_pnp.py does, and
writes the edited frames as <output_path>/img_ode/%05d.png, and the config as <output_path>/config.yaml.  The config's
sd_version, data_path, latents_path and n_inversion_steps must name the directory preprocess wrote.  It edits
min(n_frames, the latents' frame count) frames; unlike the reference's driver it does not trim that count to a
multiple of batch_size, since the editor takes a short last keyframe group (INTEGRATION.md §6).

Frames are read from `data_path` as %05d.png, else %05d.jpg (util.load_imgs), with PIL; video containers are out of
scope.  `--controlnet_dir` adds a Canny ControlNet to both stages.  Under torchrun every process edits on its local
GPU (`LOCAL_RANK`): frames are sharded over the ranks and the all-gathers run through `ops.Communicator`; rank 0 writes
the files.  With `--device cpu` the processes run on the CPU and gather over gloo.
"""
from __future__ import annotations

import argparse
import glob
import os
import re
import sys
from pathlib import Path
from typing import List, Optional

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
        p.add_argument("--controlnet_dir", default=None, help="diffusers ControlNet directory (Canny)")
        p.add_argument("--variant", default=None, help="weights variant, e.g. fp16")
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


def _run(args, world: int, rank: int, comm, device: torch.device) -> None:
    import yaml
    from . import pipeline
    from .util import add_dict_to_yaml_file, seed_everything
    dtype = torch.float16 if device.type == "cuda" else torch.float32
    parts = pipeline.load_parts(args.model_dir, device, dtype, args.controlnet_dir, args.variant)
    dist_kw = dict(world_size=world, rank=rank, comm=comm)

    if args.stage == "preprocess":
        seed_everything(1)                                                   # preprocess.py:303
        frames = read_frames(args.data_path, args.n_frames)
        _, recon = pipeline.preprocess(parts, frames, args, **dist_kw)
        if rank == 0:
            add_dict_to_yaml_file(os.path.join(args.save_dir, "inversion_prompts.yaml"), Path(args.data_path).stem,
                                  args.inversion_prompt)
            write_frames(recon, os.path.join(pipeline.latents_dir(args, frames.shape[0]), "frames"))
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
    out = pipeline.edit(parts, frames, config, source, **dist_kw)
    if rank == 0:
        os.makedirs(config["output_path"], exist_ok=True)
        with open(os.path.join(config["output_path"], "config.yaml"), "w") as f:
            yaml.dump(config, f)
        write_frames(out, os.path.join(config["output_path"], "img_ode"))


if __name__ == "__main__":
    main(sys.argv[1:])
