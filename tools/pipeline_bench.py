"""Where the time of one whole edit goes: a synthetic SD1.5 checkpoint on disk, 40 frames in, edited frames out, through
`pipeline.load_parts`, `pipeline.preprocess` and `pipeline.edit`, on one GPU.

    python tools/pipeline_bench.py [--frames 40] [--size 512] [--batch 8] [--edit-steps 50] [--inversion-steps 500]
                                   [--inversion-batch 40] [--extract-rounds 3] [--out FILE]

The defaults are one C2-sized run: 40 frames at 512², B = 8, 50-step PnP, 500 inversion (+ 500 reconstruction) steps
saving the 50 sampling timesteps.  The checkpoint (`synthetic_checkpoint.write_checkpoint`: random-init SD1.5 UNet and
VAE in fp16 safetensors under SD1.5's published configs and file names, a random text encoder of CLIP ViT-L/14's size,
SD1.5's scheduler config) is written to a temporary directory and removed afterwards; the frames are random smooth uint8
frames on the host, as if read from disk.

Each stage function the pipeline calls is wrapped with a device synchronise and a host clock before and after, so the
stages are timed inside the pipeline's own control flow: checkpoint load, text encoding, resize + encode (both stages),
Canny (none here), inversion, reconstruction, edit (the denoising loop), decode (the reconstruction and the edit).  It
prints each stage's seconds and share of the wall time, the end-to-end frames/s (frames over the wall time of load +
preprocess + edit), and the card's name, power limit and SM clock read by nvidia-smi before and after the run.  One run:
the stages are long (seconds to minutes), not a microbenchmark.

Before that run it times what `run preprocess --data_path VIDEO` does before the models load, on two synthetic 120-frame
mp4v clips written with `util.save_video` at 20 fps: one of the shape of the reference's `woman-running.mp4` (512²,
extracted at 512²) and one 1920 x 1080 clip extracted at 672 x 384.  For each clip: decoding alone (`read_video`
without a size), decode + resize on the device (`read_video(..., device="cuda")`, `tf_resize_u8`), decode + resize
with PIL (`device="cpu"`), and writing the 120 extracted frames as PNG (`run.write_frames`), the median of
`--extract-rounds` alternating rounds after one warm-up call, with the two extractions checked equal byte for byte.
Each extraction is also given as a share of a run that starts from the video: its time over itself plus the wall time
of the C2 run.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from contextlib import ExitStack
from unittest import mock

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,temperature.gpu"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable: {e}"
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")])) if "," in out else {"raw": out}


def smooth_frames(n, h, w, seed=0):
    """Random smooth uint8 frames [n, h, w, 3] on the host, made 10 at a time to bound the fp32 intermediate."""
    import torch
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(0, n, 10):
        small = torch.rand(min(10, n - i), 3, h // 16, w // 16, generator=g)
        big = torch.nn.functional.interpolate(small, size=(h, w), mode="bilinear") * 255
        out.append(big.round().to(torch.uint8).permute(0, 2, 3, 1).contiguous())
    return torch.cat(out)


def extraction(root, rounds):
    """Seconds (medians) of decoding and extracting the two 120-frame clips; see the module docstring."""
    import statistics
    import torch
    from tokenflow_b200 import run
    from tokenflow_b200.util import save_video
    from tokenflow_b200.video import read_video
    result = {}
    for name, (h, w), size in (("512x512 -> 512x512", (512, 512), (512, 512)),
                               ("1920x1080 -> 672x384", (1080, 1920), (384, 672))):
        path = os.path.join(root, "clip.mp4")
        save_video(smooth_frames(120, h, w), path, fps=20)
        calls = {"decode": lambda: read_video(path)[0], "extract_cuda": lambda: read_video(path, size, "cuda")[0],
                 "extract_cpu": lambda: read_video(path, size, "cpu")[0],
                 "write_png": lambda: run.write_frames(frames, os.path.join(root, "frames"))}
        frames = calls["extract_cuda"]()                                  # warm-up: loads the library
        assert frames.shape == (120, *size, 3) and torch.equal(frames, calls["extract_cpu"]())
        times = {k: [] for k in calls}
        for _ in range(rounds):
            for k, fn in calls.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                times[k].append(time.perf_counter() - t0)
        result[name] = {k: round(statistics.median(v), 3) for k, v in times.items()}
        os.remove(path)
    return result


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--edit-steps", type=int, default=50)
    ap.add_argument("--inversion-steps", type=int, default=500)
    ap.add_argument("--inversion-batch", type=int, default=40)
    ap.add_argument("--extract-rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from tokenflow_b200 import checkpoint, pipeline
    from tokenflow_b200 import synthetic_checkpoint as synthetic
    from tokenflow_b200.editor import TokenFlowEditor
    from tokenflow_b200.preprocess import LatentInverter

    assert torch.cuda.is_available(), "pipeline_bench.py needs a GPU"
    torch.cuda.set_device(0)
    times = {}

    def timed(stage, fn):
        def run(*a, **k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn(*a, **k)
            torch.cuda.synchronize()
            times[stage] = times.get(stage, 0.0) + time.perf_counter() - t0
            return out
        return run

    root = tempfile.mkdtemp(prefix="tf_b200_pipeline_bench_")
    try:
        model_dir, _ = synthetic.write_checkpoint(root, "sd15", dtype=torch.float16, init_device="cuda",
                                                  deprecated_vae=True, text_config=synthetic.CLIP_L)
        torch.cuda.empty_cache()
        g = torch.Generator().manual_seed(0)
        small = torch.rand(args.frames, 3, args.size // 16, args.size // 16, generator=g)
        frames = (torch.nn.functional.interpolate(small, size=(args.size, args.size), mode="bilinear") * 255).round()
        frames = frames.to(torch.uint8).permute(0, 2, 3, 1).contiguous()
        opt = {"H": args.size, "W": args.size, "steps": args.inversion_steps, "batch_size": args.inversion_batch,
               "save_steps": args.edit_steps, "inversion_prompt": "a woman running"}
        config = {"prompt": "a marble sculpture of a woman running, Venus de Milo",
                  "negative_prompt": "ugly, blurry, low res, unrealistic, unaesthetic", "guidance_scale": 7.5,
                  "n_timesteps": args.edit_steps, "batch_size": args.batch, "pnp_attn_t": 0.5, "pnp_f_t": 0.8,
                  "seed": 1, "inversion_prompt": opt["inversion_prompt"]}
        card_before = card()
        extract = extraction(root, args.extract_rounds)
        with ExitStack() as stack:
            for name, stage in (("resize_frames", "resize+encode"), ("encode_imgs", "resize+encode"),
                                ("canny_cond", "canny"), ("decode_latents", "decode")):
                stack.enter_context(mock.patch.object(pipeline, name, timed(stage, getattr(pipeline, name))))
            stack.enter_context(mock.patch.object(checkpoint, "text_embeds", timed("text", checkpoint.text_embeds)))
            stack.enter_context(mock.patch.object(LatentInverter, "ddim_inversion",
                                                  timed("inversion", LatentInverter.ddim_inversion)))
            stack.enter_context(mock.patch.object(LatentInverter, "ddim_sample",
                                                  timed("reconstruction", LatentInverter.ddim_sample)))
            stack.enter_context(mock.patch.object(TokenFlowEditor, "sample_loop",
                                                  timed("edit", TokenFlowEditor.sample_loop)))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            parts = timed("load", pipeline.load_parts)(model_dir, "cuda", torch.float16)
            t1 = time.perf_counter()
            saved, recon = pipeline.preprocess(parts, frames, opt)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            torch.manual_seed(1)
            out = pipeline.edit(parts, frames, config, saved)
            torch.cuda.synchronize()
            t3 = time.perf_counter()
        wall = t3 - t0
        times["other"] = wall - sum(times.values())
        for clip in extract.values():
            for k in ("extract_cuda", "extract_cpu"):
                clip[k + "_share_of_run_from_video"] = round(clip[k] / (clip[k] + wall), 4)
        result = {
            "card_before": card_before, "card_after": card(),
            "run": {"frames": args.frames, "size": args.size, "B": args.batch, "edit_steps": args.edit_steps,
                    "inversion_steps": args.inversion_steps, "inversion_batch": args.inversion_batch, "mode": "pnp"},
            "stage_s": {k: round(v, 3) for k, v in times.items()},
            "video_extract_120_frames_s": extract,
            "stage_share": {k: round(v / wall, 4) for k, v in times.items()},
            "wall_s": {"total": round(wall, 3), "load": round(t1 - t0, 3), "preprocess": round(t2 - t1, 3),
                       "edit": round(t3 - t2, 3)},
            "e2e_frames_per_s": round(args.frames / wall, 4),
            "edit_stage_frames_per_s": round(args.frames / (t3 - t2), 4),
            "edit_ms_per_step": round(1e3 * times["edit"] / args.edit_steps, 1),
            "inversion_ms_per_step": round(1e3 * times["inversion"] / args.inversion_steps, 1),
            "peak_allocated_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
            "outputs": {"recon": list(recon.shape), "edit": list(out.shape),
                        "edit_finite_std": float(out.float().std())},
        }
    finally:
        shutil.rmtree(root, ignore_errors=True)
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)
    print(text)


if __name__ == "__main__":
    main()
