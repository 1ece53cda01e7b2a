"""Long videos on one GPU: peak memory and step time of the graphed edit step by frame count and frames_per_pass.

    python tools/long_video_bench.py [--steps 2] [--rounds 3] [--out FILE]

Workloads (random-init fp16 UNets in channels_last, synthetic latents, fused CUDA-graphed step, SDEdit):
  * SD2.1 at 768 x 768 (96 x 96 latents) with the v-prediction scheduler, B = 8, N in {40, 80, 120, 160, 200}, with
    frames_per_pass unset (one UNet call over all frames) and 40 and 16 (frame chunks);
  * SD1.5 at 512 x 512, N = 200 frames, B = 16: every frame, against the 192 frames bench.py's C5s16 edits.

Per point: `torch.cuda.max_memory_allocated` after `reset_peak_memory_stats`, once over the first step (warm-up and
graph capture included) and once over the steady-state steps, and `max_memory_reserved` over the first step (what the
process holds: the graph's private pool keeps the capture's blocks); ms per step, the median of `--rounds` rounds of
`--steps` replayed steps.  The rounds of one point run back to back: two graphed steps at 768 x 768 and many frames do
not fit on the card together, so points are not alternated.  Chunks of at least N frames are the unchunked step and are
not run again.

The GPU may be shared, so no point is allowed to find the card's limit by allocating: before each point the peak is
extrapolated linearly in N from the points of the same arm already measured (reserved memory), and a point whose
estimate, plus 10 %, exceeds the memory `torch.cuda.mem_get_info` reports free (plus what this process holds) is
recorded as "not run" with the estimate.  The card's name, power limit and SM clock are read by nvidia-smi before and after.  One
JSON line at the end.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))

GB = 2 ** 30


def _estimate(measured, n):
    """Peak bytes at n frames from the (frames, peak) points already measured: the line through the last two, or
    proportional scaling from one; None without any."""
    if not measured:
        return None
    if len(measured) == 1:
        n0, p0 = measured[0]
        return p0 * n / n0
    (n0, p0), (n1, p1) = measured[-2], measured[-1]
    return p1 + (p1 - p0) * (n - n1) / (n1 - n0)


def run_point(kind, kind_cfg, n, chunk, steps, rounds):
    import torch
    from tokenflow_b200 import sd_unet, tokenflow_utils as tfu
    from tokenflow_b200.editor import TokenFlowEditor, synthetic_inputs
    from tokenflow_b200.scheduler import DDIMScheduler
    lat, batch, n_timesteps = kind_cfg["latent"], kind_cfg["batch"], kind_cfg["n_timesteps"]
    cfg = {"n_frames": n, "batch_size": batch, "n_timesteps": n_timesteps, "guidance_scale": 7.5, "mode": "sdedit",
           "start": 0.9, "fused_pass": True, "cuda_graph": True, "keyframe_seed": 1}
    if chunk is not None:
        cfg["frames_per_pass"] = chunk
    # a UNet per point: the blocks keep their last keyframe caches, which would keep the previous graph's pool alive
    unet = sd_unet.build_unet(kind, seed=1, device="cuda", dtype=torch.float16, init_on_device=True)
    unet = unet.to(memory_format=torch.channels_last)
    x, text, pnp, src = synthetic_inputs(n, lat, unet.config.cross_attention_dim, n_timesteps, seed=1, device="cuda",
                                         dtype=torch.float16)
    ed = TokenFlowEditor(unet, DDIMScheduler(prediction_type=kind_cfg["prediction"]), tfu, cfg, text, pnp,
                         source_latents=lambda t: src[t])
    ed.init_method()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    y = ed.step_index(x, 0)                                  # warm-up + capture + first replay (SDEdit: one variant)
    torch.cuda.synchronize()
    peak_capture = torch.cuda.max_memory_allocated()
    reserved_capture = torch.cuda.max_memory_reserved()
    torch.cuda.reset_peak_memory_stats()
    times = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(steps):
            y = ed.step_index(y, 1 + i)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / steps)
    assert torch.isfinite(y).all()
    peak_steady = torch.cuda.max_memory_allocated()
    calls = len(ed._frame_chunks(0, n))
    del ed, x, y, src, unet
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return {"peak_GB_capture": round(peak_capture / GB, 2), "peak_GB_steady": round(peak_steady / GB, 2),
            "reserved_GB_capture": round(reserved_capture / GB, 2),
            "ms_per_step": round(statistics.median(times), 1), "ms_per_step_all_rounds": [round(t, 1) for t in times],
            "unet_calls_per_step": calls, "frames_per_s": round(n * 1000.0 / statistics.median(times), 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2, help="replayed steps per round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", default="40,80,120,160,200", help="SD2.1 frame counts")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from vae_bench import card
    from tokenflow_b200 import tokenflow_utils as tfu

    assert torch.cuda.is_available(), "long_video_bench.py needs a GPU"
    torch.cuda.set_device(0)
    torch.backends.cudnn.benchmark = True
    tfu._install_ops_for_testing(None)
    result = {"card_before": card(), "points": []}
    workloads = [
        ("sd21", dict(latent=96, batch=8, n_timesteps=50, prediction="v_prediction"),
         [int(v) for v in args.frames.split(",")], (None, 40, 16)),
        ("sd15", dict(latent=64, batch=16, n_timesteps=50, prediction="epsilon"), [192, 200], (None,)),
    ]
    for kind, kcfg, frames, chunks in workloads:
        measured = {c: [] for c in chunks}
        for n in frames:
            for chunk in chunks:
                point = {"model": kind, "px": 8 * kcfg["latent"], "B": kcfg["batch"], "frames": n,
                         "frames_per_pass": "all" if chunk is None else chunk}
                if chunk is not None and chunk >= n:
                    point["not_run"] = "same as all"
                    result["points"].append(point)
                    continue
                est = _estimate(measured[chunk], n)
                free, _ = torch.cuda.mem_get_info()
                have = torch.cuda.memory_reserved()
                if est is not None and 1.1 * est > free + have:          # a 10 % margin on the estimate
                    point["not_run"] = f"needs ~{est / GB:.1f} GB, {(free + have) / GB:.1f} GB free"
                else:
                    try:
                        point.update(run_point(kind, kcfg, n, chunk, args.steps, args.rounds))
                        measured[chunk].append((n, point["reserved_GB_capture"] * GB))
                    except torch.cuda.OutOfMemoryError as e:  # the estimate was short: record it, free, go on
                        guess = "none" if est is None else f"{est / GB:.1f} GB"
                        point["not_run"] = f"out of memory (estimate {guess}): {str(e)[:120]}"
                        torch.cuda.empty_cache()
                result["points"].append(point)
                print(json.dumps(point), flush=True)
    result["card_after"] = card()
    result["workload"] = ("random-init fp16 UNets in channels_last, synthetic latents, SDEdit (start 0.9), fused "
                          "CUDA-graphed step; SD2.1 with the v-prediction scheduler")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(json.dumps(result, indent=1))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
