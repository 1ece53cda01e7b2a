"""Time the inversion stage (reference preprocess.py:198-284) on one GPU and print one JSON line.

    python tools/invert_bench.py [--config C2|C4] [--steps 24] [--warmup 3] [--rounds 3] [--batch B] [--no-full]
                                 [--out FILE]

Two arms run in the same process on the same UNet and latents, alternated round by round, each timed over
`--steps` inversion steps of the reference's 500-step grid after `--warmup` untimed steps:
  * oracle_eager   the reference's loop as oracle/inversion.py restates it (eager fp16 UNet, SDPA attn1, ATen
                   elementwise DDIM update per batch): what the stage costs without the graphed path;
  * graph_sdpa     the graphed path (`LatentInverter` on a CUDA fp16 UNet), attn1 on SDPA.
Reported per arm: the median over rounds of ms per step.  Then, unless --no-full, one full run of the stage as the
reference runs it (500 inversion steps saving the 50 sampling timesteps, then 500 reconstruction steps, graph capture
included): its wall time, frames/s of the stage, and the reconstruction's relative L2 against the input latents.  The
GPU's name, power limit and median SM clock over the timed regions are read in the same call.

The graphed arm keeps its captured step next to the eager arm's memory; the C4 figures in README.md were taken with
--batch 20 (two UNet calls per step).

Workloads (random-init UNet fp16 channels_last, synthetic N(0,1) latents, the reference's batch size 40):
  C2  40 frames, 512 x 512 (64 x 64 latents), SD1.5
  C4  40 frames, 768 x 768 (96 x 96 latents), SD2.1"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

CONFIGS = {"C2": dict(kind="sd15", n_frames=40, latent=64, batch=40),
           "C4": dict(kind="sd21", n_frames=40, latent=96, batch=40)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C2", choices=sorted(CONFIGS))
    ap.add_argument("--steps", type=int, default=24, help="timed inversion steps per arm and round")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=None, help="frames per UNet call (default: the config's, 40)")
    ap.add_argument("--no-full", action="store_true", help="skip the full 500 + 500 run")
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, repo)

    import torch
    from bench import ClockSampler
    from oracle import inversion as OI
    from tokenflow_b200 import sd_unet
    from tokenflow_b200.preprocess import LatentInverter
    from tokenflow_b200.scheduler import DDIMScheduler

    assert torch.cuda.is_available(), "invert_bench.py needs a GPU"
    c = CONFIGS[args.config]
    dev = torch.device("cuda")
    unet = sd_unet.build_unet(c["kind"], seed=1, device=dev, dtype=torch.float16, init_on_device=True)
    unet = unet.to(memory_format=torch.channels_last)
    g = torch.Generator().manual_seed(1)
    x0 = torch.randn(c["n_frames"], 4, c["latent"], c["latent"], generator=g).half().to(dev)
    cond = torch.randn(1, 77, unet.config.cross_attention_dim, generator=g).half().to(dev)
    B, K, W = args.batch or c["batch"], args.steps, args.warmup

    sch = DDIMScheduler()
    sch.set_timesteps(500)

    def oracle_arm(n):
        OI.ddim_inversion(unet, sch, cond, x0.clone(), B, timesteps_to_save=[], n_steps=n)

    graph_inv = LatentInverter(unet, DDIMScheduler(), 500)
    coef, _, ts_up, _ = graph_inv._device_tables()

    def graph_arm(n):
        graph_inv._run_steps(x0, cond, B, coef[:n], ts_up[:n])

    arms = {"oracle_eager": oracle_arm, "graph_sdpa": graph_arm}
    times = {name: [] for name in arms}
    clocks = ClockSampler(0)
    for name, fn in arms.items():                # warm-up: cuDNN / cuBLAS choices, graph capture
        fn(W)
    torch.cuda.synchronize()
    clocks.start()
    for _ in range(args.rounds):
        for name, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn(K)
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3 / K)
    res = {"config": args.config, "workload": f"{c['n_frames']} frames, {c['latent'] * 8}^2, "
           f"{'SD1.5' if c['kind'] == 'sd15' else 'SD2.1'}, batch {B}, random-init UNet fp16 channels_last",
           "steps_per_arm": K, "rounds": args.rounds,
           "ms_per_step": {k: statistics.median(v) for k, v in times.items()},
           "ms_per_step_all": times}

    if not args.no_full:
        torch.cuda.empty_cache()
        toy = DDIMScheduler()
        toy.set_timesteps(50)
        inv = LatentInverter(unet, DDIMScheduler(), 500)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        xT = inv.ddim_inversion(cond, x0, None, B, timesteps_to_save=toy.timesteps.tolist())
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        rec = inv.ddim_sample(xT, cond, B)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        res["full"] = {"inversion_s": t1 - t0, "reconstruction_s": t2 - t1, "stage_s": t2 - t0,
                       "frames_per_s": c["n_frames"] / (t2 - t0), "saved_timesteps": len(inv.saved_latents()),
                       "recon_rel_l2": ((rec.double() - x0.double()).norm() / x0.double().norm()).item(),
                       "finite": bool(torch.isfinite(rec).all())}
    res["clocks"] = clocks.stop()
    res["gpu"] = torch.cuda.get_device_name(0)
    try:
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        res["power_limit"] = None
    text = json.dumps(res)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
