"""Encode and decode time of the VAE stage on one GPU: three arms of the same random-init SD VAE, in one process,
alternated over rounds.

    python tools/vae_bench.py [--configs C2,C4] [--frames 40] [--batch 10] [--rounds 3] [--out FILE]

C2 is SD1.5's 512^2 frames, C4 SD2.1's 768^2 (the VAE is the same).  Arms:
  native   fp16 channels_last; GroupNorm(+SiLU) on tf_group_norm_nhwc, pixels on
           tf_frames_to_nhwc / tf_nhwc_to_frames (`preprocess.encode_imgs` / `decode_latents`)
  aten_cl  the same model and calls with ATen's GroupNorm (NCHW-only: it copies around every norm)
  nchw     the same weights in NCHW, ATen's GroupNorm
Per config it prints the median ms per frame of encode (uint8 frames on the host -> latents) and decode (latents ->
uint8 frames on the device) per arm, kernel time per category of one profiled encode + decode per arm (the categories
of tools/prof_body.py; the `sdpa` entry names the attention backend that ran), the algorithmic bytes per second of
the 4-channels-per-group tf_group_norm_nhwc calls, timed as tf_group_norm_g4 (3 passes of 2 bytes an element over
CUDA-event time of each call), and the card's name, power limit
and SM clock read by nvidia-smi before and after the measurement.
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import statistics
import subprocess
import sys
from unittest import mock

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))

SIDES = {"C2": 512, "C4": 768}
ARMS = ("native", "aten_cl", "nchw")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,temperature.gpu"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable: {e}"
    return dict(zip(q.split(","), [v.strip() for v in out.split(",")])) if "," in out else {"raw": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C2,C4")
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--batch", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from torch.autograd import DeviceType
    from prof_body import categorize
    from tokenflow_b200 import ops as tf_ops
    from tokenflow_b200.preprocess import decode_latents, encode_imgs
    from tokenflow_b200.vae import build_vae

    assert torch.cuda.is_available(), "vae_bench.py needs a GPU"
    torch.cuda.set_device(0)
    torch.backends.cudnn.benchmark = True
    ops = tf_ops.default_ops()
    vae = build_vae("sd", seed=1, device="cuda", dtype=torch.float16, init_on_device=True)
    models = {"native": vae.to(memory_format=torch.channels_last)}
    models["aten_cl"] = models["native"]
    models["nchw"] = copy.deepcopy(vae).to(memory_format=torch.contiguous_format)

    def arm_ctx(arm):
        # the ATen arms: norm_act finds no library ops and runs the eager GroupNorm (+ SiLU)
        return mock.patch.object(tf_ops, "_BODY_OPS", None) if arm != "native" else mock.patch.object(
            tf_ops, "_BODY_OPS", ops)

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return out, e0.elapsed_time(e1)

    result = {"card_before": card(), "frames": args.frames, "batch": args.batch, "rounds": args.rounds, "configs": {}}
    for cfg in args.configs.split(","):
        side = SIDES[cfg]
        g = torch.Generator().manual_seed(0)
        frames = torch.randint(0, 256, (args.frames, side, side, 3), dtype=torch.uint8, generator=g)
        latents = (torch.randn(args.frames, 4, side // 8, side // 8, generator=g) * 0.9).half().cuda()
        times = {a: {"encode": [], "decode": []} for a in ARMS}
        outs = {}
        with torch.no_grad():
            for a in ARMS:                                       # warm-up: cuDNN algorithm choice, allocator growth
                with arm_ctx(a):
                    encode_imgs(models[a], frames[:args.batch], batch_size=args.batch)
                    decode_latents(models[a], latents[:args.batch], batch_size=args.batch)
            for r in range(args.rounds):
                for a in (ARMS if r % 2 == 0 else ARMS[::-1]):
                    with arm_ctx(a):
                        lat, ms_e = timed(lambda: encode_imgs(models[a], frames, batch_size=args.batch))
                        img, ms_d = timed(lambda: decode_latents(models[a], latents, batch_size=args.batch))
                    times[a]["encode"].append(ms_e / args.frames)
                    times[a]["decode"].append(ms_d / args.frames)
                    outs[a] = (lat, img)
            # kernel time per category: one profiled encode + decode of one batch per arm
            profile = {}
            for a in ARMS:
                with arm_ctx(a), torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    encode_imgs(models[a], frames[:args.batch], batch_size=args.batch)
                    decode_latents(models[a], latents[:args.batch], batch_size=args.batch)
                    torch.cuda.synchronize()
                cats = {}
                for ev in prof.events():
                    if ev.device_type != DeviceType.CUDA:
                        continue
                    c = cats.setdefault(categorize(ev.name), {"ms": 0.0, "launches": 0, "top": {}})
                    c["ms"] += ev.time_range.elapsed_us() / 1e3
                    c["launches"] += 1
                    c["top"][ev.name[:120]] = c["top"].get(ev.name[:120], 0.0) + ev.time_range.elapsed_us() / 1e3
                profile[a] = {k: {"ms": round(v["ms"], 3), "launches": v["launches"],
                                  "top": sorted(((n, round(t, 3)) for n, t in v["top"].items()), key=lambda kv: -kv[1])[:3]}
                              for k, v in sorted(cats.items(), key=lambda kv: -kv[1]["ms"])}
            # tf_group_norm_g4 rate: CUDA events around each call of one native encode + decode
            ops.enable_timing(True)
            with arm_ctx("native"):
                encode_imgs(models["native"], frames[:args.batch], batch_size=args.batch)
                decode_latents(models["native"], latents[:args.batch], batch_size=args.batch)
            kt = ops.timing_summary()
            ops.enable_timing(False)
        g4 = kt.get("tf_group_norm_g4", {"ms": 0.0, "work": 0.0, "launches": 0})
        med = {a: {k: round(statistics.median(v), 3) for k, v in times[a].items()} for a in ARMS}
        diff = {a: {"latents_max_abs_vs_native": (outs[a][0].float() - outs["native"][0].float()).abs().max().item(),
                    "frames_max_abs_vs_native": (outs[a][1].int() - outs["native"][1].int()).abs().max().item()}
                for a in ARMS if a != "native"}
        result["configs"][cfg] = {
            "side": side, "ms_per_frame": med, "ms_per_frame_all_rounds": times, "outputs": diff,
            "kernel_ms_by_category": profile,
            "tf_group_norm_g4": {"calls": g4["launches"], "ms": round(g4["ms"], 3),
                                 "TB_per_s": round(g4["work"] / g4["ms"] / 1e9, 3) if g4["ms"] else None},
            "library_kernels_ms": {k: round(v["ms"], 3) for k, v in kt.items()}}
        print(f"{cfg} ({side}^2, {args.frames} frames, batches of {args.batch}):")
        for a in ARMS:
            print(f"  {a:8s} encode {med[a]['encode']:8.3f} ms/frame   decode {med[a]['decode']:8.3f} ms/frame")
        print(f"  tf_group_norm_g4: {result['configs'][cfg]['tf_group_norm_g4']}")
        for a in ARMS:
            print(f"  {a} kernel ms: " + ", ".join(f"{k} {v['ms']:.1f}" for k, v in profile[a].items()))
        print(f"  sdpa kernels: {profile['native'].get('sdpa', {}).get('top')}")
    result["card_after"] = card()
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)
    print(json.dumps({"card_before": result["card_before"], "card_after": result["card_after"],
                      **{c: v["ms_per_frame"] for c, v in result["configs"].items()}}))


if __name__ == "__main__":
    main()
