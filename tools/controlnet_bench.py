"""Canny edges and the ControlNet-conditioned stages on one GPU.

    python tools/controlnet_bench.py [--frames 40] [--steps 10] [--inv-steps 10] [--rounds 3] [--out FILE]

Canny: ms per frame of `tf_canny_u8` writing the fp16 conditioning (CUDA events over 20 calls on 40 frames already on
the device) at 512 x 512 and 384 x 672, with GB/s of the algorithmic bytes (the uint8 frames read, the fp16
[N, 3, H, W] conditioning written), next to `cv2.Canny` of the same frames on the host: one thread (OpenCV's own
threading off), and a thread pool of one worker per core.  The device edges are compared with cv2's (or, where cv2
is not installed, with oracle/canny.py), bytes equal.

Edit step: the C2 workload (SD1.5, 40 frames, B = 8, 50-step PnP, random-init fp16 UNet and ControlNet in
channels_last, fused pass, CUDA-graphed step) with and without the ControlNet, alternated over rounds: ms per
denoising step.  Inversion: ms per graph-replayed step of the inversion stage (40 frames at 512 x 512 in one UNet
call per step), with and without the ControlNet, alternated likewise.  The card's name, power limit and SM clock are
read by nvidia-smi before and after.  One JSON line at the end.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time
from concurrent.futures import ThreadPoolExecutor

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))

SIZES = {"512x512": (512, 512), "384x672": (384, 672)}


def canny_section(ops, n_frames, result):
    import numpy as np
    import torch
    from oracle import canny as oc
    from oracle import gen_canny_golden as gg
    try:
        import cv2
    except ImportError:
        cv2 = None
    rng = np.random.default_rng(0)
    for name, (h, w) in SIZES.items():
        host = np.stack([gg.make_frame("smooth", h, w, rng) for _ in range(n_frames)])
        dev = torch.from_numpy(host).cuda()
        cond = torch.empty((n_frames, 3, h, w), dtype=torch.float16, device="cuda", memory_format=torch.channels_last)
        for _ in range(3):
            ops.canny(dev, edges=False, out_cond=cond)
        reps = 20
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            ops.canny(dev, edges=False, out_cond=cond)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        nbytes = (3.0 + 6.0) * n_frames * h * w
        edges = ops.canny(dev, cond=False)[0].cpu().numpy()
        entry = {"frames": n_frames, "size": [h, w], "tf_canny_u8_ms_per_frame": round(ms / n_frames, 4),
                 "tf_canny_u8_GB_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1)}
        if cv2 is not None:
            cv2.setNumThreads(1)
            one = lambda f: cv2.Canny(f, 100, 200)
            t0 = time.perf_counter()
            want = np.stack([one(f) for f in host])
            entry["cv2_1_thread_ms_per_frame"] = round((time.perf_counter() - t0) * 1e3 / n_frames, 3)
            with ThreadPoolExecutor(os.cpu_count()) as pool:
                list(pool.map(one, host[:os.cpu_count()]))
                t0 = time.perf_counter()
                pooled = np.stack(list(pool.map(one, host)))
                entry["cv2_pool_ms_per_frame"] = round((time.perf_counter() - t0) * 1e3 / n_frames, 3)
            assert np.array_equal(pooled, want)
            entry["bit_equal_to"] = "cv2"
        else:
            want = oc.canny_frames(host, 100, 200)
            entry["cv2_1_thread_ms_per_frame"] = entry["cv2_pool_ms_per_frame"] = "not measured (no cv2)"
            entry["bit_equal_to"] = "oracle/canny.py"
        entry["bit_equal"] = bool(np.array_equal(edges, want))
        result["canny"][name] = entry
        print(f"canny {name}: {entry}")
        assert entry["bit_equal"], f"{name}: tf_canny_u8 differs"
        del dev, cond


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--steps", type=int, default=10, help="timed denoising steps per round and arm")
    ap.add_argument("--inv-steps", type=int, default=10, help="timed inversion steps per round and arm")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import bench
    from vae_bench import card
    from tokenflow_b200 import ops as tf_ops
    from tokenflow_b200 import preprocess, sd_unet, tokenflow_utils as tfu
    from tokenflow_b200.controlnet import build_controlnet
    from tokenflow_b200.editor import TokenFlowEditor, synthetic_inputs
    from tokenflow_b200.scheduler import DDIMScheduler

    assert torch.cuda.is_available(), "controlnet_bench.py needs a GPU"
    torch.cuda.set_device(0)
    torch.backends.cudnn.benchmark = True
    ops = tf_ops.default_ops()
    result = {"card_before": card(), "host_cores": os.cpu_count(), "canny": {}, "edit": {}, "inversion": {}}
    canny_section(ops, args.frames, result)

    # -- the C2 edit step with and without the ControlNet -------------------------------------------------------------
    import numpy as np
    from oracle import gen_canny_golden as gg
    c = bench.CONFIGS["C2"]
    n, lat = c["n_frames"], c["latent"]
    rng = np.random.default_rng(1)
    frames = torch.from_numpy(np.stack([gg.make_frame("smooth", 8 * lat, 8 * lat, rng) for _ in range(n)])).cuda()
    ccond = preprocess.canny_cond(frames)
    cn = build_controlnet("sd15", seed=3, device="cuda", dtype=torch.float16).to(memory_format=torch.channels_last)
    arms = {}
    for arm in ("plain", "controlnet"):            # one UNet per editor: the hooks live on its modules
        unet = sd_unet.build_unet("sd15", seed=1, device="cuda", dtype=torch.float16, init_on_device=True)
        unet = unet.to(memory_format=torch.channels_last)
        cfg = {"n_frames": n, "batch_size": c["batch"], "n_timesteps": c["n_timesteps"], "guidance_scale": 7.5,
               "mode": c["mode"], "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "fused_pass": True, "cuda_graph": True,
               "keyframe_seed": 1}
        x, text, pnp, src = synthetic_inputs(n, lat, unet.config.cross_attention_dim, c["n_timesteps"], seed=1,
                                             device="cuda", dtype=torch.float16)
        ed = TokenFlowEditor(unet, DDIMScheduler(), tfu, cfg, text, pnp, source_latents=lambda t, s=src: s[t],
                             controlnet=cn if arm == "controlnet" else None,
                             controlnet_cond=ccond if arm == "controlnet" else None)
        ed.init_method()
        for i in (0, 30, 45):                      # capture all three step variants
            ed.step_index(x, i)
        arms[arm] = (ed, x, unet)
    torch.cuda.synchronize()
    times = {a: [] for a in arms}
    for r in range(args.rounds):
        for arm in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
            ed, x, _ = arms[arm]
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            y = x
            for i in range(args.steps):
                y = ed.step_index(y, i * 50 // args.steps)
            e1.record()
            torch.cuda.synchronize()
            assert torch.isfinite(y).all()
            times[arm].append(e0.elapsed_time(e1) / args.steps)
    for arm in arms:
        med = statistics.median(times[arm])
        result["edit"][arm] = {"ms_per_step": round(med, 2), "ms_per_step_all_rounds": [round(t, 2) for t in times[arm]],
                               "frames_per_s": round(n / (med * c["n_steps"] / 1e3), 3)}
        print(f"edit {arm}: {result['edit'][arm]}")
    del arms, ed, unet
    torch.cuda.empty_cache()
    # a UNet without the TokenFlow hooks: the inversion runs the plain SD UNet
    unet = sd_unet.build_unet("sd15", seed=1, device="cuda", dtype=torch.float16, init_on_device=True)
    unet = unet.to(memory_format=torch.channels_last)

    # -- inversion steps with and without the ControlNet ----------------------------------------------------------------
    g = torch.Generator().manual_seed(1)
    x0 = torch.randn(n, 4, lat, lat, generator=g).half().cuda()
    cond = torch.randn(1, 77, unet.config.cross_attention_dim, generator=g).half().cuda()
    invs = {"plain": preprocess.LatentInverter(unet, DDIMScheduler(), 500),
            "controlnet": preprocess.LatentInverter(unet, DDIMScheduler(), 500, controlnet=cn, controlnet_cond=ccond)}
    K = args.inv_steps
    for inv in invs.values():
        coef, _, ts_up, _ = inv._device_tables()
        inv._run_steps(x0, cond, n, coef[:3], ts_up[:3])              # capture and warm up
    torch.cuda.synchronize()
    itimes = {a: [] for a in invs}
    for r in range(args.rounds):
        for arm in (list(invs) if r % 2 == 0 else list(invs)[::-1]):
            inv = invs[arm]
            coef, _, ts_up, _ = inv._device_tables()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            inv._run_steps(x0, cond, n, coef[:K], ts_up[:K])
            torch.cuda.synchronize()
            itimes[arm].append((time.perf_counter() - t0) * 1e3 / K)
    for arm in invs:
        result["inversion"][arm] = {"ms_per_step": round(statistics.median(itimes[arm]), 2),
                                    "ms_per_step_all_rounds": [round(t, 2) for t in itimes[arm]]}
        print(f"inversion {arm}: {result['inversion'][arm]}")
    result["workload"] = (f"C2: SD1.5, {n} frames at {8 * lat}^2, B = {c['batch']}, PnP, random-init fp16 UNet and "
                          "ControlNet, channels_last; inversion: one UNet call of 40 frames per step")
    result["card_after"] = card()
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
