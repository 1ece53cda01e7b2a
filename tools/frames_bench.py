"""Frame resizing and the non-square edit step on one GPU.

    python tools/frames_bench.py [--frames 40] [--steps 10] [--rounds 3] [--out FILE]

Resize: ms per frame of `tf_resize_u8` (CUDA events over 20 calls on 40 frames already on the device) for 1920 x 1080
-> 672 x 384 and -> 512 x 512, with GB/s of the algorithmic bytes (input read, intermediate written and read, output
written), next to PIL's `Image.resize(LANCZOS)` of the same frames on the host: one thread, and a thread pool of one
worker per core (Pillow releases the GIL while it resamples).  Every device result is compared with PIL's, bytes equal.

Edit step: the C2 workload (SD1.5, 40 frames, B = 8, 50-step PnP, random-init fp16 UNet in channels_last, fused pass,
CUDA-graphed step) at 384 x 672 (48 x 84 latents) and at 512 x 512 (64 x 64), in one process, alternated over
rounds: ms per denoising step and frames/s of the 50-step edit.  The card's name, power limit and SM clock are read
by nvidia-smi before and after.  One JSON line at the end.
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

RESIZES = {"1080p_to_672x384": ((1080, 1920), (384, 672)), "1080p_to_512x512": ((1080, 1920), (512, 512))}
EDITS = {"384x672": (48, 84), "512x512": 64}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--steps", type=int, default=10, help="timed denoising steps per round and shape")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from PIL import Image
    import bench
    from vae_bench import card
    from tokenflow_b200 import ops as tf_ops

    assert torch.cuda.is_available(), "frames_bench.py needs a GPU"
    torch.cuda.set_device(0)
    torch.backends.cudnn.benchmark = True
    ops = tf_ops.default_ops()
    result = {"card_before": card(), "frames": args.frames, "host_cores": os.cpu_count(), "resize": {}, "edit": {}}

    # -- resize ---------------------------------------------------------------------------------------------------
    rng = np.random.default_rng(0)
    for name, ((h_in, w_in), (h, w)) in RESIZES.items():
        host = rng.integers(0, 256, (args.frames, h_in, w_in, 3), dtype=np.uint8)
        dev = torch.from_numpy(host).cuda()
        tmp = torch.empty((args.frames, h_in, w, 3), dtype=torch.uint8, device="cuda")
        out = torch.empty((args.frames, h, w, 3), dtype=torch.uint8, device="cuda")
        for _ in range(3):
            ops.resize_frames(dev, (h, w), tmp=tmp, out=out)
        reps = 20
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            ops.resize_frames(dev, (h, w), tmp=tmp, out=out)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        nbytes = 3.0 * args.frames * (h_in * w_in + 2 * h_in * w + h * w)

        pil_one = lambda f: np.asarray(Image.fromarray(f).resize((w, h), Image.LANCZOS))
        t0 = time.perf_counter()
        want = np.stack([pil_one(f) for f in host])
        pil_1 = (time.perf_counter() - t0) * 1e3
        with ThreadPoolExecutor(os.cpu_count()) as pool:
            list(pool.map(pil_one, host[:os.cpu_count()]))                       # start the workers
            t0 = time.perf_counter()
            pooled = np.stack(list(pool.map(pil_one, host)))
            pil_n = (time.perf_counter() - t0) * 1e3
        assert np.array_equal(pooled, want)
        equal = bool(np.array_equal(out.cpu().numpy(), want))
        result["resize"][name] = {
            "in": [h_in, w_in], "out": [h, w], "tf_resize_u8_ms_per_frame": round(ms / args.frames, 4),
            "tf_resize_u8_GB_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1),
            "pil_1_thread_ms_per_frame": round(pil_1 / args.frames, 3),
            "pil_pool_ms_per_frame": round(pil_n / args.frames, 3), "bit_equal_to_pil": equal}
        print(f"{name}: {result['resize'][name]}")
        assert equal, f"{name}: tf_resize_u8 differs from PIL"
        del dev, tmp, out

    # -- the C2 edit step at 384 x 672 and 512 x 512 --------------------------------------------------------------
    from tokenflow_b200 import sd_unet
    editors = {}
    for name, latent in EDITS.items():                 # one UNet per editor: the hooks live on its modules
        unet = sd_unet.build_unet("sd15", seed=1, device="cuda", dtype=torch.float16, init_on_device=True)
        bench.CONFIGS[f"frames_bench_{name}"] = dict(bench.CONFIGS["C2"], latent=latent)
        ed, x, _ = bench.build_editor("cuda", f"frames_bench_{name}", unet=unet.to(memory_format=torch.channels_last))
        for i in range(3):                                                    # capture all three step variants
            ed.step_index(x, [0, 30, 45][i])
        editors[name] = (ed, x)
    torch.cuda.synchronize()
    times = {n: [] for n in EDITS}
    for r in range(args.rounds):
        for name in (list(EDITS) if r % 2 == 0 else list(EDITS)[::-1]):
            ed, x = editors[name]
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            y = x
            for i in range(args.steps):
                y = ed.step_index(y, i * 50 // args.steps)
            e1.record()
            torch.cuda.synchronize()
            assert torch.isfinite(y).all()
            times[name].append(e0.elapsed_time(e1) / args.steps)
    n_steps = bench.CONFIGS["C2"]["n_steps"]
    for name in EDITS:
        med = statistics.median(times[name])
        result["edit"][name] = {"ms_per_step": round(med, 2), "ms_per_step_all_rounds": [round(t, 2) for t in times[name]],
                                "frames_per_s": round(bench.CONFIGS["C2"]["n_frames"] / (med * n_steps / 1e3), 3)}
        print(f"edit {name}: {result['edit'][name]}")
    result["card_after"] = card()
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
