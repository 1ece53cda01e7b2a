"""What a LoRA costs: reading and merging it at load time, and the edit step after the merge.

    python tools/lora_bench.py [--ranks 32 128] [--rounds 3] [--steps 10] [--out FILE]

A synthetic SD1.5 checkpoint (random-init fp16 UNet and VAE, a random text encoder of CLIP ViT-L/14's size) is written
to a temporary directory, and for each rank a random kohya LoRA (fp16 safetensors, `synthetic_checkpoint.write_lora`)
at kohya's full target set: the 192 Transformer2DModel modules, the 72 CLIPAttention / CLIPMLP modules of the text
encoder and LoCon's ResnetBlock2D / Downsample2D / Upsample2D convolutions.  Timed, each the median of `--rounds`
after one warm-up: `pipeline.load_parts` of the checkpoint (the load a LoRA adds to), and `lora.merge` of each file
into the loaded CUDA fp16 channels_last parts (the file read included), each ending in a device synchronise.

Then the C2 edit step (SD1.5, 40 frames at 512², B = 8, PnP, CUDA-graphed) on the base UNet and on a UNet with the
rank-128 LoRA merged, alternated over the rounds in one process: ms per step.  The merge changes weight values only,
so the two should cost the same.  GPU name, power limit and SM clock are read with nvidia-smi before and after.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import statistics
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", type=int, nargs="+", default=[32, 128])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10, help="timed denoising steps per round and arm")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import bench
    from vae_bench import card
    from tokenflow_b200 import lora, pipeline, tokenflow_utils as tfu
    from tokenflow_b200 import synthetic_checkpoint as fx
    from tokenflow_b200.editor import TokenFlowEditor, synthetic_inputs
    from tokenflow_b200.scheduler import DDIMScheduler

    assert torch.cuda.is_available(), "lora_bench.py needs a GPU"
    torch.cuda.set_device(0)
    torch.backends.cudnn.benchmark = True
    result = {"card_before": card(), "load_s": None, "merge_s": {}, "edit": {}}
    targets = ("transformer", "conv", "text_encoder")
    tmp = tempfile.mkdtemp(prefix="lora_bench_")
    try:
        model_dir, _ = fx.write_checkpoint(tmp, "sd15", dtype=torch.float16, init_device="cuda",
                                           text_config=fx.CLIP_L)

        def load():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            parts = pipeline.load_parts(model_dir, "cuda", torch.float16)
            torch.cuda.synchronize()
            return parts, time.perf_counter() - t0

        load()
        loads, parts = [], None
        for _ in range(args.rounds):
            del parts
            parts, s = load()
            loads.append(s)
        result["load_s"] = round(statistics.median(loads), 3)
        print(f"load_parts: {result['load_s']} s")
        files = {}
        for rank in args.ranks:
            files[rank] = os.path.join(tmp, f"r{rank}.safetensors")
            found = fx.write_lora(files[rank], parts.unet, parts.text_encoder, "kohya", rank, targets, rank / 2, rank)
            times = []
            for i in range(args.rounds + 1):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                lora.merge(parts.unet, parts.text_encoder, [(files[rank], 0.1)])
                torch.cuda.synchronize()
                if i:
                    times.append(time.perf_counter() - t0)
            result["merge_s"][rank] = {"s": round(statistics.median(times), 3),
                                       "all_rounds": [round(t, 3) for t in times], "modules": len(found),
                                       "file_mb": round(os.path.getsize(files[rank]) / 2 ** 20, 1)}
            print(f"merge rank {rank}: {result['merge_s'][rank]}")
        del parts
        torch.cuda.empty_cache()

        c = bench.CONFIGS["C2"]
        n, lat = c["n_frames"], c["latent"]
        arms = {}
        for arm in ("base", "merged"):              # one UNet per editor: the hooks live on its modules
            p = pipeline.load_parts(model_dir, "cuda", torch.float16,
                                    loras=[(files[max(args.ranks)], 0.8)] if arm == "merged" else None)
            unet = p.unet
            del p
            cfg = {"n_frames": n, "batch_size": c["batch"], "n_timesteps": c["n_timesteps"], "guidance_scale": 7.5,
                   "mode": c["mode"], "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "fused_pass": True, "cuda_graph": True,
                   "keyframe_seed": 1}
            x, text, pnp, src = synthetic_inputs(n, lat, unet.config.cross_attention_dim, c["n_timesteps"], seed=1,
                                                 device="cuda", dtype=torch.float16)
            ed = TokenFlowEditor(unet, DDIMScheduler(), tfu, cfg, text, pnp, source_latents=lambda t, s=src: s[t])
            ed.init_method()
            for i in (0, 30, 45):                      # capture all three step variants
                ed.step_index(x, i)
            arms[arm] = (ed, x)
        torch.cuda.synchronize()
        times = {a: [] for a in arms}
        for r in range(args.rounds):
            for arm in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
                ed, x = arms[arm]
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
            result["edit"][arm] = {"ms_per_step": round(statistics.median(times[arm]), 2),
                                   "ms_per_step_all_rounds": [round(t, 2) for t in times[arm]]}
            print(f"edit {arm}: {result['edit'][arm]}")
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    result["workload"] = (f"SD1.5 fp16 channels_last, random init, CLIP ViT-L/14-sized text encoder; kohya LoRAs at "
                          f"kohya's full target set with LoCon convs; C2 edit step: {n} frames at {8 * lat}^2, "
                          f"B = {c['batch']}, PnP, graphed")
    result["card_after"] = card()
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
