"""The v-prediction step against the eps step on one GPU.

    python tools/vpred_bench.py [--frames 40] [--steps 10] [--rounds 3] [--out FILE]

Kernel: ms per call of `tf_cfg_ddim_v` and `tf_cfg_ddim` (CUDA events over 200 calls) on the C2 (40 x 4 x 64 x 64)
and C4 (40 x 4 x 96 x 96) latents, alternated over rounds, with GB/s of the algorithmic bytes (three fp16 reads and
one fp16 write per latent element).  Each v call is checked bit for bit against the v scheduler's eager step.

Edit step: the C4 workload (SD2.1, 40 frames at 768 x 768, B = 8, SDEdit, random-init fp16 UNet in channels_last,
fused pass, CUDA-graphed step) with an eps and a v scheduler, alternated over rounds of `--steps` steps: ms per
denoising step.  The card's name, power limit and SM clock are read by nvidia-smi before and after.  One JSON line at
the end.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import types

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))


def _coef_row(sch, row, device):
    from tokenflow_b200.editor import TokenFlowEditor
    stub = types.SimpleNamespace(scheduler=sch, _t_host=[int(t) for t in sch.timesteps], device=device)
    return TokenFlowEditor._make_coef_table(stub)[row]


def kernel_section(ops, n_frames, rounds, result):
    import torch
    from tokenflow_b200.scheduler import DDIMScheduler
    reps = 200
    for name, lat in (("C2", 64), ("C4", 96)):
        g = torch.Generator(device="cuda").manual_seed(0)
        u, c, x = (torch.randn(n_frames, 4, lat, lat, device="cuda", generator=g).half() for _ in range(3))
        out = torch.empty_like(x)
        arms = {}
        for kind, fn in (("epsilon", ops.cfg_ddim), ("v_prediction", ops.cfg_ddim_v)):
            sch = DDIMScheduler(prediction_type=kind)
            sch.set_timesteps(50)
            coef = _coef_row(sch, 20, torch.device("cuda"))
            fn(u, c, x, coef, 7.5, out=out)
            want = sch.step(u + 7.5 * (c - u), int(sch.timesteps[20]), x)["prev_sample"]
            assert torch.equal(out, want), f"{name} {kind}: the kernel differs from the eager step"
            arms[kind] = (fn, coef)
        times = {k: [] for k in arms}
        for r in range(rounds):
            for kind in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
                fn, coef = arms[kind]
                for _ in range(3):
                    fn(u, c, x, coef, 7.5, out=out)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(reps):
                    fn(u, c, x, coef, 7.5, out=out)
                e1.record()
                torch.cuda.synchronize()
                times[kind].append(e0.elapsed_time(e1) / reps)
        nbytes = 8.0 * x.numel()
        entry = {"latents": list(x.shape)}
        for kind, ts in times.items():
            ms = statistics.median(ts)
            kname = "tf_cfg_ddim_v" if kind == "v_prediction" else "tf_cfg_ddim"
            entry[kname] = {"ms": round(ms, 5), "ms_all_rounds": [round(t, 5) for t in ts],
                            "GB_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1)}
        result["kernel"][name] = entry
        print(f"kernel {name}: {entry}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--steps", type=int, default=10, help="timed denoising steps per round and arm")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import bench
    from vae_bench import card
    from tokenflow_b200 import ops as tf_ops
    from tokenflow_b200 import sd_unet, tokenflow_utils as tfu
    from tokenflow_b200.editor import TokenFlowEditor, synthetic_inputs
    from tokenflow_b200.scheduler import DDIMScheduler

    assert torch.cuda.is_available(), "vpred_bench.py needs a GPU"
    torch.cuda.set_device(0)
    torch.backends.cudnn.benchmark = True
    tfu._install_ops_for_testing(None)
    ops = tf_ops.default_ops()
    result = {"card_before": card(), "kernel": {}, "edit": {}}
    kernel_section(ops, args.frames, args.rounds, result)

    # -- the C4 edit step with an eps and a v scheduler --------------------------------------------------------------
    c = bench.CONFIGS["C4"]
    n, lat = args.frames, c["latent"]
    arms = {}
    for kind in ("epsilon", "v_prediction"):       # one UNet per editor: the hooks live on its modules
        unet = sd_unet.build_unet(c["kind"], seed=1, device="cuda", dtype=torch.float16, init_on_device=True)
        unet = unet.to(memory_format=torch.channels_last)
        cfg = {"n_frames": n, "batch_size": c["batch"], "n_timesteps": c["n_timesteps"], "guidance_scale": 7.5,
               "mode": c["mode"], "start": 0.9, "fused_pass": True, "cuda_graph": True, "keyframe_seed": 1}
        x, text, pnp, src = synthetic_inputs(n, lat, unet.config.cross_attention_dim, c["n_timesteps"], seed=1,
                                             device="cuda", dtype=torch.float16)
        ed = TokenFlowEditor(unet, DDIMScheduler(prediction_type=kind), tfu, cfg, text, pnp,
                             source_latents=lambda t, s=src: s[t])
        ed.init_method()
        ed.step_index(x, 0)                        # capture (SDEdit: one step variant)
        arms[kind] = (ed, x)
    torch.cuda.synchronize()
    times = {a: [] for a in arms}
    for r in range(args.rounds):
        for kind in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
            ed, x = arms[kind]
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            y = x
            for i in range(args.steps):
                y = ed.step_index(y, i * len(ed._t_host) // args.steps)
            e1.record()
            torch.cuda.synchronize()
            assert torch.isfinite(y).all()
            times[kind].append(e0.elapsed_time(e1) / args.steps)
    for kind in arms:
        med = statistics.median(times[kind])
        result["edit"][kind] = {"ms_per_step": round(med, 2), "ms_per_step_all_rounds": [round(t, 2) for t in times[kind]]}
        print(f"edit {kind}: {result['edit'][kind]}")
    result["workload"] = (f"C4: SD2.1, {n} frames at {8 * lat}^2, B = {c['batch']}, SDEdit, random-init fp16 UNet, "
                          "channels_last, fused CUDA-graphed step; kernels on C2 and C4 latents of as many frames")
    result["card_after"] = card()
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
