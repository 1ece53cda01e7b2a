"""Kernel time of one warmed-up C2 step, per category, under torch.profiler (CUDA activities).

    python tools/prof_body.py [--config C2] [--repo DIR] [--out FILE]

Builds the editor the way bench.py does (eager, no CUDA graph, channels_last UNet), runs `--warmup` steps, then
profiles one step and writes a JSON summary: milliseconds and launches per category of kernel (layout copies,
GroupNorm, SiLU, GELU, elementwise mul/add/div, cat, conv, GEMM, SDPA, LayerNorm, the library's `tf::` kernels,
other), the ten most expensive kernel names of each category, and the step time measured with CUDA events in
an unprofiled step just before.  `--repo` imports bench.py and the package from another checkout of this
project (to profile two versions with the same tool)."""
from __future__ import annotations

import argparse
import json
import os
import re
import sys

# first match wins: cat / layer_norm / group_norm kernels contain "copy" or "norm" in other categories' patterns
CATEGORIES = [
    ("tf", r"\btf::"),
    ("group_norm", r"GroupNorm|RowwiseMoments|ComputeFusedParams|group_norm"),
    ("layer_norm", r"LayerNorm|layer_norm"),
    ("cat", r"CatArray|cat_"),
    ("copy", r"copy|Copy"),
    ("silu", r"silu|SiLU"),
    ("gelu", r"[Gg]elu"),
    ("upsample", r"upsample"),
    ("conv", r"conv|fprop|dgrad|implicit|nhwc|nchw|NHWC|NCHW|Winograd|winograd|cudnn"),
    ("mul", r"MulFunctor|mul_kernel"),
    ("add", r"Functor_add|AddFunctor|add_kernel"),
    ("div", r"DivFunctor|div_kernel"),
    ("sdpa", r"flash|fmha|[Aa]ttention|efficient_attention"),
    ("gemm", r"gemm|Gemm|GEMM|nvjet|cutlass|xmma|cublas|Kernel2"),
]


def categorize(name: str) -> str:
    for cat, pat in CATEGORIES:
        if re.search(pat, name):
            return cat
    return "other"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C2")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repo", default=None, help="checkout to import bench.py / tokenflow_b200 from (default: this one)")
    ap.add_argument("--out", default=None, help="write the JSON here (default: stdout only)")
    args = ap.parse_args()
    repo = os.path.abspath(args.repo) if args.repo else os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, repo)

    import torch
    from torch.autograd import DeviceType
    import bench
    from tokenflow_b200 import tokenflow_utils as tfu

    assert torch.cuda.is_available(), "prof_body.py needs a GPU"
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    tfu._ops()
    torch.backends.cudnn.benchmark = True
    ed, x, _ = bench.build_editor(device, args.config, cuda_graph=False)
    for i in range(args.warmup):
        x = ed.step_index(x, i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    x = ed.step_index(x, args.warmup)
    e1.record()
    torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1)

    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        x = ed.step_index(x, args.warmup + 1)
        torch.cuda.synchronize()

    cats = {}
    for ev in prof.events():
        if ev.device_type != DeviceType.CUDA:
            continue
        us = ev.time_range.elapsed_us()
        c = cats.setdefault(categorize(ev.name), {"ms": 0.0, "launches": 0, "kernels": {}})
        c["ms"] += us / 1e3
        c["launches"] += 1
        c["kernels"][ev.name] = c["kernels"].get(ev.name, 0.0) + us / 1e3
    total = sum(c["ms"] for c in cats.values())
    summary = {}
    for name, c in sorted(cats.items(), key=lambda kv: -kv[1]["ms"]):
        top = sorted(c["kernels"].items(), key=lambda kv: -kv[1])[:10]
        summary[name] = {"ms": round(c["ms"], 3), "share": round(c["ms"] / total, 4), "launches": c["launches"],
                         "top": [[k[:160], round(v, 3)] for k, v in top]}
    out = {"config": args.config, "repo": repo, "gpu": torch.cuda.get_device_name(device),
           "step_ms_unprofiled_eager": round(step_ms, 2), "kernel_ms_total": round(total, 2),
           "launches_total": sum(c["launches"] for c in cats.values()), "categories": summary}
    text = json.dumps(out, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)
    print(json.dumps({k: v for k, v in out.items() if k != "categories"}))
    for name, c in summary.items():
        print(f"{name:12s} {c['ms']:9.2f} ms {100 * c['share']:5.1f} % {c['launches']:6d} launches")


if __name__ == "__main__":
    main()
