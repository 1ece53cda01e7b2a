"""Extended-attention micro-benchmark + accuracy check for one shape (CUDA events, L2 flushed).
Usage: python tools/attn_bench.py [--S 4096 --dim 320 --heads 8 --n 5 --inject 0] [--tag name]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tokenflow_b200.ops import CudaOps  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--S", type=int, default=4096)
    ap.add_argument("--dim", type=int, default=320)
    ap.add_argument("--heads", type=int, default=8)
    ap.add_argument("--n", type=int, default=5)
    ap.add_argument("--inject", type=int, default=0)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--tag", default="")
    ap.add_argument("--video-like", type=int, default=1, help="keys correlated with queries (peaked softmax rows)")
    args = ap.parse_args()
    ops = CudaOps()
    S, dim, heads, n = args.S, args.dim, args.heads, args.n
    d = dim // heads
    torch.manual_seed(0)
    q = torch.randn(3 * n, S, dim, device="cuda")
    k = torch.randn(3 * n, S, dim, device="cuda")
    if args.video_like:                 # some keys resemble their query: rows with a few dominant probabilities
        k = k + 1.5 * q
    v = torch.randn(3 * n, S, dim, device="cuda")
    q, k, v = q.half(), k.half(), v.half()
    scale = d ** -0.5
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    fn = lambda: ops.ext_attn(q, k, v, heads, scale, bool(args.inject))
    for _ in range(3):
        out = fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(args.iters):
        flush.zero_()
        flush[::64].sum()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    # accuracy: fp32 softmax reference for sampled (sample, head) slabs, all S query rows
    errs = []
    for (smp, head) in ((0, 0), (n, 1), (2 * n + n - 1, heads - 1), (n + 1, heads // 2)):
        s_, f_ = divmod(smp, n)
        qs = (f_ if (args.inject and s_ > 0) else smp)
        qq = q[qs, :, head * d:(head + 1) * d].float()
        if s_ == 0:
            kk = k[smp, :, head * d:(head + 1) * d].float()
            vv = v[smp, :, head * d:(head + 1) * d].float()
        else:
            k0 = 0 if args.inject else s_ * n
            kk = k[k0:k0 + n, :, head * d:(head + 1) * d].reshape(n * S, d).float()
            vv = v[s_ * n:(s_ + 1) * n, :, head * d:(head + 1) * d].reshape(n * S, d).float()
        ref = torch.softmax(qq @ kk.T * scale, dim=-1) @ vv
        errs.append((out[smp, :, head * d:(head + 1) * d].float() - ref).abs().max().item())
    flops = 4.0 * n * S * S * dim * (2 * n + 1)
    med = ts[len(ts) // 2]
    rec = {"tag": args.tag, "S": S, "d": d, "n": n, "inject": args.inject, "ms": round(med, 4), "best_ms": round(ts[0], 4),
           "tflops": round(flops / med / 1e9, 1), "max_err": max(errs)}
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
