"""How far the native UNet body moves the C2 edit, against a GroupNorm-rounding noise floor (oracle/body_drift.py).

    python tools/body_drift.py [--frames 40] [--batch 8] [--steps 8] [--kind sd15] [--latent 64] [--out FILE]

Runs the same seeded PnP edit for `--steps` steps in four arms (native channels_last body, ATen channels_last
body, ATen NCHW body, ATen channels_last body with fp32 GroupNorm statistics) and prints one JSON line: the
pairwise relative L2 differences of the final latents, the GPU's name and power limit.  The defaults are the C2 workload (40 frames, B = 8, SD1.5 at a 64 x 64 latent)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kind", default="sd15")
    ap.add_argument("--latent", type=int, default=64)
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

    import torch
    from oracle.body_drift import body_drift

    assert torch.cuda.is_available(), "body_drift.py needs a GPU"
    res = body_drift(args.kind, n_frames=args.frames, batch=args.batch, latent=args.latent, steps=args.steps)
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
