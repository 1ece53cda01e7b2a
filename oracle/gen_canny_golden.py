"""ORACLE (test infrastructure) — tests/golden/canny.pt: `cv2.Canny`'s own edge maps of seeded frames, so that the GPU
tests check `tf_canny_u8` against OpenCV without OpenCV on the GPU machine.

The frames are not stored: `case_frames(case)` makes them again from the case's seed with integer numpy operations
only (the same bytes on every machine), and the golden holds the edges as packed bits.

    python -m oracle.gen_canny_golden          # rewrites tests/golden/canny.pt (needs cv2)
"""
from __future__ import annotations

import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "canny.pt")

# name: (kind, n, h, w, low, high, seed)
CASES = {
    "noise_1x37x53": ("noise", 1, 37, 53, 100, 200, 1),
    "smooth_40x64x96": ("smooth", 40, 64, 96, 100, 200, 2),
    "smooth_2x384x672": ("smooth", 2, 384, 672, 100, 200, 3),
    "smooth_1x512x512": ("smooth", 1, 512, 512, 100, 200, 4),
    "smooth_3x97x131_swapped": ("smooth", 3, 97, 131, 180.5, 60.25, 5),
    "checker_2x40x72": ("checker", 2, 40, 72, 50, 120, 6),
    "lines_1x160x160": ("lines", 1, 160, 160, 100, 200, 7),
    "ties_1x48x80": ("ties", 1, 48, 80, 30, 90, 8),
    "flat_1x33x17": ("flat", 1, 33, 17, 100, 200, 9),
    "tiny_1x1x1": ("noise", 1, 1, 1, 0, 0, 10),
    "thin_1x3x300": ("smooth", 1, 3, 300, 20, 40, 11),
}


def _box(img: np.ndarray, r: int) -> np.ndarray:
    """Integer box mean over (2r+1)^2 with edge padding, per channel (floor division)."""
    p = np.pad(img.astype(np.int64), ((r, r), (r, r), (0, 0)), mode="edge")
    c = p.cumsum(0).cumsum(1)
    c = np.pad(c, ((1, 0), (1, 0), (0, 0)))
    k = 2 * r + 1
    h, w = img.shape[:2]
    s = c[k:k + h, k:k + w] - c[0:h, k:k + w] - c[k:k + h, 0:w] + c[0:h, 0:w]
    return (s // (k * k)).astype(np.uint8)


def make_frame(kind: str, h: int, w: int, rng: np.random.Generator) -> np.ndarray:
    yy, xx = np.mgrid[0:h, 0:w]
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "smooth":                  # blobs at several scales: edges of every orientation and strength
        coarse = rng.integers(0, 256, ((h + 7) // 8, (w + 7) // 8, 3), dtype=np.uint8)
        up = np.repeat(np.repeat(coarse, 8, 0), 8, 1)[:h, :w]
        return _box(up, 2)
    if kind == "checker":
        cell = int(rng.integers(3, 9))
        v = (((xx // cell) + (yy // cell)) % 2 * 200 + 20).astype(np.uint8)
        return np.stack([v, 255 - v, v // 2], -1)
    if kind == "lines":                   # one-pixel lines through the centre at 5-degree steps
        img = np.zeros((h, w, 3), dtype=np.uint8)
        cy, cx = h // 2, w // 2
        for a in range(0, 180, 5):
            t = np.arange(-min(h, w) // 2 + 2, min(h, w) // 2 - 2)
            ys = np.clip(cy + np.round(t * np.sin(np.deg2rad(a))).astype(int), 0, h - 1)
            xs = np.clip(cx + np.round(t * np.cos(np.deg2rad(a))).astype(int), 0, w - 1)
            img[ys, xs] = (255, 128 + a // 2, 255 - a)
        return img
    if kind == "ties":                    # the same gradient in every channel, and channel-permuted steps
        v = ((xx // 6 + yy // 5) % 4 * 60).astype(np.uint8)
        g = np.stack([v, v, v], -1)
        g[h // 2:, :, 1] = g[h // 2:, :, 0][:, ::-1]
        return g
    if kind == "flat":
        return np.full((h, w, 3), int(rng.integers(0, 256)), dtype=np.uint8)
    raise ValueError(kind)


def case_frames(name: str) -> np.ndarray:
    kind, n, h, w, _, _, seed = CASES[name]
    rng = np.random.default_rng(seed)
    return np.stack([make_frame(kind, h, w, rng) for _ in range(n)])


def serpentine(h: int, w: int, pitch: int = 10, width: int = 4):
    """One band winding over the whole frame: horizontal runs `pitch` rows apart joined at alternating ends, value 60
    on 0, and brighter (200) over its first pixels.  With thresholds between the plain band's gradient (240) and the
    bright part's (100 and 500), every edge pixel but those of the bright start is only a candidate, so hysteresis must
    carry the edge along the whole band."""
    img = np.zeros((h, w), dtype=np.uint8)
    rows = list(range(3, h - width - 2, pitch))
    for k, y in enumerate(rows):
        img[y:y + width, 3:w - 3] = 60
        if k + 1 < len(rows):
            x = w - 3 - width if k % 2 == 0 else 3
            img[y:rows[k + 1] + width, x:x + width] = 60
    img[rows[0]:rows[0] + width, 3:3 + 2 * width] = 200
    return np.stack([img] * 3, -1)


def unpack(bits: np.ndarray, shape) -> np.ndarray:
    n = int(np.prod(shape))
    return (np.unpackbits(bits)[:n].reshape(shape) * 255).astype(np.uint8)


def main():
    import cv2
    import torch
    out = {}
    for name, (kind, n, h, w, low, high, seed) in CASES.items():
        frames = case_frames(name)
        edges = np.stack([cv2.Canny(f, low, high) for f in frames])
        out[name] = {"shape": (n, h, w), "low": low, "high": high,
                     "edges_bits": torch.from_numpy(np.packbits(edges > 0))}
    out["_opencv"] = cv2.__version__
    torch.save(out, GOLDEN)
    print(f"wrote {GOLDEN}: {len(CASES)} cases, OpenCV {cv2.__version__}")


if __name__ == "__main__":
    main()
