"""ORACLE (test infrastructure) — tests/golden/canny.pt and canny_probes.pt: `cv2.Canny`'s own edge maps of seeded
frames, so that the GPU tests check `tf_canny_u8` against OpenCV without OpenCV on the GPU machine.

The frames are not stored: `case_frames(case)` makes them again from the case's seed with integer numpy operations
only (the same bytes on every machine), and the golden holds the edges as packed bits.  canny.pt holds `CASES`;
canny_probes.pt holds `PROBE_CASES`, the hysteresis probes at 512 x 512 and a 1080p frame.  A case once written never
changes: the generator refuses to rewrite an existing entry with other bits.

    python -m oracle.gen_canny_golden          # rewrites both files (needs cv2)
"""
from __future__ import annotations

import os

import numpy as np

_GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
GOLDEN = os.path.join(_GOLDEN_DIR, "canny.pt")
PROBE_GOLDEN = os.path.join(_GOLDEN_DIR, "canny_probes.pt")

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

# the same form, in canny_probes.pt
PROBE_CASES = {
    "hysteresis_8x512x512": ("hysteresis", 8, 512, 512, 100, 500, 12),
    "smooth_1x1080x1920": ("smooth", 1, 1080, 1920, 100, 200, 13),
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


def make_frame(kind: str, h: int, w: int, rng: np.random.Generator, index: int = 0) -> np.ndarray:
    """Frame `index` of a case of `kind`; only "hysteresis" frames depend on the index."""
    if kind == "hysteresis":              # the hysteresis probes in turn, turned by 180 degrees from the fifth on
        probes = (dense, comb, serpentine, lambda h, w: rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        img = probes[index % 4](h, w)
        return np.ascontiguousarray(img[::-1, ::-1]) if (index // 4) % 2 else img
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
    kind, n, h, w, _, _, seed = {**CASES, **PROBE_CASES}[name]
    rng = np.random.default_rng(seed)
    return np.stack([make_frame(kind, h, w, rng, i) for i in range(n)])


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


def dense(h: int, w: int) -> np.ndarray:
    """Two thirds of the pixels candidates, all in one 8-connected component over the whole frame: a 3 x 3 tile whose
    non-suppressed magnitudes lie in [120, 420], and one bright pixel near the last corner (placed where it joins the
    component at every frame size), whose neighbourhood holds the only strong pixels at thresholds (100, 500).
    Hysteresis has to carry the edge from the frame's last tile to its first pixel, and every candidate of the frame
    links to one root."""
    tile = np.array([[60, 90, 90], [30, 60, 0], [90, 90, 60]], dtype=np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    img = tile[yy % 3, xx % 3]
    img[max(h - 4, 0), max(w - 5, 0)] = 255
    return np.stack([img] * 3, -1)


def comb(h: int, w: int, pitch: int = 10, width: int = 4) -> np.ndarray:
    """Vertical teeth of value 60 on 0, `pitch` columns apart, joined only by a bar along the last rows, and brighter
    (200) at the top of the first tooth: at thresholds (100, 500) the edge must run down the first tooth, along the
    bar and up every other one; above the bar each tooth is a component of its own."""
    img = np.zeros((h, w), dtype=np.uint8)
    bar = h - 3 - width
    for x in range(3, w - width - 2, pitch):
        img[3:bar, x:x + width] = 60
    img[bar:bar + width, 3:w - 3] = 60
    img[3:3 + 2 * width, 3:3 + width] = 200
    return np.stack([img] * 3, -1)


def unpack(bits: np.ndarray, shape) -> np.ndarray:
    n = int(np.prod(shape))
    return (np.unpackbits(bits)[:n].reshape(shape) * 255).astype(np.uint8)


def _write(path, cases):
    import cv2
    import torch
    old = torch.load(path, weights_only=False) if os.path.exists(path) else {}
    out = {}
    for name, (kind, n, h, w, low, high, seed) in cases.items():
        frames = case_frames(name)
        edges = np.stack([cv2.Canny(f, low, high) for f in frames])
        out[name] = {"shape": (n, h, w), "low": low, "high": high,
                     "edges_bits": torch.from_numpy(np.packbits(edges > 0))}
        if name in old:                   # a case once written never changes
            assert old[name]["shape"] == (n, h, w) and (old[name]["low"], old[name]["high"]) == (low, high), name
            assert torch.equal(old[name]["edges_bits"], out[name]["edges_bits"]), name
    out["_opencv"] = cv2.__version__
    torch.save(out, path)
    print(f"wrote {path}: {len(cases)} cases, OpenCV {cv2.__version__}")


def main():
    _write(GOLDEN, CASES)
    _write(PROBE_GOLDEN, PROBE_CASES)


if __name__ == "__main__":
    main()
