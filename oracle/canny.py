"""ORACLE (test infrastructure) — OpenCV's `cv2.Canny(img, low, high)` restated in numpy for aperture 3,
`L2gradient=False` and 1- or 3-channel uint8 images (imgproc/src/canny.cpp), the edge map the reference's
ControlNet path conditions on (preprocess.py:113-127 `get_canny_cond`).

  1. 3x3 Sobel dx, dy of every channel (int16), replicated borders;
  2. per pixel the channel with the largest |dx| + |dy|, the first one on a tie;
  3. non-maximum suppression in OpenCV's integer form: tan(22.5 deg) in 15-bit fixed point decides the sector, the
     neighbour comparisons are `>` on one side and `>=` on the other for the horizontal and vertical sectors and
     `>` on both for the diagonals, and the magnitude is 0 outside the image;
  4. thresholds floor(low), floor(high) (swapped first when low > high): a pixel that survives suppression is a
     candidate when its magnitude is > low and strong when it is > high;
  5. hysteresis: the 8-connected components of candidates that contain a strong pixel are the edges (255).

`classes` returns the per-pixel class (0 none, 1 candidate, 2 strong) before hysteresis, the map the kernel's first
launch writes.
"""
from __future__ import annotations

import math

import numpy as np
from scipy import ndimage

CANNY_SHIFT = 15
TG22 = 13573           # int(tan(22.5 deg) * 2 ** 15 + 0.5)


def thresholds(low: float, high: float):
    if low > high:
        low, high = high, low
    return math.floor(low), math.floor(high)


def sobel(img: np.ndarray):
    """int32 dx, dy [h, w, c] of an [h, w, c] uint8 image with replicated borders."""
    p = np.pad(img.astype(np.int32), ((1, 1), (1, 1), (0, 0)), mode="edge")
    col = lambda x0: p[0:-2, x0:x0 + img.shape[1]] + 2 * p[1:-1, x0:x0 + img.shape[1]] + p[2:, x0:x0 + img.shape[1]]
    row = lambda y0: (p[y0:y0 + img.shape[0], 0:-2] + 2 * p[y0:y0 + img.shape[0], 1:-1]
                      + p[y0:y0 + img.shape[0], 2:])
    return col(2) - col(0), row(2) - row(0)


def gradients(img: np.ndarray):
    """(dx, dy, mag) [h, w] int32 of the channel with the largest L1 magnitude (first on ties)."""
    if img.ndim == 2:
        img = img[:, :, None]
    dx, dy = sobel(img)
    mag = np.abs(dx) + np.abs(dy)
    ch = np.argmax(mag, axis=2)[:, :, None]             # argmax returns the first maximum
    take = lambda a: np.take_along_axis(a, ch, axis=2)[:, :, 0]
    return take(dx), take(dy), take(mag)


def classes(img: np.ndarray, low: float, high: float) -> np.ndarray:
    lo, hi = thresholds(low, high)
    dx, dy, m = gradients(img)
    h, w = m.shape
    mp = np.zeros((h + 2, w + 2), dtype=np.int64)
    mp[1:-1, 1:-1] = m
    nb = lambda oy, ox: mp[1 + oy:1 + oy + h, 1 + ox:1 + ox + w]
    x = np.abs(dx).astype(np.int64)
    y = np.abs(dy).astype(np.int64) << CANNY_SHIFT
    tg22x = x * TG22
    tg67x = tg22x + (x << (CANNY_SHIFT + 1))
    s = np.where((dx ^ dy) < 0, -1, 1)
    horiz = y < tg22x
    vert = ~horiz & (y > tg67x)
    diag = ~horiz & ~vert
    keep_h = (m > nb(0, -1)) & (m >= nb(0, 1))
    keep_v = (m > nb(-1, 0)) & (m >= nb(1, 0))
    # diagonal: previous row at x - s, next row at x + s
    keep_d = np.where(s > 0, (m > nb(-1, -1)) & (m > nb(1, 1)), (m > nb(-1, 1)) & (m > nb(1, -1)))
    keep = (m > lo) & ((horiz & keep_h) | (vert & keep_v) | (diag & keep_d))
    out = np.zeros((h, w), dtype=np.uint8)
    out[keep] = 1
    out[keep & (m > hi)] = 2
    return out


def hysteresis(cls: np.ndarray) -> np.ndarray:
    labels, n = ndimage.label(cls > 0, structure=np.ones((3, 3), dtype=bool))
    strong = np.zeros(n + 1, dtype=bool)
    strong[labels[cls == 2]] = True
    strong[0] = False
    return np.where(strong[labels], 255, 0).astype(np.uint8)


def canny(img: np.ndarray, low: float, high: float) -> np.ndarray:
    """uint8 [h, w] edges (0 / 255) of a uint8 [h, w] or [h, w, c] image: `cv2.Canny(img, low, high)`."""
    return hysteresis(classes(img, low, high))


def canny_frames(frames: np.ndarray, low: float = 100, high: float = 200) -> np.ndarray:
    return np.stack([canny(f, low, high) for f in frames])


def canny_cond(edges: np.ndarray):
    """The reference's conditioning tensor from edge maps [n, h, w] (preprocess.py:122-126): the map stacked three
    times, divided by 255 in fp32, to fp16, as [n, 3, h, w]."""
    import torch
    image = np.concatenate([edges[..., None]] * 3, axis=-1)
    return torch.from_numpy(image.astype(np.float32) / 255.0).permute(0, 3, 1, 2).to(torch.float16)


def chain_span(edges: np.ndarray, start) -> tuple:
    """(rows, cols) covered by the 8-connected edge component through `start` — how far hysteresis had to reach."""
    labels, _ = ndimage.label(edges > 0, structure=np.ones((3, 3), dtype=bool))
    ys, xs = np.nonzero(labels == labels[start])
    return (int(ys.min()), int(ys.max())), (int(xs.min()), int(xs.max()))
