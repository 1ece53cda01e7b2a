"""ORACLE (test infrastructure) — the launch shapes of the frame-preparation kernels, and the cases that reach them.

`resize_layout` restates how tf_resize.cu's launch_resize_h / launch_resize_v shape their launches (rows staged per
block, opt-in shared memory, 16- or 4-byte columns, column blocks, grid sizes), so that a CPU test can check that the
GPU cases below reach every branch.  `canny_threshold_classes` names what tf_capi.cu's tf_canny_u8 does with a
threshold pair: swap, floor, clamp to [-1, 2040].
"""
from __future__ import annotations

import math

RESIZE_V_THREADS = 128
RESIZE_DEFAULT_SMEM = 48 * 1024          # bytes of dynamic shared memory a launch gets without opting in
RESIZE_MAX_SMEM = 227 * 1024             # opt-in shared memory per block on sm_90
MAX_GRID = 2 ** 31 - 1                   # blocks of one 1-D launch
CANNY_MAX_MAG = 2040                     # 4 * 255 * 2: the largest L1 Sobel magnitude of a uint8 frame


def resize_h_rows(w_in: int) -> int:
    """Input rows one horizontal-pass block stages in shared memory: as many as fit in 48 KB, 1 to 4."""
    return min(max(RESIZE_DEFAULT_SMEM // (3 * w_in + 16), 1), 4)


def resize_layout(n: int, h_in: int, w_in: int, h: int, w: int, in_off: int = 0, tmp_off: int = 0,
                  out_off: int = 0) -> dict:
    """The launches of tf_resize_u8 for n frames [h_in, w_in, 3] -> [h, w, 3] whose input, intermediate and output
    start `*_off` bytes past a 16-byte boundary.  "h" / "v" is None for a pass the call skips, else:
      v_first: the vertical pass goes first (into tmp [n, h, w_in, 3]), see resize_v_first
      h: rows (input rows per block), smem (bytes), opt_in (smem past the default 48 KB), grid (blocks)
      v: vec (bytes per thread, 16 when the row pitch and the pass's input and output are 16-byte aligned),
         col_blocks (blocks of 128 threads per output row), grid (blocks)."""
    need_h, need_v = w != w_in, h != h_in
    v_first = resize_v_first(h_in, w_in, h, w)
    out = {"h": None, "v": None, "v_first": v_first}
    if need_h:
        rows = resize_h_rows(w_in)
        smem = rows * 3 * w_in + 16
        rows_in = h if v_first else h_in
        out["h"] = {"rows": rows, "smem": smem, "opt_in": smem > RESIZE_DEFAULT_SMEM, "grid": -(-n * rows_in // rows)}
    if need_v:
        src_off, dst_off = (in_off, tmp_off) if v_first else (tmp_off if need_h else in_off, out_off)
        pitch = 3 * (w_in if v_first else w)
        vec = 16 if pitch % 16 == 0 and src_off % 16 == 0 and dst_off % 16 == 0 else 4
        col_blocks = -(-pitch // (RESIZE_V_THREADS * vec))
        out["v"] = {"vec": vec, "col_blocks": col_blocks, "grid": n * h * col_blocks}
    return out


def resize_v_first(h_in: int, w_in: int, h: int, w: int) -> bool:
    """Both passes, the vertical one first: Pillow's Image.resize takes a frame more than 100 times taller than wide
    whose height shrinks through a vertical-only resize to (w_in, h), then a horizontal-only one."""
    return w != w_in and h != h_in and h_in > 100 * w_in and h < h_in


def resize_h_class(layout: dict):
    """(rows, opt_in) of the horizontal pass, or None."""
    return None if layout["h"] is None else (layout["h"]["rows"], layout["h"]["opt_in"])


def resize_v_class(layout: dict):
    """(vec, more than one column block) of the vertical pass, or None."""
    return None if layout["v"] is None else (layout["v"]["vec"], layout["v"]["col_blocks"] > 1)


# Widths where the horizontal pass changes class: the last width of one class and the first of the next.
RESIZE_H_BOUNDARIES = [(4090, 4091), (5456, 5457), (8186, 8187), (16378, 16379)]
RESIZE_H_CLASSES = [(rows, False) for rows in (4, 3, 2, 1)] + [(1, True)]
RESIZE_V_CLASSES = [(vec, several) for vec in (4, 16) for several in (False, True)]

# ---------------------------------------------------------------------------------------------------------------------
# GPU cases of tests/test_gpu_frame_prep.py, here so that the CPU tier can check what they reach
# ---------------------------------------------------------------------------------------------------------------------
# Horizontal classes: 2 frames a few rows high (odd row counts leave the last block part full), (h_in, w_in) -> (h, w).
RESIZE_ROWS_CASES = [
    ((5, 4090), (3, 1021)), ((5, 4091), (3, 1021)),
    ((5, 4096), (3, 1024)),                              # DCI 4K
    ((5, 5456), (3, 1363)), ((5, 5457), (3, 1364)),
    ((3, 7680), (2, 1920)),                              # 8K UHD
    ((3, 8186), (2, 2047)), ((3, 8187), (2, 2047)),
    ((3, 16378), (2, 4093)), ((3, 16379), (2, 4095)),
    ((3, 65536), (2, 16384)),                            # the widest input the library takes
    ((3, 16384), (3, 512)),                              # opt-in, horizontal pass only
]
# 16-byte columns with 1, 2 and 3 column blocks per output row, aligned tmp / out; then the 4-byte path at those
# widths, and the column-block boundary 3w = 2048 (w = 672 | 688).
RESIZE_VEC_CASES = [
    ((1080, 1920), (672, 672), 0), ((1080, 1920), (768, 768), 0), ((720, 1280), (1080, 1920), 0),
    ((97, 700), (61, 688), 0), ((97, 700), (61, 688), 3), ((65, 99), (31, 160), 5),
]
# Large-tap downscales and the exact 3x ratios (the Lanczos argument lands on 0 and on the x < 3 edge); the frames
# 4096 x 5 and 65536 x 7 are more than 100 times taller than wide, which Pillow resizes vertically first.
RESIZE_RATIO_CASES = [
    ((3, 65536), (2, 7)), ((4096, 5), (3, 4)), ((5, 4096), (4, 3)), ((3, 16384), (2, 1)),
    ((9, 3), (27, 9)), ((27, 9), (9, 3)), ((9, 27), (3, 9)), ((768, 1024), (1024, 768)), ((1024, 768), (768, 1024)),
    ((65536, 7), (2, 3)), ((4096, 5), (41, 9)), ((8192, 2), (8000, 7)), ((500, 5), (100, 4)), ((501, 5), (100, 4)),
]
# One size per vertical path (16-byte when aligned, 4-byte always), at every (in, tmp, out) byte offset.
RESIZE_OFFSETS = [0, 1, 8, 15]
RESIZE_OFFSET_SIZES = [((97, 700), (61, 688)), ((45, 80), (24, 42))]


def resize_gpu_layouts():
    """(case, layout) of every launch tests/test_gpu_frame_prep.py makes, 2 frames each (the frame count does not
    change a class)."""
    out = []
    for src, dst in RESIZE_ROWS_CASES + RESIZE_RATIO_CASES:
        out.append(((src, dst, 0), resize_layout(2, *src, *dst)))
    for src, dst, off in RESIZE_VEC_CASES:
        out.append(((src, dst, off), resize_layout(2, *src, *dst, tmp_off=off, out_off=off)))
    for src, dst in RESIZE_OFFSET_SIZES:
        for a in RESIZE_OFFSETS:
            for t in RESIZE_OFFSETS:
                for o in RESIZE_OFFSETS:
                    out.append(((src, dst, (a, t, o)), resize_layout(2, *src, *dst, a, t, o)))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# Canny thresholds
# ---------------------------------------------------------------------------------------------------------------------
def canny_threshold_classes(low: float, high: float) -> set:
    """What tf_canny_u8 does with (low, high): "swapped" (low > high), "fractional" (a threshold is no integer),
    "equal" (one value after the floor), "below" (a threshold under 0: clamped to -1, every non-suppressed pixel
    passes it), "above" (over 2040: clamped, no magnitude passes it), "inside" (both in [0, 2040])."""
    tags = set()
    if low > high:
        tags.add("swapped")
    if low != math.floor(low) or high != math.floor(high):
        tags.add("fractional")
    lo, hi = sorted((math.floor(low), math.floor(high)))
    if lo == hi:
        tags.add("equal")
    if lo < 0:
        tags.add("below")
    if hi > CANNY_MAX_MAG:
        tags.add("above")
    if 0 <= lo and hi <= CANNY_MAX_MAG:
        tags.add("inside")
    return tags


CANNY_THRESHOLD_CLASSES = ["below", "inside", "above", "equal", "swapped", "fractional"]
CANNY_THRESHOLDS = [(100, 200), (-5, 60), (-300, -20), (40, 2100), (2100, 5000), (2040, 2040), (120, 120),
                    (200.9, 200.2), (200, 100), (50.7, 120.2), (-0.5, 0.5), (0, 0)]
