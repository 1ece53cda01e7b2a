"""Video files in: the package's one decode loop.

Decoding is FFmpeg's, through OpenCV (`cv2.VideoCapture`), on the host: the H100 has NVDEC engines, but the CUDA
toolkit ships no NVDEC headers, so frames come off the host decoder as BGR bytes and are converted to RGB there.  The
per-pixel work after decoding, the Lanczos resize to the size the edit runs at, is `preprocess.resize_frames`: on a
CUDA device that is `tf_resize_u8`, bit for bit PIL's `Image.resize(..., LANCZOS)`, which is what runs on the CPU.

Frames are decoded in chunks and each chunk is resized as soon as it is complete, so only the resized frames are kept:
a long 1080p video never sits in host memory at its full size.  (The reference's `save_video_frames` holds the whole
decoded video.)

Rotation follows the container's display matrix, which OpenCV applies by default (`CAP_PROP_ORIENTATION_AUTO`): a
phone video recorded upright comes out upright.  The reference instead rotates every `.mov` file by -90 degrees
(util.py:21-22), a workaround for torchvision's decoder ignoring that matrix; `read_video` does not.
`util.save_video_frames` keeps the reference's rotation for the reference's scripts.
"""
from __future__ import annotations

from typing import Iterator, Optional, Tuple, Union

import numpy as np
import torch


def decoded_chunks(path: str, chunk: int = 64) -> Tuple[float, Iterator[torch.Tensor]]:
    """(fps, chunks): the container's frame rate and an iterator of uint8 RGB host frames [<= chunk, H, W, 3] of
    `path`, in decode order, at the decoded (display-rotated) size.  The frames are counted by decoding them, not
    taken from the container's frame count.  Raises ValueError naming the path when OpenCV cannot open it."""
    import cv2
    if chunk < 1:
        raise ValueError(f"chunk must be at least 1, got {chunk}")
    cap = cv2.VideoCapture(path)
    if not cap.isOpened():
        cap.release()
        raise ValueError(f"cannot open {path!r} as a video")
    fps = float(cap.get(cv2.CAP_PROP_FPS))

    def chunks():
        try:
            buf = []
            while True:
                ok, frame = cap.read()
                if not ok:
                    break
                buf.append(cv2.cvtColor(frame, cv2.COLOR_BGR2RGB))
                if len(buf) == chunk:
                    yield torch.from_numpy(np.stack(buf))
                    buf = []
            if buf:
                yield torch.from_numpy(np.stack(buf))
        finally:
            cap.release()

    return fps, chunks()


def read_video(path: str, size: Optional[Union[int, Tuple[int, int]]] = None, device="cpu",
               chunk: int = 64) -> Tuple[torch.Tensor, float]:
    """Every frame of the video file `path` -> (uint8 RGB frames [N, H, W, 3] on the host, fps).

    With `size` ((H, W), or an int for a square, as `preprocess.resize_frames` takes it) each chunk of `chunk`
    decoded frames is moved to `device`, resized there by `resize_frames` and brought back, and only the resized
    frames are kept; the result does not depend on `chunk` or `device`.  Without it the frames keep their decoded
    size.  Raises ValueError naming the path when the file does not open or yields no frames."""
    from .preprocess import resize_frames
    fps, chunks = decoded_chunks(path, chunk)
    device = torch.device(device)
    out = [c if size is None else resize_frames(c.to(device), size).cpu() for c in chunks]
    if not out:
        raise ValueError(f"{path!r} has no frames that decode")
    return torch.cat(out), fps
