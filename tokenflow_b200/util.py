"""Drop-in for the names the reference drivers, hooks and preprocess script import from `util`
(run_tokenflow_pnp.py:17 `save_video, seed_everything`; tokenflow_utils.py:5 `isinstance_str,
batch_cosine_sim`; preprocess.py `from util import *`: `load_imgs`, `save_video_frames`,
`add_dict_to_yaml_file`).  Video/image file I/O is host-side and out of the hot-path scope (SURVEY.md §2);
the helpers are kept, on OpenCV / PIL instead of the torchvision.io video API that torchvision 0.26 removed,
so the reference scripts import and run with this repo on sys.path.
"""
from __future__ import annotations

import random

import numpy as np
import torch


def isinstance_str(x: object, cls_name: str) -> bool:
    """True if any class in x's MRO is *named* cls_name (reference util.py:46-58): the hooks patch
    modules without importing their classes."""
    return any(c.__name__ == cls_name for c in type(x).__mro__)


def batch_cosine_sim(x, y):
    """Reference util.py:61-69.  Kept for API parity only: the TokenFlow block never materialises
    this matrix (tf_nn_field fuses normalise -> GEMM -> argmax); callers that really want the
    full matrix get the fp16 unit rows from the CUDA kernel and one library GEMM."""
    from . import tokenflow_utils as _tf

    if isinstance(x, list):
        x = torch.cat(x, dim=0)
    if isinstance(y, list):
        y = torch.cat(y, dim=0)
    ops = _tf._ops()
    return ops.unit_rows(x) @ ops.unit_rows(y).T


def seed_everything(seed: int):
    """Reference util.py:99-103."""
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed(seed)
    random.seed(seed)
    np.random.seed(seed)


def save_video(raw_frames: torch.Tensor, save_path: str, fps: int = 10):
    """Reference util.py:88-96 writes h264 through torchvision.io.write_video, which torchvision
    0.26 no longer ships; frames ([N,3,H,W] in [0,1], or uint8 [N,H,W,3] as `preprocess.decode_latents`
    returns them) are written with OpenCV instead."""
    import cv2

    if raw_frames.dtype == torch.uint8:
        frames = raw_frames.cpu().numpy()
    else:
        frames = (raw_frames * 255).to(torch.uint8).cpu().permute(0, 2, 3, 1).numpy()
    h, w = frames.shape[1:3]
    writer = cv2.VideoWriter(save_path, cv2.VideoWriter_fourcc(*"mp4v"), fps, (w, h))
    try:
        for fr in frames:
            writer.write(cv2.cvtColor(fr, cv2.COLOR_RGB2BGR))
    finally:
        writer.release()


def add_dict_to_yaml_file(file_path, key, value):
    """Reference util.py:31-44."""
    import os
    import yaml

    data = {}
    if os.path.exists(file_path):
        with open(file_path, "r") as f:
            data = yaml.safe_load(f) or {}
    data[key] = value
    with open(file_path, "w") as f:
        yaml.dump(data, f)


def load_imgs(data_path, n_frames, device="cuda", pil=False):
    """Reference util.py:72-85: frames %05d.jpg / %05d.png -> [n_frames, 3, H, W] in [0, 1]."""
    import os
    from PIL import Image

    imgs, pils = [], []
    for i in range(n_frames):
        img_path = os.path.join(data_path, "%05d.jpg" % i)
        if not os.path.exists(img_path):
            img_path = os.path.join(data_path, "%05d.png" % i)
        img_pil = Image.open(img_path)
        pils.append(img_pil)
        arr = torch.from_numpy(np.array(img_pil.convert("RGB"), dtype=np.uint8)).permute(2, 0, 1).float() / 255.0
        imgs.append(arr.unsqueeze(0))
    out = torch.cat(imgs).to(device)
    return (out, pils) if pil else out


def save_video_frames(video_path, img_size=(512, 512)):
    """Reference util.py:18-29: decode a video into data/<name>/%05d.png resized to img_size = (W, H) with PIL's
    Lanczos, and return the number of frames.  Decoding is `video.decoded_chunks`; like the reference, a `.mov` file
    is rotated by -90 degrees before the resize (`video.read_video` does not do this)."""
    import os
    from pathlib import Path

    from PIL import Image

    from .preprocess import resize_frames
    from .video import decoded_chunks

    name = Path(video_path).stem
    os.makedirs(f"data/{name}", exist_ok=True)
    _, chunks = decoded_chunks(video_path)
    i = 0
    for frames in chunks:
        if video_path.endswith(".mov"):                  # PIL's rotate(-90, expand=True): a quarter turn clockwise
            frames = frames.rot90(-1, (1, 2)).contiguous()
        for f in resize_frames(frames, (img_size[1], img_size[0])).numpy():
            Image.fromarray(f).save(f"data/{name}/{str(i).zfill(5)}.png")
            i += 1
    return i
