"""CPU tier: reading video files (tokenflow_b200/video.py) and `util.save_video_frames` on top of it.

* the reference's sample `wolf.mp4` (H.264, tests/golden/) decodes to its 40 frames of 512² at 20 fps; a clip written
  by `util.save_video` (MPEG-4 Part 2) reads back with its frame count, size and fps, and close to what was written;
* a clip whose track header carries a 90-degree display matrix decodes to the unrotated clip turned a quarter turn
  clockwise, exactly, as OpenCV applies the container's rotation;
* the chunk size does not change the bytes, and resizing in `read_video` is PIL's Lanczos on the full decode;
* `save_video_frames` writes the PNG bytes its OpenCV + PIL loop wrote before it was put on `read_video`'s decoder,
  for `.mp4` names and for `.mov` names, which it rotates as the reference does;
* a missing file, a file that is not a video and `--n_frames` larger than the video raise ValueError.
"""
import os
import shutil
import struct

import numpy as np
import pytest
import torch

from tokenflow_b200 import run
from tokenflow_b200.preprocess import resize_frames
from tokenflow_b200.util import save_video, save_video_frames
from tokenflow_b200.video import read_video

WOLF = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wolf.mp4")
# PSNR of `clip()` written by save_video (mp4v at OpenCV's default bitrate) and decoded again: 35.1 dB measured
MIN_PSNR_DB = 33.0


def clip(n=12, h=48, w=80, seed=0):
    """Smooth random uint8 frames [n, h, w, 3]."""
    g = torch.Generator().manual_seed(seed)
    base = torch.nn.functional.interpolate(torch.rand(n, 3, h // 16, w // 16, generator=g), size=(h, w),
                                           mode="bilinear", align_corners=False)
    return (base * 255).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def rotated_copy(src, dst):
    """`src` with the matrix of its (only) track header set to a 90-degree rotation (ISO/IEC 14496-12 tkhd, version
    0: the matrix starts 40 bytes after the box's version and flags)."""
    data = bytearray(open(src, "rb").read())
    assert data.count(b"tkhd") == 1
    at = data.index(b"tkhd") + 4
    assert data[at] == 0                                              # version 0
    m = at + 40
    assert struct.unpack(">9i", data[m:m + 36]) == (65536, 0, 0, 0, 65536, 0, 0, 0, 1 << 30)
    data[m:m + 36] = struct.pack(">9i", 0, 65536, 0, -65536, 0, 0, 0, 0, 1 << 30)
    with open(dst, "wb") as f:
        f.write(bytes(data))


def test_the_references_sample_decodes_to_its_frames():
    frames, fps = read_video(WOLF)
    assert frames.shape == (40, 512, 512, 3) and frames.dtype == torch.uint8 and fps == 20.0
    assert frames.float().std() > 10


def test_a_written_clip_reads_back(tmp_path):
    fr = clip()
    path = str(tmp_path / "clip.mp4")
    save_video(fr, path, fps=10)
    got, fps = read_video(path)
    assert got.shape == fr.shape and fps == 10.0
    mse = (got.double() - fr.double()).pow(2).mean().item()
    assert 10 * np.log10(255 ** 2 / mse) > MIN_PSNR_DB


def test_the_display_matrix_rotates_the_frames(tmp_path):
    import cv2
    path, turned = str(tmp_path / "clip.mp4"), str(tmp_path / "turned.mp4")
    save_video(clip(), path, fps=10)
    rotated_copy(path, turned)
    cap = cv2.VideoCapture(turned)
    assert cap.get(cv2.CAP_PROP_ORIENTATION_META) == 90
    cap.release()
    upright, _ = read_video(path)
    got, fps = read_video(turned)
    assert got.shape == (12, 80, 48, 3) and fps == 10.0
    assert np.array_equal(got.numpy(), np.rot90(upright.numpy(), -1, axes=(1, 2)))


def test_chunks_and_resizing_do_not_change_the_bytes():
    from PIL import Image
    full, _ = read_video(WOLF)
    for chunk in (1, 7, 64):
        assert torch.equal(read_video(WOLF, chunk=chunk)[0], full), chunk
    want = np.stack([np.asarray(Image.fromarray(f).resize((96, 56), Image.LANCZOS)) for f in full.numpy()])
    for chunk in (1, 7, 64):
        got, fps = read_video(WOLF, (56, 96), chunk=chunk)
        assert fps == 20.0 and np.array_equal(got.numpy(), want), chunk
    assert torch.equal(read_video(WOLF, 40, chunk=7)[0], resize_frames(full, 40))


def save_video_frames_before(video_path, img_size=(512, 512)):
    """util.save_video_frames as it was written before it decoded through `video.decoded_chunks`."""
    import os
    from pathlib import Path

    import cv2
    from PIL import Image

    name = Path(video_path).stem
    os.makedirs(f"data/{name}", exist_ok=True)
    cap = cv2.VideoCapture(video_path)
    i = 0
    while True:
        ok, frame = cap.read()
        if not ok:
            break
        img = Image.fromarray(cv2.cvtColor(frame, cv2.COLOR_BGR2RGB))
        if video_path.endswith(".mov"):
            img = img.rotate(-90, expand=True)
        img.resize(img_size, resample=Image.Resampling.LANCZOS).save(f"data/{name}/{str(i).zfill(5)}.png")
        i += 1
    cap.release()
    return i


@pytest.mark.parametrize("source,name,img_size", [("wolf", "wolf.mp4", (96, 56)), ("clip", "clip.mp4", (64, 40)),
                                                  ("clip", "clip.mov", (64, 40)), ("clip", "phone.mov", (40, 64))])
def test_save_video_frames_writes_the_same_pngs(tmp_path, monkeypatch, source, name, img_size):
    monkeypatch.chdir(tmp_path)
    if source == "wolf":
        shutil.copy(WOLF, name)
    else:
        save_video(clip(), name, fps=10)
    stem = os.path.splitext(name)[0]
    n = save_video_frames(name, img_size)
    os.rename(f"data/{stem}", "written")
    assert save_video_frames_before(name, img_size) == n == (40 if source == "wolf" else 12)
    names = [f"{i:05d}.png" for i in range(n)]
    assert sorted(os.listdir("written")) == sorted(os.listdir(f"data/{stem}")) == names
    for f in names:
        with open(f"written/{f}", "rb") as a, open(f"data/{stem}/{f}", "rb") as b:
            assert a.read() == b.read(), f


def test_unreadable_inputs_raise(tmp_path):
    missing = str(tmp_path / "missing.mp4")
    with pytest.raises(ValueError, match="missing.mp4"):
        read_video(missing)
    text = tmp_path / "notes.mp4"
    text.write_text("not a video\n" * 100)
    with pytest.raises(ValueError, match="notes.mp4"):
        read_video(str(text))
    # a container that opens but whose frame data is blanked: no frame decodes
    save_video(clip(n=3), str(tmp_path / "clip.mp4"), fps=10)
    data = bytearray((tmp_path / "clip.mp4").read_bytes())
    at = data.index(b"mdat")
    size = struct.unpack(">I", data[at - 4:at])[0]
    data[at + 4:at - 4 + size] = bytes(size - 8)
    (tmp_path / "blank.mp4").write_bytes(bytes(data))
    with pytest.raises(ValueError, match="blank.mp4.* no frames"):
        read_video(str(tmp_path / "blank.mp4"))


def test_more_frames_than_the_video_are_refused(tmp_path, monkeypatch):
    """Refused while decoding, before a model is loaded: the checkpoint directory is never opened."""
    monkeypatch.chdir(tmp_path)
    save_video(clip(), "clip.mp4", fps=10)
    with pytest.raises(ValueError, match=r"--n_frames 13 .*clip.mp4.* 12 frames"):
        run.main(["preprocess", "--model_dir", str(tmp_path / "no-checkpoint"), "--device", "cpu",
                  "--data_path", "clip.mp4", "--H", "48", "--W", "80", "--n_frames", "13"])
