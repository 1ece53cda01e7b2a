"""In-tree nvcc build of libtokenflow_b200.so (sm_90a only).

The shared library is a plain C-ABI object (include/tokenflow_b200.h): no pybind, no ATen, cudart
linked statically, the driver API resolved at run time — so it also *loads* on a machine without a GPU
(the CPU test tier checks the exported symbols that way).  The built .so is git-ignored.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
LIB_PATH = PKG_DIR / "libtokenflow_b200.so"
STAMP = PKG_DIR / ".libtokenflow_b200.stamp"

SOURCES = ["tf_capi.cu", "tf_unit_rows.cu", "tf_propagate.cu", "tf_nn_field.cu", "tf_ext_attn.cu", "tf_cfg_ddim.cu",
           "tf_comm.cu", "tf_body.cu", "tf_pixels.cu", "tf_resize.cu",
           "tf_canny.cu"]
HEADERS = ["tf_common.cuh", "tf_kernels.h", "tf_wgmma.cuh", "../../include/tokenflow_b200.h"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "-Xcompiler", "-ffp-contract=off",     # host code: tf_resize_coeffs must round like Pillow's C build
    "-Xptxas", "-v",
    "--expt-relaxed-constexpr",
    "-cudart", "static",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")


def _digest() -> str:
    h = hashlib.sha256()
    for name in SOURCES + HEADERS:
        h.update((CSRC / name).read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def needs_build() -> bool:
    return not (LIB_PATH.exists() and STAMP.exists() and STAMP.read_text().strip() == _digest())


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every CUDA source for sm_90a into one shared library.  Objects are built in
    parallel (one nvcc per translation unit) then linked."""
    if not force and not needs_build():
        return LIB_PATH
    nvcc = _nvcc()
    obj_dir = PKG_DIR / "build"
    obj_dir.mkdir(exist_ok=True)
    procs = []
    for src in SOURCES:
        obj = obj_dir / (src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(CSRC / src), "-o", str(obj)]
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    objs = []
    log = []
    for src, obj, p in procs:
        out, _ = p.communicate()
        log.append(f"== {src} ==\n{out}")
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out}")
        objs.append(str(obj))
    link = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static",
            "-Xcompiler", "-fPIC", "-o", str(LIB_PATH), *objs, "-ldl", "-lpthread", "-lrt"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}")
    (PKG_DIR / "build" / "ptxas.log").write_text("\n".join(log))
    STAMP.write_text(_digest())
    if verbose:
        print("\n".join(log))
    return LIB_PATH


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(path)
