"""CPU tier: the C-ABI shared library loads without a GPU and exports exactly the entry points
include/tokenflow_b200.h declares (no compute calls here)."""
import ctypes
import os
import re

import pytest

from tokenflow_b200 import ops
from tokenflow_b200 import _build

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    text = open(os.path.join(REPO, "include", "tokenflow_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(tf_[a-z0-9_]+)\s*\(", text)))


@pytest.fixture(scope="module")
def lib():
    if not ops.library_path().exists():
        _build.build()
    return ops.load_library()


def test_header_and_binding_agree():
    assert _header_functions() == sorted(ops.exported_symbols())


def test_library_exports_every_declared_symbol(lib):
    for name in _header_functions():
        assert hasattr(lib, name), f"{name} declared in include/tokenflow_b200.h but not exported"


def test_version_and_error_string(lib):
    assert lib.tf_version() >= 1000
    assert lib.tf_last_error() == b"" or isinstance(lib.tf_last_error(), bytes)
    assert lib.tf_launch_count() == 0 or lib.tf_launch_count() > 0


def test_argument_validation_needs_no_gpu(lib):
    """Bad shapes are rejected on the host before anything touches the device."""
    st = lib.tf_unit_rows(None, 1, 4, 12, 12, None, None)            # dim % 8 != 0
    assert st == 1 and b"dim" in lib.tf_last_error()
    kf = (ctypes.c_int32 * 2)(0, 7)
    st = lib.tf_nn_field(None, None, kf, None, 2, 16, 32, 3, None, None, None)   # keyframe id 7 >= K
    assert st == 1 and b"keyframe" in lib.tf_last_error()
    st = lib.tf_propagate(None, None, None, kf, None, None, 65, 16, 32, 8, None, None, 0, None)  # F > 64
    assert st == 1
    st = lib.tf_ext_attn_fwd(None, None, None, 64, 100, 16, 2, 32, 0.1, 0, None, None)            # 3n > 160
    assert st == 1
    # empty inputs are a no-op success (reference: empty batch does nothing)
    assert lib.tf_unit_rows(None, 1, 0, 32, 32, None, None) == 0
    assert lib.tf_nn_field(None, None, kf, None, 0, 16, 32, 3, None, None, None) == 0


@pytest.mark.parametrize("inject", [0, 1])
def test_ext_attn_head_dim_over_192_is_rejected_before_any_cuda_call(lib, inject):
    """No attention variant is compiled above d = 192: the head-dim dispatch fails on the host.  The pointers
    are host memory, never dereferenced (and no CUDA device is needed)."""
    buf = (ctypes.c_uint8 * 4096)()
    p = (ctypes.addressof(buf) + 15) & ~15
    st = lib.tf_ext_attn_fwd(p, p, p, 200, 2, 16, 1, 200, 200 ** -0.5, inject, p, None)
    assert st == 3 and b"head dim 200" in lib.tf_last_error()         # TF_ERR_UNSUPPORTED


def test_library_is_sm90a_and_uses_wgmma():
    """The shipped cubin is sm_90a and the hot kernels really use wgmma / TMA / mbarrier."""
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", str(ops.library_path())], capture_output=True, text=True).stdout
    assert "sm_90a" in sass and "sm_100" not in sass
    for mnemonic in ("HGMMA.64x128x16.F32", "UTMALDG.4D", "UTMALDG.3D", "SYNCS.PHASECHK"):
        assert mnemonic in sass, mnemonic
