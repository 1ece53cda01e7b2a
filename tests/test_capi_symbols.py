"""CPU tier: the C-ABI shared library loads without a GPU and exports exactly the entry points
include/tokenflow_b200.h declares, bound with the header's signatures (no compute calls here).

* Alignment contract.  Every pointer the header requires to be 16-byte aligned, passed one element off, is refused
  with "misaligned": the misaligned-operand tests of the GPU tier rely on this refusal happening on the host.
* The element-wise entry points refuse a NULL operand and a negative length.
"""
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


def test_library_binds_every_entry_point_as_declared(lib):
    for name in _header_functions():
        restype, argtypes = ops._SIGNATURES[name]
        fn = getattr(lib, name)
        assert fn.argtypes == argtypes and fn.restype == restype, name
    assert lib.tf_version() == 1004


def test_v_prediction_entry_points_are_declared_with_the_eps_signatures():
    """tf_cfg_ddim_v / tf_ddim_v are tf_cfg_ddim / tf_ddim with the v-branch of the step: same arguments, same
    conventions, declared and bound next to them."""
    declared = _header_functions()
    for v, eps in (("tf_cfg_ddim_v", "tf_cfg_ddim"), ("tf_ddim_v", "tf_ddim")):
        assert v in declared and eps in declared
        assert ops._SIGNATURES[v] == ops._SIGNATURES[eps], v


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


# ------------------------------------------------------------------------------------------------
# alignment contract of the C ABI
# ------------------------------------------------------------------------------------------------
_BUF = (ctypes.c_uint8 * (1 << 20))()
_P = (ctypes.addressof(_BUF) + 255) & ~255


def _i32(*v):
    return (ctypes.c_int32 * len(v))(*v)


# entry point -> {pointer: element bytes} for every pointer the header requires to be 16-byte aligned (the canny
# conditioning output only 2-byte aligned); coefficient rows, index tables and the frames of tf_resize_u8 / tf_canny_u8
# need only their element's alignment and are not listed
POINTERS = {
    "tf_unit_rows[f16]": {"x": 2, "out": 2},
    "tf_unit_rows[f32]": {"x": 4, "out": 2},
    "tf_layernorm_unit_rows": {"x": 2, "gamma": 4, "beta": 4, "out": 2},
    "tf_layernorm_rows": {"x": 2, "gamma": 4, "beta": 4, "y": 2, "unit": 2},
    "tf_cfg_ddim": {"u": 2, "c": 2, "x": 2, "out": 2},
    "tf_ddim": {"eps": 2, "x": 2, "out": 2},
    "tf_cfg_ddim_v": {"u": 2, "c": 2, "x": 2, "out": 2},
    "tf_ddim_v": {"v": 2, "x": 2, "out": 2},
    "tf_nn_field": {"x_unit": 2, "piv_unit": 2},
    "tf_propagate[f16]": {"A": 2, "residual": 2, "out": 2},
    "tf_propagate[f32]": {"out": 4},
    "tf_ext_attn_fwd": {"q": 2, "k": 2, "v": 2, "out": 2},
    "tf_ext_attn_fwd_rows": {"q": 2, "k": 2, "v": 2, "out": 2},
    "tf_group_norm_nhwc": {"x": 2, "bias": 2, "workspace": 1, "out": 2},
    "tf_geglu": {"xh": 2, "gate": 2, "out": 2},
    "tf_frames_to_nhwc": {"frames": 1, "out": 2},
    "tf_nhwc_to_frames": {"x": 2, "frames": 1},
    "tf_canny_u8": {"workspace": 1, "cond": 1},
}


def _calls(lib):
    """entry point -> call(p): `p(name)` is the address of pointer `name`.  The shapes are valid, so the pointer
    check is the only one that can refuse the call."""
    kf = _i32(0, 0)
    kfb = _i32(-1, 0)
    w = (ctypes.c_float * 2)(1.0, 0.5)
    one = _i32(1)
    zero = _i32(0)
    canny_ws = lib.tf_canny_workspace(1, 8, 8)
    gn_ws = lib.tf_group_norm_nhwc_workspace(2, 16, 64, 8)
    return {
        "tf_unit_rows[f16]": lambda p: lib.tf_unit_rows(p("x"), 0, 4, 8, 8, p("out"), None),
        "tf_unit_rows[f32]": lambda p: lib.tf_unit_rows(p("x"), 1, 4, 8, 8, p("out"), None),
        "tf_layernorm_unit_rows": lambda p: lib.tf_layernorm_unit_rows(
            p("x"), 4, 8, 8, p("gamma"), p("beta"), 1e-5, p("out"), None),
        "tf_layernorm_rows": lambda p: lib.tf_layernorm_rows(
            p("x"), 4, 8, 8, p("gamma"), p("beta"), 1e-5, p("y"), 8, p("unit"), 8, 2, None),
        "tf_cfg_ddim": lambda p: lib.tf_cfg_ddim(p("u"), p("c"), p("x"), _P, 7.5, 64, p("out"), None),
        "tf_ddim": lambda p: lib.tf_ddim(p("eps"), p("x"), _P, 64, p("out"), None),
        "tf_cfg_ddim_v": lambda p: lib.tf_cfg_ddim_v(p("u"), p("c"), p("x"), _P, 7.5, 64, p("out"), None),
        "tf_ddim_v": lambda p: lib.tf_ddim_v(p("v"), p("x"), _P, 64, p("out"), None),
        "tf_nn_field": lambda p: lib.tf_nn_field(p("x_unit"), p("piv_unit"), kf, kfb, 2, 16, 8, 1, _P, _P, None),
        "tf_propagate[f16]": lambda p: lib.tf_propagate(
            p("A"), _P, _P, kf, kfb, w, 2, 16, 8, 1, p("residual"), p("out"), 0, None),
        "tf_propagate[f32]": lambda p: lib.tf_propagate(p("A"), _P, _P, kf, kfb, w, 2, 16, 8, 1, None, p("out"), 1, None),
        "tf_ext_attn_fwd": lambda p: lib.tf_ext_attn_fwd(p("q"), p("k"), p("v"), 16, 1, 16, 1, 16, 0.25, 0, p("out"),
                                                         None),
        "tf_ext_attn_fwd_rows": lambda p: lib.tf_ext_attn_fwd_rows(
            p("q"), 1, 16, p("k"), p("v"), 1, 16, 1, zero, zero, zero, zero, one, 16, 1, 16, 0.25, 0, 16, p("out"), None),
        "tf_group_norm_nhwc": lambda p: lib.tf_group_norm_nhwc(
            p("x"), p("bias"), 64, _P, _P, 2, 16, 64, 8, 1e-5, 1, p("workspace"), gn_ws, p("out"), None),
        "tf_geglu": lambda p: lib.tf_geglu(p("xh"), p("gate"), 64, p("out"), None),
        "tf_frames_to_nhwc": lambda p: lib.tf_frames_to_nhwc(p("frames"), 16, p("out"), None),
        "tf_nhwc_to_frames": lambda p: lib.tf_nhwc_to_frames(p("x"), 16, p("frames"), None),
        "tf_canny_u8": lambda p: lib.tf_canny_u8(_P, 1, 8, 8, 100.0, 200.0, p("workspace"), canny_ws, None, p("cond"),
                                                 None),
    }


# entry points with device pointers that need no more than element alignment: the resize tables and frames, NCCL's
# buffers
ANY_ALIGNMENT = {"tf_resize_u8", "tf_allgather"}


def test_every_entry_point_with_device_pointers_is_covered():
    with_pointers = {name for name, (_, args) in ops._SIGNATURES.items()
                     if any(a is ctypes.c_void_p for a in args) and not name.startswith(("tf_comm_", "tf_resize_coeffs"))}
    covered = {entry.split("[")[0] for entry in POINTERS}
    assert with_pointers - ANY_ALIGNMENT == covered


def _addresses(entry, off=None, null=None):
    """`p(name)` for the calls of `entry`: disjoint 4 KB regions of one host buffer, pointer `off` one element past its
    region's start, pointer `null` NULL."""
    ptrs = POINTERS[entry]
    slot = {name: i * 4096 for i, name in enumerate(ptrs)}
    return lambda name: None if name == null else _P + 65536 + slot.get(name, 0) + (ptrs[name] if name == off else 0)


_CASES = [(entry, ptr) for entry, ptrs in POINTERS.items() for ptr in ptrs]


@pytest.mark.parametrize("entry,ptr", _CASES, ids=[f"{e}-{p}" for e, p in _CASES])
def test_pointer_one_element_off_is_refused_on_the_host(lib, entry, ptr):
    status = _calls(lib)[entry](_addresses(entry, off=ptr))
    assert status == 1 and b"misaligned" in lib.tf_last_error(), (entry, ptr, status, lib.tf_last_error())


# the element-wise entry points and their arguments before the length: operand pointers, then any coefficient row and
# guidance
ELEMENTWISE = {
    "tf_cfg_ddim": 5, "tf_ddim": 3, "tf_cfg_ddim_v": 5, "tf_ddim_v": 3, "tf_geglu": 2, "tf_frames_to_nhwc": 1,
    "tf_nhwc_to_frames": 1,
}


@pytest.mark.parametrize("entry", sorted(ELEMENTWISE))
def test_null_pointers_and_negative_lengths_are_refused(lib, entry):
    for name in POINTERS[entry]:
        assert _calls(lib)[entry](_addresses(entry, null=name)) == 1 and b"NULL" in lib.tf_last_error(), (entry, name)
    args = [None] * ELEMENTWISE[entry]
    if entry.startswith("tf_cfg_ddim"):
        args[-1] = 7.5                                    # guidance
    assert getattr(lib, entry)(*args, -1, None, None) == 1
