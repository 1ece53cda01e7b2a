"""ctypes binding of libtokenflow_b200.so (include/tokenflow_b200.h) and the op layer the hooks call.

`CudaOps` is the product and the only op implementation in this package: every method enqueues a
hand-written sm_90a kernel on the current CUDA stream through the C ABI.  There is no CPU or
PyTorch fallback — constructing `CudaOps` without the built library or without a CUDA device
raises, loudly.  (Tests substitute an oracle-backed op object through
`tokenflow_utils._install_ops_for_testing`; that object lives under `oracle/`, not here.)
"""
from __future__ import annotations

import ctypes
import math
from pathlib import Path
from typing import Optional, Sequence, Tuple

import torch

LIB_NAME = "libtokenflow_b200.so"
TF_MAX_FRAMES = 64
TF_MAX_ATTN_SAMPLES = 160
TF_COMM_ID_BYTES = 128

_c_i32p = ctypes.POINTER(ctypes.c_int32)
_c_f32p = ctypes.POINTER(ctypes.c_float)

# name -> (restype, argtypes); mirrors include/tokenflow_b200.h one to one
_SIGNATURES = {
    "tf_version": (ctypes.c_int, []),
    "tf_last_error": (ctypes.c_char_p, []),
    "tf_launch_count": (ctypes.c_int64, []),
    "tf_unit_rows": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_int64,
                                    ctypes.c_void_p, ctypes.c_void_p]),
    "tf_layernorm_unit_rows": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int64,
                                              ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p,
                                              ctypes.c_void_p]),
    "tf_layernorm_rows": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p,
                                         ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p, ctypes.c_int64,
                                         ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_void_p]),
    "tf_cfg_ddim": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float,
                                   ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
    "tf_ddim": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p,
                               ctypes.c_void_p]),
    "tf_cfg_ddim_v": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                     ctypes.c_float, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
    "tf_ddim_v": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p,
                                 ctypes.c_void_p]),
    "tf_comm_nccl_version": (ctypes.c_int, []),
    "tf_comm_unique_id": (ctypes.c_int, [ctypes.c_void_p]),
    "tf_comm_init": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_void_p)]),
    "tf_allgather": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p]),
    "tf_comm_destroy": (ctypes.c_int, [ctypes.c_void_p]),
    "tf_nn_field": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, _c_i32p, _c_i32p, ctypes.c_int, ctypes.c_int,
                                   ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "tf_propagate": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, _c_i32p, _c_i32p, _c_f32p,
                                    ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                    ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]),
    "tf_ext_attn_fwd": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64,
                                       ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                       ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "tf_ext_attn_fwd_rows": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p,
                                            ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int, _c_i32p,
                                            _c_i32p, _c_i32p, _c_i32p, _c_i32p, ctypes.c_int, ctypes.c_int,
                                            ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                            ctypes.c_void_p]),
    "tf_group_norm_nhwc_workspace": (ctypes.c_int64, [ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int]),
    "tf_group_norm_nhwc": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p,
                                          ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
                                          ctypes.c_float, ctypes.c_int, ctypes.c_void_p, ctypes.c_int64,
                                          ctypes.c_void_p, ctypes.c_void_p]),
    "tf_frames_to_nhwc": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
    "tf_nhwc_to_frames": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
    "tf_resize_taps": (ctypes.c_int, [ctypes.c_int, ctypes.c_int]),
    "tf_resize_coeffs": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    "tf_resize_u8": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                    ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                    ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "tf_canny_workspace": (ctypes.c_int64, [ctypes.c_int64, ctypes.c_int, ctypes.c_int]),
    "tf_canny_u8": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_double,
                                   ctypes.c_double, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p,
                                   ctypes.c_void_p]),
    "tf_geglu": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
}


class TokenflowB200Error(RuntimeError):
    pass


def library_path() -> Path:
    return Path(__file__).resolve().parent / LIB_NAME


_LIB = None


def load_library() -> ctypes.CDLL:
    """dlopen the in-tree library and declare every prototype.  Needs no GPU."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = library_path()
    if not path.exists():
        raise TokenflowB200Error(
            f"{path} is missing: build it with `python -m tokenflow_b200._build` "
            "(or __graft_entry__.build()).  tokenflow_b200 has no fallback path.")
    lib = ctypes.CDLL(str(path))
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)           # AttributeError here = header and library disagree
        fn.restype = res
        fn.argtypes = args
    _LIB = lib
    return lib


def exported_symbols() -> Sequence[str]:
    return tuple(_SIGNATURES.keys())


def blend_weights(n_frames: int) -> Sequence[float]:
    """w[f] = sigmoid(d2/(d1+d2)), d1=|g-(iB+B//2)|, d2=|g-((i-1)B+B//2)|, g=iB+f (reference
    tokenflow_utils.py:375-383); the batch index i cancels, so the table depends on B only.
    Evaluated in fp32 with the same torch ops as the reference so the weights are bit-identical."""
    f = torch.arange(0, n_frames)
    d1 = torch.abs(f - n_frames // 2)
    d2 = torch.abs(f + n_frames - n_frames // 2)
    return torch.sigmoid(d2 / (d1 + d2)).tolist()


def propagate_bytes(F_: int, S: int, dim: int, kf_a, kf_b, with_residual: bool, out_esz: int = 2) -> float:
    """Algorithmic HBM bytes of one tf_propagate launch (DESIGN.md / SURVEY.md §8d): output write +
    residual read + each referenced keyframe slab once for the three streams + the int32 indices.
    Re-touched keyframe rows are L2 hits and are not counted."""
    kfs = {int(a) for a in kf_a} | {int(b) for b in kf_b if int(b) >= 0}
    n_idx = F_ + sum(1 for b in kf_b if int(b) >= 0)
    return (3.0 * F_ * S * dim * out_esz + (3.0 * F_ * S * dim * 2 if with_residual else 0.0)
            + 3.0 * len(kfs) * S * dim * 2 + 4.0 * S * n_idx)


def _dense(t: torch.Tensor, memory_format=torch.contiguous_format) -> torch.Tensor:
    """`t` itself when it is dense in `memory_format` and starts on a 16-byte boundary (the C ABI refuses any other
    pointer: the kernels load 16-byte vectors and address operands through TMA descriptors), else a copy that is both
    (the caching allocator aligns every block).  An operand may start at any element offset: a slice along the first
    dimension of an odd number of odd-sized latents, for one, starts 8 bytes off."""
    if t.is_contiguous(memory_format=memory_format) and t.data_ptr() % 16 == 0:
        return t
    return t.clone(memory_format=memory_format)


def _rows(t: torch.Tensor, multiple: int) -> torch.Tensor:
    """`t` itself when the kernels can address its rows (its last dimension) in place: last dimension contiguous, rows
    equally spaced by a pitch of a multiple of `multiple` elements, the first one on a 16-byte boundary (a column slice
    of a packed buffer qualifies); else a dense copy, as in `_dense`."""
    spaced = all(t.stride(i) == t.shape[i + 1] * t.stride(i + 1) for i in range(t.dim() - 2) if t.shape[i] > 1)
    if t.stride(-1) == 1 and t.stride(-2) % multiple == 0 and spaced and t.data_ptr() % 16 == 0:
        return t
    return t.clone(memory_format=torch.contiguous_format)


def _out_buffer(out: Optional[torch.Tensor], shape, device, scratch: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Where a kernel writes the fp16 output `out`: `out` itself when it starts on a 16-byte boundary, else `scratch`
    or a new dense buffer of `shape` (also when `out` is None), which `_written` copies back."""
    if out is not None and out.data_ptr() % 16 == 0:
        return out
    return scratch if scratch is not None else torch.empty(shape, dtype=torch.float16, device=device)


def _written(out: Optional[torch.Tensor], buf: torch.Tensor) -> torch.Tensor:
    """The output `out` (or `buf` when there is none) holding what the kernel wrote into `_out_buffer`'s `buf`."""
    return buf if out is None or out is buf else out.copy_(buf)


def _check(lib: ctypes.CDLL, status: int, what: str):
    if status != 0:
        msg = lib.tf_last_error().decode(errors="replace")
        raise TokenflowB200Error(f"{what} failed (status {status}): {msg}")


def _i32(vals: Sequence[int]):
    return (ctypes.c_int32 * len(vals))(*[int(v) for v in vals])


def _f32(vals: Sequence[float]):
    return (ctypes.c_float * len(vals))(*[float(v) for v in vals])


class CudaOps:
    """The hot-path operators, each one C-ABI call = one sm_90a kernel launch on the current stream."""

    name = "cuda-sm90a"

    def __init__(self):
        self.lib = load_library()
        if not torch.cuda.is_available():
            raise TokenflowB200Error(
                "tokenflow_b200 needs a CUDA device (sm_90a / H100); there is no CPU path.")
        major, minor = torch.cuda.get_device_capability()
        if (major, minor) != (9, 0):
            raise TokenflowB200Error(f"tokenflow_b200 kernels are compiled for sm_90a only (got sm_{major}{minor})")

    # -- helpers ---------------------------------------------------------------------------
    @staticmethod
    def _stream() -> int:
        return torch.cuda.current_stream().cuda_stream

    def launch_count(self) -> int:
        return int(self.lib.tf_launch_count())

    # -- optional per-launch CUDA-event timing (bench.py's live roofline measurement) ------------
    _timing = None

    def enable_timing(self, on: bool = True):
        """When on, every kernel launch is bracketed by CUDA events recorded on the launching
        (current) stream; `timing_summary()` synchronises and aggregates them per kernel."""
        self._timing = [] if on else None

    def _launch(self, timer: str, work: float, fn: str, *args):
        """Enqueue the C entry point `fn`(*args, stream) on the current stream, timed as `timer` with `work` when timing
        is on, and raise on a nonzero status."""
        entry = getattr(self.lib, fn)
        if self._timing is None:
            return _check(self.lib, entry(*args, self._stream()), fn)
        ext = torch.cuda.is_current_stream_capturing()    # inside a CUDA-graph capture: event-record NODES
        start = torch.cuda.Event(enable_timing=True, external=ext)
        end = torch.cuda.Event(enable_timing=True, external=ext)
        start.record()
        _check(self.lib, entry(*args, self._stream()), fn)
        end.record()
        self._timing.append((timer, float(work), start, end))

    def timing_summary(self):
        """{kernel: {"launches", "ms", "work"}}; `work` = algorithmic flops (tensor-bound kernels)
        or bytes (HBM-bound kernels) summed over launches."""
        torch.cuda.synchronize()
        agg = {}
        for name, work, s, e in (self._timing or []):
            a = agg.setdefault(name, {"launches": 0, "ms": 0.0, "work": 0.0})
            a["launches"] += 1
            a["ms"] += s.elapsed_time(e)
            a["work"] += work
        if self._timing is not None:
            self._timing = []
        return agg

    # -- operators -------------------------------------------------------------------------
    def unit_rows(self, x: torch.Tensor) -> torch.Tensor:
        """[..., dim] fp32/fp16 → fp16 unit rows (reference util.py:66-67 + autocast fp16 cast); x may start at any
        element offset."""
        if x.dtype not in (torch.float32, torch.float16):
            x = x.float()
        dim = x.shape[-1]
        x2 = _rows(x.reshape(-1, dim), 4)
        out = torch.empty(x2.shape, dtype=torch.float16, device=x.device)
        nbytes = x2.shape[0] * dim * (x2.element_size() + 2)
        self._launch("tf_unit_rows", nbytes, "tf_unit_rows", x2.data_ptr(), int(x2.dtype == torch.float32), x2.shape[0],
                     dim, x2.stride(0), out.data_ptr())
        return out.view(*x.shape)

    @staticmethod
    def _affine_f32(norm: torch.nn.LayerNorm, device):
        """fp32 copies of norm.weight / norm.bias for the fused LayerNorm kernels, re-made whenever either
        parameter's storage or version counter changes (load_state_dict, .half(), in-place updates)."""
        key = (norm.weight.data_ptr(), norm.weight._version, norm.bias.data_ptr(), norm.bias._version, str(device))
        cache = norm.__dict__.get("_tf_affine_f32")
        if cache is None or cache[0] != key:
            cache = (key, norm.weight.detach().to(device=device, dtype=torch.float32).contiguous(),
                     norm.bias.detach().to(device=device, dtype=torch.float32).contiguous())
            norm.__dict__["_tf_affine_f32"] = cache
        return cache[1], cache[2]

    @staticmethod
    def _ln_fusable(x: torch.Tensor, norm) -> bool:
        return (x.dtype == torch.float16 and x.shape[-1] <= 1280 and getattr(norm, "weight", None) is not None
                and getattr(norm, "bias", None) is not None and tuple(norm.normalized_shape) == (x.shape[-1],))

    def layernorm_unit_rows(self, x: torch.Tensor, norm: torch.nn.LayerNorm) -> torch.Tensor:
        """fp16 [..., dim] → fp16 unit rows of LayerNorm(x) (fp32 statistics): norm1 + unit_rows in one
        pass over the source stream (reference tokenflow_utils.py:323 + util.py:66-67); x may start at any element
        offset."""
        dim = x.shape[-1]
        if not self._ln_fusable(x, norm):
            return self.unit_rows(norm(x))                       # shapes the fused kernel does not cover
        gamma, beta = self._affine_f32(norm, x.device)
        x2 = _rows(x.reshape(-1, dim), 8)
        out = torch.empty(x2.shape, dtype=torch.float16, device=x.device)
        self._launch("tf_layernorm_unit_rows", x2.shape[0] * dim * 4, "tf_layernorm_unit_rows", x2.data_ptr(),
                     x2.shape[0], dim, x2.stride(0), gamma.data_ptr(), beta.data_ptr(), float(norm.eps), out.data_ptr())
        return out.view(*x.shape)

    def layernorm_rows(self, x: torch.Tensor, norm: torch.nn.LayerNorm, n_unit: int,
                       y_out: Optional[torch.Tensor] = None, unit_out: Optional[torch.Tensor] = None):
        """Pivotal-pass norm1 fused with its two consumers: x [b, S, dim] fp16 → (y, unit) with
        y = fp16(LN(x)) [b, S, dim] (the QKV GEMM operand) and unit = fp16 unit rows of LN(x) for the first
        `n_unit` samples [n_unit, S, dim] (the pivot features of the NN field) — one read of x
        (reference tokenflow_utils.py:323 -> :120-122, :326-327, util.py:66-67).  `y_out` / `unit_out` may be
        views into packed buffers (last dim contiguous, row pitch a multiple of 8); x and both outputs may start at
        any element offset (a misaligned output is written through an aligned buffer and a copy)."""
        b, S, dim = x.shape
        if not self._ln_fusable(x, norm):
            y = norm(x)
            unit = self.unit_rows(y[:n_unit]) if n_unit else None
            if y_out is not None:
                y_out.copy_(y); y = y_out
            if unit_out is not None and unit is not None:
                unit_out.copy_(unit); unit = unit_out
            return y, unit
        gamma, beta = self._affine_f32(norm, x.device)
        x2 = _rows(x.reshape(-1, dim), 8)
        y = _out_buffer(y_out, (b, S, dim), x.device)
        unit = _out_buffer(unit_out, (n_unit, S, dim), x.device) if n_unit else None
        def pitch(t):      # row pitch of a [.., S, dim] view whose rows are equally spaced
            assert t.stride(-1) == 1 and t.stride(-2) % 8 == 0 and (t.shape[0] <= 1 or t.stride(0) == S * t.stride(-2))
            return t.stride(-2)
        self._launch("tf_layernorm_rows", x2.shape[0] * dim * 4 + n_unit * S * dim * 2, "tf_layernorm_rows",
                     x2.data_ptr(), x2.shape[0], dim, x2.stride(0), gamma.data_ptr(), beta.data_ptr(), float(norm.eps),
                     y.data_ptr(), pitch(y), unit.data_ptr() if unit is not None else None,
                     pitch(unit) if unit is not None else dim, n_unit * S)
        return _written(y_out, y), _written(unit_out, unit) if unit is not None else None

    def cfg_ddim(self, eps_uncond: torch.Tensor, eps_cond: torch.Tensor, x: torch.Tensor, coef: torch.Tensor,
                 guidance: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Classifier-free guidance + DDIM update (reference run_tokenflow_pnp.py:213-217) in one pass;
        `coef` = device fp32 [4]: sqrt(1-a_t), 1/sqrt(a_t), sqrt(a_prev), sqrt(1-a_prev).  The operands may have any
        layout and start at any element offset; `out` (contiguous, made here when None) too: a misaligned one is
        written through an aligned buffer and a copy."""
        return self._cfg_step("tf_cfg_ddim", eps_uncond, eps_cond, x, coef, guidance, out)

    def cfg_ddim_v(self, v_uncond: torch.Tensor, v_cond: torch.Tensor, x: torch.Tensor, coef: torch.Tensor,
                   guidance: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """`cfg_ddim` for a v-prediction model (include/tokenflow_b200.h): guidance on the two velocity
        predictions, then diffusers' v-branch of the DDIM step; `coef` = device fp32 [4]: sqrt(a_t), sqrt(1-a_t),
        sqrt(a_prev), sqrt(1-a_prev).  Operands and `out` as in `cfg_ddim`."""
        return self._cfg_step("tf_cfg_ddim_v", v_uncond, v_cond, x, coef, guidance, out)

    def _cfg_step(self, fn: str, u: torch.Tensor, c: torch.Tensor, x: torch.Tensor, coef: torch.Tensor,
                  guidance: float, out: Optional[torch.Tensor]) -> torch.Tensor:
        assert u.dtype == c.dtype == x.dtype == torch.float16 and coef.dtype == torch.float32
        eu, ec, xx = (_dense(t) for t in (u, c, x))
        assert eu.shape == ec.shape == xx.shape
        assert out is None or (out.shape == xx.shape and out.dtype == torch.float16 and out.is_contiguous())
        dst = _out_buffer(out, xx.shape, xx.device)
        n = xx.numel()
        self._launch(fn, n * 8.0, fn, eu.data_ptr(), ec.data_ptr(), xx.data_ptr(), coef.data_ptr(), float(guidance), n,
                     dst.data_ptr())
        return _written(out, dst)

    def ddim(self, eps: torch.Tensor, x: torch.Tensor, coef: torch.Tensor,
             out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Guidance-free DDIM update of the inversion stage (reference preprocess.py:217-225 / :251-260);
        `coef` = device fp32 [4] (s1, inv_s2, s3, s4), see include/tokenflow_b200.h.  `out` may be `x` (in place).
        eps may have any layout; x and `out` are contiguous.  All three may start at any element offset: a misaligned
        operand is read from an aligned copy, a misaligned `out` (or `x`, in place) is written through an aligned
        buffer and a copy back."""
        return self._step("tf_ddim", eps, x, coef, out)

    def ddim_v(self, v: torch.Tensor, x: torch.Tensor, coef: torch.Tensor,
               out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """`ddim` for a v-prediction model (include/tokenflow_b200.h), diffusers' DDIMInverseScheduler /
        DDIMScheduler v-branch; `coef` = device fp32 [4]: inversion (mu_prev, sigma_prev, mu, sigma), reconstruction
        (mu, sigma, mu_prev, sigma_prev).  Operands, `out` and in place as in `ddim`."""
        return self._step("tf_ddim_v", v, x, coef, out)

    def _step(self, fn: str, m: torch.Tensor, x: torch.Tensor, coef: torch.Tensor,
              out: Optional[torch.Tensor]) -> torch.Tensor:
        assert m.dtype == x.dtype == torch.float16 and coef.dtype == torch.float32 and coef.is_cuda
        assert m.shape == x.shape and x.is_contiguous()
        assert out is None or (out.shape == x.shape and out.dtype == torch.float16 and out.is_contiguous())
        e, xx = _dense(m), _dense(x)
        dst = _out_buffer(out, x.shape, x.device, scratch=xx if out is x else None)     # in place: x's aligned copy
        n = x.numel()
        self._launch(fn, n * 6.0, fn, e.data_ptr(), xx.data_ptr(), coef.data_ptr(), n, dst.data_ptr())
        return _written(out, dst)

    def nn_field(self, x_unit: torch.Tensor, piv_unit: torch.Tensor, kf_a: Sequence[int],
                 kf_b: Sequence[int]) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """x_unit [F,S,dim], piv_unit [K,S,dim] fp16 unit rows → int32 idx_a, idx_b [F,S]
        (reference tokenflow_utils.py:335-343).  The idx_b rows of frames with kf_b < 0 are left unwritten
        (idx_b is None when no frame has a second keyframe).  Both operands may have any layout and start at any element
        offset."""
        F_, S, dim = x_unit.shape
        K = piv_unit.shape[0]
        assert x_unit.dtype == torch.float16 and piv_unit.dtype == torch.float16
        x_unit, piv_unit = _dense(x_unit), _dense(piv_unit)
        idx_a = torch.empty((F_, S), dtype=torch.int32, device=x_unit.device)
        any_b = any(int(b) >= 0 for b in kf_b)
        idx_b = torch.empty((F_, S), dtype=torch.int32, device=x_unit.device) if any_b else None
        pairs = F_ + sum(1 for b in kf_b if int(b) >= 0)
        self._launch("tf_nn_field", 2.0 * pairs * S * S * dim, "tf_nn_field", x_unit.data_ptr(), piv_unit.data_ptr(),
                     _i32(kf_a), _i32(kf_b), F_, S, dim, K, idx_a.data_ptr(),
                     idx_b.data_ptr() if idx_b is not None else None)
        return idx_a, idx_b

    def propagate(self, A: torch.Tensor, idx_a: torch.Tensor, idx_b: Optional[torch.Tensor],
                  kf_a: Sequence[int], kf_b: Sequence[int], w: Sequence[float],
                  residual: Optional[torch.Tensor], out_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
        """A [3,K,S,dim] fp16; idx [F,S] int32; residual [3F,S,dim] fp16 or None → [3F,S,dim]
        (reference tokenflow_utils.py:361-397).  A and residual may have any layout and start at any element offset,
        the int32 indices at any element offset."""
        three, K, S, dim = A.shape
        out_dtype = torch.float16 if out_dtype is None else out_dtype
        A = _dense(A.to(torch.float16))
        assert three == 3
        F_ = idx_a.shape[0]
        if residual is not None:
            residual = _dense(residual.to(torch.float16)).view(3, F_, S, dim)
        out = torch.empty((3, F_, S, dim), dtype=out_dtype, device=A.device)
        assert out_dtype in (torch.float16, torch.float32)
        self._launch("tf_propagate", propagate_bytes(F_, S, dim, kf_a, kf_b, residual is not None, out.element_size()),
                     "tf_propagate", A.data_ptr(), idx_a.data_ptr(), idx_b.data_ptr() if idx_b is not None else None,
                     _i32(kf_a), _i32(kf_b), _f32(w), F_, S, dim, K,
                     residual.data_ptr() if residual is not None else None, out.data_ptr(),
                     int(out_dtype == torch.float32))
        return out.view(3 * F_, S, dim)

    def ext_attn(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, scale: float,
                 inject: bool) -> torch.Tensor:
        """q,k,v [3n,S,dim] fp16 (same token stride) → [3n,S,dim] fp16, before to_out
        (reference tokenflow_utils.py:124-197 / :234-279).  q, k and v may start at any element offset; views with
        other strides are copied."""
        b, S, dim = q.shape
        n = b // 3
        d = dim // heads
        q, k, v = (_rows(t.to(torch.float16), 8) for t in (q, k, v))
        if len({t.stride() for t in (q, k, v)}) != 1:         # one token stride for all three
            q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        out = torch.empty((b, S, dim), dtype=torch.float16, device=q.device)
        flops = 4.0 * n * S * S * dim * (2 * n + 1)        # QK^T + PV; source: S keys, uncond+cond: n*S keys
        self._launch("tf_ext_attn", flops, "tf_ext_attn_fwd", q.data_ptr(), k.data_ptr(), v.data_ptr(), q.stride(1),
                     n, S, heads, d, float(scale), int(bool(inject)), out.data_ptr())
        return out

    def ext_attn_table(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, table, heads: int,
                       scale: float, row0: int = 0, nrows: Optional[int] = None) -> torch.Tensor:
        """General form (sharded pivotal pass): `table[j] = (q slab, first k slab, first v slab, number of
        consecutive key slabs)` for output sample j.  q [Q,S,dim], k/v [KV,S,dim] fp16 (column slices of packed
        buffers are read in place) → [len(table), nrows, dim]: only the query tokens [row0, row0 + nrows) are
        computed (default: all S; row0 a multiple of 128).  When row0 + nrows > S, the output rows of tokens
        past S (rows S - row0 onwards) are left unwritten."""
        _, S, dim = q.shape
        d = dim // heads
        nrows = S if nrows is None else int(nrows)
        q, k, v = (_rows(t.to(torch.float16), 8) for t in (q, k, v))
        if k.stride(1) != v.stride(1):
            k, v = k.contiguous(), v.contiguous()
        n_out = len(table)
        out = torch.empty((n_out, nrows, dim), dtype=torch.float16, device=q.device)
        rows_eff = max(0, min(S, row0 + nrows) - row0)
        flops = sum(4.0 * rows_eff * (nkv * S) * dim for (_, _, _, nkv) in table)
        self._launch("tf_ext_attn", flops, "tf_ext_attn_fwd_rows", q.data_ptr(), q.shape[0], q.stride(1), k.data_ptr(),
                     v.data_ptr(), k.shape[0], k.stride(1), n_out, _i32(range(n_out)), _i32([t[0] for t in table]),
                     _i32([t[1] for t in table]), _i32([t[2] for t in table]), _i32([t[3] for t in table]), S, heads,
                     d, float(scale), int(row0), nrows, out.data_ptr())
        return out

    # -- UNet body ----------------------------------------------------------------------------
    @staticmethod
    def group_norm_nhwc_supported(x: torch.Tensor, norm: torch.nn.GroupNorm,
                                  bias: Optional[torch.Tensor] = None) -> bool:
        """Operands tf_group_norm_nhwc covers: CUDA fp16 channels_last [N, C, H, W] with C % 8 == 0, C <= 4096, groups
        dividing C, fp16 affine parameters, and either at least 8 channels per group with an fp16 or no bias, or
        exactly 4 channels per group without a bias."""
        if not (x.is_cuda and x.dtype == torch.float16 and x.dim() == 4
                and x.is_contiguous(memory_format=torch.channels_last)):
            return False
        c, g = x.shape[1], norm.num_groups
        w, b = norm.weight, norm.bias
        if not (c % 8 == 0 and c <= 4096 and c % g == 0 and w is not None and b is not None
                and w.dtype == b.dtype == torch.float16 and w.is_contiguous() and b.is_contiguous()):
            return False
        if c == 4 * g:
            return bias is None
        return c // g >= 8 and (bias is None or bias.dtype == torch.float16)

    def group_norm_nhwc(self, x: torch.Tensor, norm: torch.nn.GroupNorm, bias: Optional[torch.Tensor] = None,
                        silu: bool = False) -> torch.Tensor:
        """[SiLU](GroupNorm(x [+ bias[:, :, None, None]])) of a channels_last fp16 [N, C, H, W] tensor, channels_last
        out, with the eager fp16 rounding sequence.  `bias` is fp16 [N, C] or [1, C] (the resnet's time-embedding
        projection), and None at 4 channels per group.  Two launches, timed as "tf_group_norm_g4" at 4 channels per
        group (the VAE's 128-channel levels) and "tf_group_norm" otherwise; the statistics workspace comes from the
        caching allocator on this stream.  x and bias may start at any element offset."""
        n, c, h, w = x.shape
        x = _dense(x, torch.channels_last)
        if bias is not None:
            assert bias.dtype == torch.float16 and bias.dim() == 2 and bias.shape[1] == c and bias.shape[0] in (1, n)
            bias = _rows(bias, 8)
            bias_stride = 0 if bias.shape[0] == 1 else bias.stride(0)
        ws_bytes = int(self.lib.tf_group_norm_nhwc_workspace(n, h * w, c, norm.num_groups))
        if ws_bytes < 0:
            _check(self.lib, 3, "tf_group_norm_nhwc_workspace")
        ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=x.device)
        out = torch.empty_like(x, memory_format=torch.channels_last)
        work = 3.0 * x.numel() * 2 + (n * c * 2 if bias is not None else 0)
        name = "tf_group_norm_g4" if c == 4 * norm.num_groups else "tf_group_norm"
        self._launch(name, work, "tf_group_norm_nhwc", x.data_ptr(), bias.data_ptr() if bias is not None else None,
                     bias_stride if bias is not None else 0, norm.weight.data_ptr(), norm.bias.data_ptr(), n, h * w, c,
                     norm.num_groups, float(norm.eps), int(bool(silu)), ws.data_ptr(), ws.numel(), out.data_ptr())
        return out

    def frames_to_nhwc(self, frames: torch.Tensor) -> torch.Tensor:
        """uint8 RGB frames [N, H, W, 3] (CUDA) -> the encoder input 2 * ToTensor(frames) - 1 as a channels_last fp16
        [N, 3, H, W] tensor, bit-equal to the reference's host conversion followed by the fp16 ops.  `frames` may start
        at any element offset."""
        assert frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[-1] == 3 and frames.is_cuda
        frames = _dense(frames)
        n, h, w, _ = frames.shape
        out = torch.empty((n, 3, h, w), dtype=torch.float16, device=frames.device, memory_format=torch.channels_last)
        self._launch("tf_frames_to_nhwc", 3.0 * n * h * w, "tf_frames_to_nhwc", frames.data_ptr(), n * h * w,
                     out.data_ptr())
        return out

    def nhwc_to_frames(self, x: torch.Tensor) -> torch.Tensor:
        """fp16 decoder output [N, 3, H, W] -> uint8 frames [N, H, W, 3], bit-equal to
        `((x / 2 + 0.5).clamp(0, 1) * 255).to(torch.uint8)` in fp16 (NaN -> 0).  x may start at any element offset."""
        assert x.dtype == torch.float16 and x.dim() == 4 and x.shape[1] == 3 and x.is_cuda
        x = _dense(x, torch.channels_last)
        n, _, h, w = x.shape
        out = torch.empty((n, h, w, 3), dtype=torch.uint8, device=x.device)
        self._launch("tf_nhwc_to_frames", 3.0 * n * h * w, "tf_nhwc_to_frames", x.data_ptr(), n * h * w, out.data_ptr())
        return out

    def _resize_tables(self, n_in: int, n_out: int, device):
        """Device (bounds, coeffs, taps) of one axis n_in -> n_out (tf_resize_coeffs), made once per pair and device."""
        cache = self.__dict__.setdefault("_resize_cache", {})
        key = (n_in, n_out, str(device))
        if key not in cache:
            taps = int(self.lib.tf_resize_taps(n_in, n_out))
            if taps < 0:
                _check(self.lib, 1, "tf_resize_taps")
            bounds = torch.empty((n_out, 2), dtype=torch.int32)
            coeffs = torch.empty((n_out, taps), dtype=torch.int32)
            _check(self.lib, self.lib.tf_resize_coeffs(n_in, n_out, bounds.data_ptr(), coeffs.data_ptr()), "tf_resize_coeffs")
            cache[key] = (bounds.to(device), coeffs.to(device), taps)
        return cache[key]

    def resize_frames(self, frames: torch.Tensor, size: Tuple[int, int], tmp: Optional[torch.Tensor] = None,
                      out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """uint8 RGB frames [N, H_in, W_in, 3] (CUDA) -> [N, H, W, 3] for size = (H, W), bit-equal to PIL's
        `Image.resize((W, H), Image.LANCZOS)` of every frame.  `tmp` ([N, H_in, W, 3] uint8, or [N, H, W_in, 3] for a
        frame more than 100 times taller than wide whose height shrinks: Pillow resizes those vertically first) and
        `out` may be given; they are made here otherwise.  Every buffer may start at any element offset (the kernels
        read and write bytes)."""
        assert frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[-1] == 3 and frames.is_cuda
        frames = frames.contiguous()
        n, h_in, w_in, _ = frames.shape
        h, w = int(size[0]), int(size[1])
        dev = frames.device
        need_h, need_v = w != w_in, h != h_in
        hb, hk, ht = self._resize_tables(w_in, w, dev) if need_h else (None, None, 0)
        vb, vk, vt = self._resize_tables(h_in, h, dev) if need_v else (None, None, 0)
        if out is None:
            out = torch.empty((n, h, w, 3), dtype=torch.uint8, device=dev)
        assert out.shape == (n, h, w, 3) and out.dtype == torch.uint8 and out.is_contiguous()
        v_first = need_h and need_v and h_in > 100 * w_in and h < h_in
        tmp_shape = (n, h, w_in, 3) if v_first else (n, h_in, w, 3)
        if need_h and need_v and tmp is None:
            tmp = torch.empty(tmp_shape, dtype=torch.uint8, device=dev)
        if tmp is not None:
            assert tmp.numel() >= math.prod(tmp_shape) and tmp.dtype == torch.uint8 and tmp.is_contiguous()
        work = 3.0 * n * (h_in * w_in + (2 * math.prod(tmp_shape[1:3]) if need_h and need_v else 0) + h * w)
        ptr = lambda t: t.data_ptr() if t is not None else None
        self._launch("tf_resize_u8", work, "tf_resize_u8", frames.data_ptr(), n, h_in, w_in, h, w, ptr(hb), ptr(hk), ht,
                     ptr(vb), ptr(vk), vt, ptr(tmp), out.data_ptr())
        return out

    def canny(self, frames: torch.Tensor, low: float = 100, high: float = 200, edges: bool = True, cond: bool = True,
              out_edges: Optional[torch.Tensor] = None, out_cond: Optional[torch.Tensor] = None):
        """uint8 RGB frames [N, H, W, 3] (CUDA) -> (edges, cond): `cv2.Canny(frame, low, high)` of every frame as uint8
        [N, H, W] (0 / 255) and the reference's `get_canny_cond` tensor, fp16 [N, 3, H, W] channels_last with 0 / 1 in
        every channel.  Either output can be skipped (None is returned in its place) or given.  The workspace comes from
        the caching allocator on this stream.  Frames and outputs may start at any element offset."""
        assert frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[-1] == 3 and frames.is_cuda
        assert edges or cond
        frames = frames.contiguous()
        n, h, w, _ = frames.shape
        dev = frames.device
        ws_bytes = int(self.lib.tf_canny_workspace(n, h, w))
        if ws_bytes < 0:
            _check(self.lib, 1, "tf_canny_workspace")
        ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=dev)
        e = c = None
        if edges:
            e = out_edges if out_edges is not None else torch.empty((n, h, w), dtype=torch.uint8, device=dev)
            assert e.shape == (n, h, w) and e.dtype == torch.uint8 and e.is_contiguous()
        if cond:
            c = out_cond if out_cond is not None else torch.empty((n, 3, h, w), dtype=torch.float16, device=dev,
                                                                  memory_format=torch.channels_last)
            assert c.shape == (n, 3, h, w) and c.dtype == torch.float16 and c.is_contiguous(memory_format=torch.channels_last)
        work = 3.0 * n * h * w + (n * h * w if edges else 0) + (6.0 * n * h * w if cond else 0)
        ptr = lambda t: t.data_ptr() if t is not None else None
        self._launch("tf_canny_u8", work, "tf_canny_u8", frames.data_ptr(), n, h, w, float(low), float(high),
                     ws.data_ptr(), ws.numel(), ptr(e), ptr(c))
        return e, c

    def geglu(self, xh: torch.Tensor, gate: torch.Tensor) -> torch.Tensor:
        """xh * gelu(gate) of two fp16 tensors of one shape (the GEGLU GEMM outputs), bit-equal to the eager product.
        Both may start at any element offset."""
        assert xh.dtype == gate.dtype == torch.float16 and xh.shape == gate.shape
        xh, gate = _dense(xh), _dense(gate)
        out = torch.empty_like(xh)
        n = xh.numel()
        self._launch("tf_geglu", 3.0 * n * 2, "tf_geglu", xh.data_ptr(), gate.data_ptr(), n, out.data_ptr())
        return out


_DEFAULT_OPS = None


def default_ops() -> CudaOps:
    """The process-wide CudaOps (built on first use; raises without the library or an sm_90 device)."""
    global _DEFAULT_OPS
    if _DEFAULT_OPS is None:
        _DEFAULT_OPS = CudaOps()
    return _DEFAULT_OPS


_BODY_OPS = False           # not looked up yet


def body_ops() -> Optional[CudaOps]:
    """The CudaOps the UNet body's fused GroupNorm / GEGLU run on — the same object as the hook layer's, so its
    per-launch timing covers them — or None when the library or an sm_90 device is missing (the body then runs its
    ATen ops: CPU runs, fp32 models)."""
    global _BODY_OPS
    if _BODY_OPS is False:
        try:
            _BODY_OPS = default_ops()
        except TokenflowB200Error:
            _BODY_OPS = None
    return _BODY_OPS


def all_gather(t: torch.Tensor, world_size: int, group=None, comm=None) -> torch.Tensor:
    """[n, ...] on every rank -> [world_size * n, ...] in rank order: the one collective of the package.  A CUDA tensor
    goes through `comm` (a `Communicator`) when one is attached, everything else through torch.distributed on
    `group`; one rank returns `t` itself."""
    if world_size == 1:
        return t
    if comm is not None and t.is_cuda:
        return comm.all_gather(t)
    import torch.distributed as dist
    t = t.contiguous()
    out = torch.empty((world_size * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    dist.all_gather_into_tensor(out, t, group=group)
    return out


def frame_share(n: int, world_size: int, rank: int) -> Tuple[int, int]:
    """Frames [lo, hi) of `rank` when n frames are dealt to `world_size` ranks in contiguous shares of ceil(n / G):
    the split of the inversion stage and of the edit.  The last shares may be short, or empty (hi <= lo)."""
    per = -(-n // world_size)
    return rank * per, min(n, (rank + 1) * per)


def gather_frames(x_local: torch.Tensor, n: int, world_size: int, group=None, comm=None) -> torch.Tensor:
    """All n frames in order from every rank's `frame_share`: each share is padded to ceil(n / G) frames for the
    all-gather and the padding is sliced off.  One rank returns `x_local` itself."""
    if world_size == 1:
        return x_local
    pad = -(-n // world_size) - x_local.shape[0]
    if pad:
        x_local = torch.cat([x_local, x_local.new_zeros((pad,) + tuple(x_local.shape[1:]))])
    return all_gather(x_local, world_size, group, comm)[:n]


class Communicator:
    """NCCL all-gather through the C ABI (tf_comm_init / tf_allgather, include/tokenflow_b200.h): the data
    plane of the multi-GPU pivotal pass.  The 128-byte NCCL id travels over torch.distributed (control
    plane), the collectives themselves are enqueued by the library on the current CUDA stream."""

    def __init__(self, world_size: int, rank: int, group=None):
        import torch.distributed as dist
        self.lib = load_library()
        self.world_size, self.rank = world_size, rank
        idbuf = (ctypes.c_uint8 * TF_COMM_ID_BYTES)()
        if rank == 0:
            _check(self.lib, self.lib.tf_comm_unique_id(idbuf), "tf_comm_unique_id")
        t = torch.tensor(list(idbuf), dtype=torch.uint8)
        if dist.get_backend(group) == "nccl":
            t = t.cuda()
        dist.broadcast(t, src=0, group=group)
        raw = bytes(t.cpu().tolist())
        handle = ctypes.c_void_p()
        _check(self.lib, self.lib.tf_comm_init(ctypes.create_string_buffer(raw, TF_COMM_ID_BYTES), world_size, rank,
                                               ctypes.byref(handle)), "tf_comm_init")
        self.handle = handle

    def all_gather(self, t: torch.Tensor) -> torch.Tensor:
        # tf_allgather reads numel * esz bytes from the pointer: it must be device memory of this rank's GPU, dense
        if not t.is_cuda or t.device.index != torch.cuda.current_device():
            raise TokenflowB200Error(f"Communicator.all_gather needs a tensor on the current CUDA device, got one on "
                                     f"{t.device}")
        t = t.contiguous()
        out = torch.empty((self.world_size * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        _check(self.lib, self.lib.tf_allgather(self.handle, t.data_ptr(), out.data_ptr(), t.numel() * t.element_size(),
                                               torch.cuda.current_stream().cuda_stream), "tf_allgather")
        return out

    def destroy(self):
        if self.handle:
            self.lib.tf_comm_destroy(self.handle)
            self.handle = None
