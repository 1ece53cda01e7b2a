"""ctypes binding of libtokenflow_b200.so (include/tokenflow_b200.h) and the op layer the hooks call.

`CudaOps` is the product and the only op implementation in this package: every method enqueues a
hand-written sm_90a kernel on the current CUDA stream through the C ABI.  There is no CPU or
PyTorch fallback — constructing `CudaOps` without the built library or without a CUDA device
raises, loudly.  (Tests substitute an oracle-backed op object through
`tokenflow_utils._install_ops_for_testing`; that object lives under `oracle/`, not here.)
"""
from __future__ import annotations

import ctypes
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
    "tf_ext_attn_fwd_table": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p,
                                             ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_int, _c_i32p,
                                             _c_i32p, _c_i32p, _c_i32p, _c_i32p, ctypes.c_int, ctypes.c_int,
                                             ctypes.c_int, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p]),
    "tf_group_norm_nhwc_workspace": (ctypes.c_int64, [ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int]),
    "tf_group_norm_nhwc": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p,
                                          ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int,
                                          ctypes.c_float, ctypes.c_int, ctypes.c_void_p, ctypes.c_int64,
                                          ctypes.c_void_p, ctypes.c_void_p]),
    "tf_group_norm_nhwc_g4_workspace": (ctypes.c_int64, [ctypes.c_int64, ctypes.c_int64, ctypes.c_int, ctypes.c_int]),
    "tf_group_norm_nhwc_g4": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64,
                                             ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_int,
                                             ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
    "tf_frames_to_nhwc": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
    "tf_nhwc_to_frames": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
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
    def _check(self, status: int, what: str):
        if status != 0:
            msg = self.lib.tf_last_error().decode(errors="replace")
            raise TokenflowB200Error(f"{what} failed (status {status}): {msg}")

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

    def _timed(self, name: str, work: float, fn):
        if self._timing is None:
            return fn()
        ext = torch.cuda.is_current_stream_capturing()    # inside a CUDA-graph capture: event-record NODES
        start = torch.cuda.Event(enable_timing=True, external=ext)
        end = torch.cuda.Event(enable_timing=True, external=ext)
        start.record()
        out = fn()
        end.record()
        self._timing.append((name, float(work), start, end))
        return out

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
        """[..., dim] fp32/fp16 → fp16 unit rows (reference util.py:66-67 + autocast fp16 cast)."""
        if x.dtype not in (torch.float32, torch.float16):
            x = x.float()
        dim = x.shape[-1]
        x2 = x.reshape(-1, dim)
        if x2.stride(-1) != 1 or x2.stride(0) % 4 or x2.data_ptr() % 16:
            x2 = x2.clone(memory_format=torch.contiguous_format)     # rows the kernel's loads cannot address
        out = torch.empty(x2.shape, dtype=torch.float16, device=x.device)
        nbytes = x2.shape[0] * dim * (x2.element_size() + 2)
        self._timed("tf_unit_rows", nbytes, lambda: self._check(
            self.lib.tf_unit_rows(x2.data_ptr(), int(x2.dtype == torch.float32), x2.shape[0], dim,
                                  x2.stride(0), out.data_ptr(), self._stream()), "tf_unit_rows"))
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
        pass over the source stream (reference tokenflow_utils.py:323 + util.py:66-67)."""
        dim = x.shape[-1]
        if not self._ln_fusable(x, norm):
            return self.unit_rows(norm(x))                       # shapes the fused kernel does not cover
        gamma, beta = self._affine_f32(norm, x.device)
        x2 = x.reshape(-1, dim)
        if x2.stride(-1) != 1 or x2.stride(0) % 8 or x2.data_ptr() % 16:
            x2 = x2.clone(memory_format=torch.contiguous_format)     # rows the kernel's 16-byte loads cannot address
        out = torch.empty(x2.shape, dtype=torch.float16, device=x.device)
        self._timed("tf_layernorm_unit_rows", x2.shape[0] * dim * 4, lambda: self._check(
            self.lib.tf_layernorm_unit_rows(x2.data_ptr(), x2.shape[0], dim, x2.stride(0), gamma.data_ptr(),
                                            beta.data_ptr(), float(norm.eps), out.data_ptr(), self._stream()),
            "tf_layernorm_unit_rows"))
        return out.view(*x.shape)

    def layernorm_rows(self, x: torch.Tensor, norm: torch.nn.LayerNorm, n_unit: int,
                       y_out: Optional[torch.Tensor] = None, unit_out: Optional[torch.Tensor] = None):
        """Pivotal-pass norm1 fused with its two consumers: x [b, S, dim] fp16 → (y, unit) with
        y = fp16(LN(x)) [b, S, dim] (the QKV GEMM operand) and unit = fp16 unit rows of LN(x) for the first
        `n_unit` samples [n_unit, S, dim] (the pivot features of the NN field) — one read of x
        (reference tokenflow_utils.py:323 -> :120-122, :326-327, util.py:66-67).  `y_out` / `unit_out` may be
        views into packed buffers (last dim contiguous, row pitch a multiple of 8)."""
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
        x2 = x.reshape(-1, dim)
        if x2.stride(-1) != 1 or x2.stride(0) % 8 or x2.data_ptr() % 16:
            x2 = x2.clone(memory_format=torch.contiguous_format)     # rows the kernel's 16-byte loads cannot address
        y = torch.empty((b, S, dim), dtype=torch.float16, device=x.device) if y_out is None else y_out
        unit = None
        if n_unit:
            unit = torch.empty((n_unit, S, dim), dtype=torch.float16, device=x.device) if unit_out is None else unit_out
        def pitch(t):      # row pitch of a [.., S, dim] view whose rows are equally spaced
            assert t.stride(-1) == 1 and t.stride(-2) % 8 == 0 and (t.shape[0] <= 1 or t.stride(0) == S * t.stride(-2))
            return t.stride(-2)
        self._timed("tf_layernorm_rows", x2.shape[0] * dim * 4 + n_unit * S * dim * 2, lambda: self._check(
            self.lib.tf_layernorm_rows(x2.data_ptr(), x2.shape[0], dim, x2.stride(0), gamma.data_ptr(), beta.data_ptr(),
                                       float(norm.eps), y.data_ptr(), pitch(y),
                                       unit.data_ptr() if unit is not None else None,
                                       pitch(unit) if unit is not None else dim, n_unit * S, self._stream()),
            "tf_layernorm_rows"))
        return y, unit

    def cfg_ddim(self, eps_uncond: torch.Tensor, eps_cond: torch.Tensor, x: torch.Tensor, coef: torch.Tensor,
                 guidance: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Classifier-free guidance + DDIM update (reference run_tokenflow_pnp.py:213-217) in one pass;
        `coef` = device fp32 [4]: sqrt(1-a_t), 1/sqrt(a_t), sqrt(a_prev), sqrt(1-a_prev)."""
        assert eps_uncond.dtype == eps_cond.dtype == x.dtype == torch.float16 and coef.dtype == torch.float32
        eu, ec, xx = (t if t.is_contiguous() else t.contiguous() for t in (eps_uncond, eps_cond, x))
        assert eu.shape == ec.shape == xx.shape
        if out is None:
            out = torch.empty_like(xx)
        n = xx.numel()
        self._timed("tf_cfg_ddim", n * 8.0, lambda: self._check(
            self.lib.tf_cfg_ddim(eu.data_ptr(), ec.data_ptr(), xx.data_ptr(), coef.data_ptr(), float(guidance), n,
                                 out.data_ptr(), self._stream()), "tf_cfg_ddim"))
        return out

    def ddim(self, eps: torch.Tensor, x: torch.Tensor, coef: torch.Tensor,
             out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Guidance-free DDIM update of the inversion stage (reference preprocess.py:217-225 / :251-260);
        `coef` = device fp32 [4] (s1, inv_s2, s3, s4), see include/tokenflow_b200.h.  `out` may be `x` (in place)."""
        assert eps.dtype == x.dtype == torch.float16 and coef.dtype == torch.float32 and coef.is_cuda
        assert eps.shape == x.shape
        e = eps if eps.is_contiguous() else eps.contiguous()
        if out is None:
            out = torch.empty_like(x, memory_format=torch.contiguous_format)
        assert out.shape == x.shape and out.dtype == torch.float16 and out.is_contiguous() and x.is_contiguous()
        n = x.numel()
        self._timed("tf_ddim", n * 6.0, lambda: self._check(
            self.lib.tf_ddim(e.data_ptr(), x.data_ptr(), coef.data_ptr(), n, out.data_ptr(), self._stream()), "tf_ddim"))
        return out

    def nn_field(self, x_unit: torch.Tensor, piv_unit: torch.Tensor, kf_a: Sequence[int],
                 kf_b: Sequence[int]) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """x_unit [F,S,dim], piv_unit [K,S,dim] fp16 unit rows → int32 idx_a, idx_b [F,S]
        (reference tokenflow_utils.py:335-343).  The idx_b rows of frames with kf_b < 0 are left unwritten
        (idx_b is None when no frame has a second keyframe)."""
        F_, S, dim = x_unit.shape
        K = piv_unit.shape[0]
        assert x_unit.dtype == torch.float16 and piv_unit.dtype == torch.float16
        x_unit = x_unit.contiguous()
        piv_unit = piv_unit.contiguous()
        idx_a = torch.empty((F_, S), dtype=torch.int32, device=x_unit.device)
        any_b = any(int(b) >= 0 for b in kf_b)
        idx_b = torch.empty((F_, S), dtype=torch.int32, device=x_unit.device) if any_b else None
        pairs = F_ + sum(1 for b in kf_b if int(b) >= 0)
        self._timed("tf_nn_field", 2.0 * pairs * S * S * dim, lambda: self._check(self.lib.tf_nn_field(
            x_unit.data_ptr(), piv_unit.data_ptr(), _i32(kf_a), _i32(kf_b), F_, S, dim, K, idx_a.data_ptr(),
            idx_b.data_ptr() if idx_b is not None else None, self._stream()), "tf_nn_field"))
        return idx_a, idx_b

    def propagate(self, A: torch.Tensor, idx_a: torch.Tensor, idx_b: Optional[torch.Tensor],
                  kf_a: Sequence[int], kf_b: Sequence[int], w: Sequence[float],
                  residual: Optional[torch.Tensor], out_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
        """A [3,K,S,dim] fp16; idx [F,S] int32; residual [3F,S,dim] fp16 or None → [3F,S,dim]
        (reference tokenflow_utils.py:361-397)."""
        three, K, S, dim = A.shape
        out_dtype = torch.float16 if out_dtype is None else out_dtype
        if A.dtype != torch.float16 or not A.is_contiguous():
            A = A.to(torch.float16).contiguous()
        assert three == 3
        F_ = idx_a.shape[0]
        if residual is not None:
            residual = residual.to(torch.float16).contiguous().view(3, F_, S, dim)
        out = torch.empty((3, F_, S, dim), dtype=out_dtype, device=A.device)
        assert out_dtype in (torch.float16, torch.float32)
        self._timed("tf_propagate", propagate_bytes(F_, S, dim, kf_a, kf_b, residual is not None,
                                                    out.element_size()), lambda: self._check(
            self.lib.tf_propagate(
                A.data_ptr(), idx_a.data_ptr(), idx_b.data_ptr() if idx_b is not None else None, _i32(kf_a),
                _i32(kf_b), _f32(w), F_, S, dim, K, residual.data_ptr() if residual is not None else None,
                out.data_ptr(), int(out_dtype == torch.float32), self._stream()), "tf_propagate"))
        return out.view(3 * F_, S, dim)

    def ext_attn(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, scale: float,
                 inject: bool) -> torch.Tensor:
        """q,k,v [3n,S,dim] fp16 (same token stride) → [3n,S,dim] fp16, before to_out
        (reference tokenflow_utils.py:124-197 / :234-279)."""
        b, S, dim = q.shape
        n = b // 3
        d = dim // heads
        q, k, v = (t if t.dtype == torch.float16 else t.to(torch.float16) for t in (q, k, v))
        strides = {(t.stride(0), t.stride(1), t.stride(2)) for t in (q, k, v)}
        tok = q.stride(1)
        if len(strides) != 1 or q.stride(2) != 1 or q.stride(0) != S * tok:
            q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
            tok = dim
        out = torch.empty((b, S, dim), dtype=torch.float16, device=q.device)
        flops = 4.0 * n * S * S * dim * (2 * n + 1)        # QK^T + PV; source: S keys, uncond+cond: n*S keys
        self._timed("tf_ext_attn", flops, lambda: self._check(
            self.lib.tf_ext_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), tok, n, S, heads, d,
                                     float(scale), int(bool(inject)), out.data_ptr(), self._stream()),
            "tf_ext_attn_fwd"))
        return out

    @staticmethod
    def _slab_view(t: torch.Tensor):
        """(tensor, token stride) of a [slabs, S, dim] fp16 operand the kernels can address in place: last dim
        contiguous, slabs S tokens apart (a column slice of a packed [slabs, S, n*dim] buffer qualifies)."""
        if t.dtype != torch.float16:
            t = t.to(torch.float16)
        S = t.shape[1]
        if t.stride(2) != 1 or t.stride(1) % 8 or (t.shape[0] > 1 and t.stride(0) != S * t.stride(1)) \
                or t.data_ptr() % 16:
            t = t.contiguous()
        return t, t.stride(1)

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
        (q, q_tok), (k, k_tok), (v, v_tok) = self._slab_view(q), self._slab_view(k), self._slab_view(v)
        if k_tok != v_tok:
            k, v = k.contiguous(), v.contiguous()
            k_tok = v_tok = dim
        n_out = len(table)
        out = torch.empty((n_out, nrows, dim), dtype=torch.float16, device=q.device)
        rows_eff = max(0, min(S, row0 + nrows) - row0)
        flops = sum(4.0 * rows_eff * (nkv * S) * dim for (_, _, _, nkv) in table)
        self._timed("tf_ext_attn", flops, lambda: self._check(self.lib.tf_ext_attn_fwd_rows(
            q.data_ptr(), q.shape[0], q_tok, k.data_ptr(), v.data_ptr(), k.shape[0], k_tok, n_out,
            _i32(range(n_out)), _i32([t[0] for t in table]), _i32([t[1] for t in table]),
            _i32([t[2] for t in table]), _i32([t[3] for t in table]), S, heads, d, float(scale), int(row0), nrows,
            out.data_ptr(), self._stream()), "tf_ext_attn_fwd_rows"))
        return out

    # -- UNet body ----------------------------------------------------------------------------
    @staticmethod
    def _group_norm_nhwc_operands(x: torch.Tensor, norm: torch.nn.GroupNorm) -> bool:
        """CUDA fp16 channels_last [N, C, H, W] with C % 8 == 0, C <= 4096, groups dividing C and fp16 affine
        parameters: what both GroupNorm entry points need besides their channels per group."""
        if not (x.is_cuda and x.dtype == torch.float16 and x.dim() == 4
                and x.is_contiguous(memory_format=torch.channels_last)):
            return False
        c, g = x.shape[1], norm.num_groups
        w, b = norm.weight, norm.bias
        return (c % 8 == 0 and c <= 4096 and c % g == 0 and w is not None and b is not None
                and w.dtype == b.dtype == torch.float16 and w.is_contiguous() and b.is_contiguous())

    @staticmethod
    def group_norm_nhwc_supported(x: torch.Tensor, norm: torch.nn.GroupNorm) -> bool:
        """Shapes tf_group_norm_nhwc covers: CUDA fp16 channels_last [N, C, H, W] with C % 8 == 0, C <= 4096, at least
        8 channels per group and fp16 affine parameters."""
        return CudaOps._group_norm_nhwc_operands(x, norm) and x.shape[1] // norm.num_groups >= 8

    @staticmethod
    def group_norm_nhwc_g4_supported(x: torch.Tensor, norm: torch.nn.GroupNorm) -> bool:
        """Shapes tf_group_norm_nhwc_g4 covers: the same operands with exactly 4 channels per group."""
        return CudaOps._group_norm_nhwc_operands(x, norm) and x.shape[1] == 4 * norm.num_groups

    def group_norm_nhwc(self, x: torch.Tensor, norm: torch.nn.GroupNorm, bias: Optional[torch.Tensor] = None,
                        silu: bool = False) -> torch.Tensor:
        """[SiLU](GroupNorm(x [+ bias[:, :, None, None]])) of a channels_last fp16 [N, C, H, W] tensor, channels_last
        out, with the eager fp16 rounding sequence.  `bias` is fp16 [N, C] or [1, C] (the resnet's time-embedding
        projection).  Two launches; the statistics workspace comes from the caching allocator on this stream."""
        n, c, h, w = x.shape
        if bias is not None:
            assert bias.dtype == torch.float16 and bias.dim() == 2 and bias.shape[1] == c and bias.shape[0] in (1, n)
            if bias.stride(1) != 1 or bias.stride(0) % 8 or bias.data_ptr() % 16:
                bias = bias.contiguous()
            bias_stride = 0 if bias.shape[0] == 1 else bias.stride(0)
        ws_bytes = int(self.lib.tf_group_norm_nhwc_workspace(n, h * w, c, norm.num_groups))
        if ws_bytes < 0:
            self._check(3, "tf_group_norm_nhwc_workspace")
        ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=x.device)
        out = torch.empty_like(x, memory_format=torch.channels_last)
        work = 3.0 * x.numel() * 2 + (n * c * 2 if bias is not None else 0)
        self._timed("tf_group_norm", work, lambda: self._check(self.lib.tf_group_norm_nhwc(
            x.data_ptr(), bias.data_ptr() if bias is not None else None, bias_stride if bias is not None else 0,
            norm.weight.data_ptr(), norm.bias.data_ptr(), n, h * w, c, norm.num_groups, float(norm.eps), int(bool(silu)),
            ws.data_ptr(), ws.numel(), out.data_ptr(), self._stream()), "tf_group_norm_nhwc"))
        return out

    def group_norm_nhwc_g4(self, x: torch.Tensor, norm: torch.nn.GroupNorm, silu: bool = False) -> torch.Tensor:
        """[SiLU](GroupNorm(x)) of a channels_last fp16 [N, C, H, W] tensor with 4 channels per group (no bias add),
        channels_last out, with the eager fp16 rounding sequence; the statistics workspace comes from the caching
        allocator on this stream."""
        n, c, h, w = x.shape
        ws_bytes = int(self.lib.tf_group_norm_nhwc_g4_workspace(n, h * w, c, norm.num_groups))
        if ws_bytes < 0:
            self._check(1, "tf_group_norm_nhwc_g4_workspace")
        ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=x.device)
        out = torch.empty_like(x, memory_format=torch.channels_last)
        self._timed("tf_group_norm_g4", 3.0 * x.numel() * 2, lambda: self._check(self.lib.tf_group_norm_nhwc_g4(
            x.data_ptr(), norm.weight.data_ptr(), norm.bias.data_ptr(), n, h * w, c, norm.num_groups, float(norm.eps),
            int(bool(silu)), ws.data_ptr(), ws.numel(), out.data_ptr(), self._stream()), "tf_group_norm_nhwc_g4"))
        return out

    def frames_to_nhwc(self, frames: torch.Tensor) -> torch.Tensor:
        """uint8 RGB frames [N, H, W, 3] (CUDA) -> the encoder input 2 * ToTensor(frames) - 1 as a channels_last fp16
        [N, 3, H, W] tensor, bit-equal to the reference's host conversion followed by the fp16 ops."""
        assert frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[-1] == 3 and frames.is_cuda
        if not frames.is_contiguous() or frames.data_ptr() % 16:
            frames = frames.contiguous()
        n, h, w, _ = frames.shape
        out = torch.empty((n, 3, h, w), dtype=torch.float16, device=frames.device, memory_format=torch.channels_last)
        self._timed("tf_frames_to_nhwc", 3.0 * n * h * w, lambda: self._check(self.lib.tf_frames_to_nhwc(
            frames.data_ptr(), n * h * w, out.data_ptr(), self._stream()), "tf_frames_to_nhwc"))
        return out

    def nhwc_to_frames(self, x: torch.Tensor) -> torch.Tensor:
        """fp16 decoder output [N, 3, H, W] -> uint8 frames [N, H, W, 3], bit-equal to
        `((x / 2 + 0.5).clamp(0, 1) * 255).to(torch.uint8)` in fp16 (NaN -> 0)."""
        assert x.dtype == torch.float16 and x.dim() == 4 and x.shape[1] == 3 and x.is_cuda
        if not x.is_contiguous(memory_format=torch.channels_last) or x.data_ptr() % 16:
            x = x.contiguous(memory_format=torch.channels_last)
        n, _, h, w = x.shape
        out = torch.empty((n, h, w, 3), dtype=torch.uint8, device=x.device)
        self._timed("tf_nhwc_to_frames", 3.0 * n * h * w, lambda: self._check(self.lib.tf_nhwc_to_frames(
            x.data_ptr(), n * h * w, out.data_ptr(), self._stream()), "tf_nhwc_to_frames"))
        return out

    def geglu(self, xh: torch.Tensor, gate: torch.Tensor) -> torch.Tensor:
        """xh * gelu(gate) of two fp16 tensors of one shape (the GEGLU GEMM outputs), bit-equal to the eager product."""
        assert xh.dtype == gate.dtype == torch.float16 and xh.shape == gate.shape
        xh, gate = (t if t.is_contiguous() and t.data_ptr() % 16 == 0 else t.contiguous() for t in (xh, gate))
        out = torch.empty_like(xh)
        n = xh.numel()
        self._timed("tf_geglu", 3.0 * n * 2, lambda: self._check(
            self.lib.tf_geglu(xh.data_ptr(), gate.data_ptr(), n, out.data_ptr(), self._stream()), "tf_geglu"))
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
            self._check(self.lib.tf_comm_unique_id(idbuf), "tf_comm_unique_id")
        t = torch.tensor(list(idbuf), dtype=torch.uint8)
        if dist.get_backend(group) == "nccl":
            t = t.cuda()
        dist.broadcast(t, src=0, group=group)
        raw = bytes(t.cpu().tolist())
        handle = ctypes.c_void_p()
        self._check(self.lib.tf_comm_init(ctypes.create_string_buffer(raw, TF_COMM_ID_BYTES), world_size, rank,
                                          ctypes.byref(handle)), "tf_comm_init")
        self.handle = handle

    def _check(self, status, what):
        if status != 0:
            raise TokenflowB200Error(f"{what} failed (status {status}): "
                                     f"{self.lib.tf_last_error().decode(errors='replace')}")

    def all_gather(self, t: torch.Tensor) -> torch.Tensor:
        t = t.contiguous()
        out = torch.empty((self.world_size * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        self._check(self.lib.tf_allgather(self.handle, t.data_ptr(), out.data_ptr(), t.numel() * t.element_size(),
                                          torch.cuda.current_stream().cuda_stream), "tf_allgather")
        return out

    def destroy(self):
        if self.handle:
            self.lib.tf_comm_destroy(self.handle)
            self.handle = None
