"""ORACLE (test infrastructure) — the two latent updates for a v-prediction model, restated in numpy from a coefficient
row: `tf_cfg_ddim_v` and `tf_ddim_v` (include/tokenflow_b200.h, tokenflow_b200/csrc/tf_cfg_ddim.cu).

The same guidance as `tf_cfg_ddim` (oracle/latent_step.py), then diffusers' v-branch of the DDIM step (eta = 0) with the
fp32 coefficient row (a, b, c, d), each operation in fp32 on fp16 operands and rounded to fp16 (h):

    v  = h(u + h(g * h(c - u)))                                     (guidance; tf_ddim_v: v = the model output)
    p  = h(h(a * x) - h(b * v))      e = h(h(a * v) + h(b * x))      out = h(h(c * p) + h(d * e))

As in oracle/latent_step.py, numpy's IEEE binary32 arithmetic and its round-to-nearest-even float16 cast make this an
exact model of the rounding sequence that depends on neither ATen nor the kernel.
"""
from __future__ import annotations

import numpy as np

from .latent_step import _f32, _h


def vpred_half(v: np.ndarray, x: np.ndarray, coef) -> np.ndarray:
    """fp32 arrays of fp16 values -> out = h(h(c * h(h(a * x) - h(b * v))) + h(d * h(h(a * v) + h(b * x)))) as fp32."""
    a, b, c, d = (np.float32(k) for k in coef)
    with np.errstate(over="ignore", invalid="ignore"):
        p = _h(_h(a * x) - _h(b * v))
        e = _h(_h(a * v) + _h(b * x))
        return _h(_h(c * p) + _h(d * e))


def cfg_ddim_v(u, c, x, coef, guidance: float) -> np.ndarray:
    """`tf_cfg_ddim_v`: fp16 arrays (v_uncond, v_cond, latents), coef = (a, b, c, d) -> fp16."""
    u, c, x = _f32(u), _f32(c), _f32(x)
    g = np.float32(guidance)
    with np.errstate(over="ignore", invalid="ignore"):
        v = _h(u + _h(g * _h(c - u)))
    return vpred_half(v, x, coef).astype(np.float16)


def ddim_v(v, x, coef) -> np.ndarray:
    """`tf_ddim_v`: fp16 arrays (v, latents), coef = (a, b, c, d) -> fp16."""
    return vpred_half(_f32(v), _f32(x), coef).astype(np.float16)
