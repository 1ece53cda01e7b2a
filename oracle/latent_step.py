"""ORACLE (test infrastructure) — the two latent updates of the hot path, restated in numpy from a coefficient row.

`tf_cfg_ddim` (the edit's classifier-free guidance + DDIM step, reference run_tokenflow_pnp.py:213-217) and `tf_ddim`
(the inversion's guidance-free step, reference preprocess.py:224-225 / :259-260) evaluate the eager fp16 expressions
one operation at a time: each operation in fp32 on fp16 operands, its result rounded to fp16
(tokenflow_b200/csrc/tf_cfg_ddim.cu):

    d  = h(c - u)            m  = h(g * d)            e  = h(u + m)                 (guidance; u = uncond, c = cond)
    a  = h(s1 * e)           b  = h(x - a)            p  = h(b * inv_s2)            (pred_x0)
    c1 = h(s3 * p)           c2 = h(s4 * e)           out = h(c1 + c2)

with the fp32 coefficient row (s1, inv_s2, s3, s4) and the fp32 guidance g.  numpy's float32 arithmetic is IEEE
binary32 and its float32 -> float16 cast rounds to nearest even (overflow to inf, subnormals kept), so this is an exact
model of the rounding sequence that depends on neither ATen nor the kernel.  `tf_ddim` is the second and third lines
with e = eps.
"""
from __future__ import annotations

import numpy as np

#: every fp16 value, in bit-pattern order 0x0000 ... 0xFFFF
ALL_FP16 = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16)


def structured_fp16(n_normal: int = 40, seed: int = 0) -> np.ndarray:
    """The values the sweeps pair with every fp16 input: signed zeros, the smallest and largest subnormal, the smallest
    normal, +-1, +-65504, +-inf, NaN, magnitudes where g * (c - u) overflows at the guidances tested (9000 and 20000
    against g = 7.5 and 30), and `n_normal` N(0, 1) values."""
    bits = np.array([0x0000, 0x8000, 0x0001, 0x8001, 0x03FF, 0x0400], dtype=np.uint16).view(np.float16)
    special = np.array([1, -1, 65504, -65504, np.inf, -np.inf, np.nan, 9000, -9000, 20000, -20000], dtype=np.float16)
    normal = np.random.default_rng(seed).standard_normal(n_normal).astype(np.float16)
    return np.concatenate([bits, special, normal])


def _h(v: np.ndarray) -> np.ndarray:
    """Round an fp32 array to fp16 and back."""
    return v.astype(np.float16).astype(np.float32)


def _f32(a) -> np.ndarray:
    return np.asarray(a, dtype=np.float16).astype(np.float32)


def ddim_half(e: np.ndarray, x: np.ndarray, coef) -> np.ndarray:
    """fp32 arrays of fp16 values -> out = h(h(s3 * h(h(x - h(s1 * e)) * inv_s2)) + h(s4 * e)) as fp32."""
    s1, inv_s2, s3, s4 = (np.float32(c) for c in coef)
    with np.errstate(over="ignore", invalid="ignore"):
        p = _h(_h(x - _h(s1 * e)) * inv_s2)
        return _h(_h(s3 * p) + _h(s4 * e))


def cfg_ddim(u, c, x, coef, guidance: float) -> np.ndarray:
    """`tf_cfg_ddim`: fp16 arrays (eps_uncond, eps_cond, latents), coef = (s1, inv_s2, s3, s4) -> fp16."""
    u, c, x = _f32(u), _f32(c), _f32(x)
    g = np.float32(guidance)
    with np.errstate(over="ignore", invalid="ignore"):
        e = _h(u + _h(g * _h(c - u)))
    return ddim_half(e, x, coef).astype(np.float16)


def ddim(eps, x, coef) -> np.ndarray:
    """`tf_ddim`: fp16 arrays (eps, latents), coef = (s1, inv_s2, s3, s4) -> fp16."""
    return ddim_half(_f32(eps), _f32(x), coef).astype(np.float16)


def same_bits(got: np.ndarray, want: np.ndarray) -> np.ndarray:
    """Elementwise: equal fp16 bit patterns, or both NaN (whatever their payloads)."""
    got, want = np.asarray(got, np.float16), np.asarray(want, np.float16)
    return (got.view(np.uint16) == want.view(np.uint16)) | (np.isnan(got) & np.isnan(want))
