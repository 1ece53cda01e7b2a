"""fp64 check of a LoRA merge (`tokenflow_b200.lora.merge`) into 16-bit weights.

For a weight W and the LoRAs i = 1..n of its module (up U_i [out, r_i], down D_i [r_i, in·kh·kw], c_i = s_i·α_i/r_i),
the exact merged value is v = W + Σ_i c_i·(U_i @ D_i), recomputed here in fp64 from the file's tensors and the weight
before the merge.  The merge computes v in fp32 and rounds once to the weight's dtype, so each output must be the
correctly rounded (nearest, ties to even) value of v, except where v lies within δ of a rounding midpoint: there
every value between the roundings of v − δ and v + δ passes (both neighbours of the midpoint).  Those cases are
counted and capped.

δ, per element, bounds |v_fp32 − v| + |v_fp64 − v|.  With u = 2^-24 (fp32), γ_r = r·u / (1 − r·u), M_i = |U_i| @ |D_i|
and A = |W| + Σ_i |c_i|·M_i:

  * fl32(U_i @ D_i), in any summation order, with or without FMA, is within γ_r·M_i of U_i @ D_i;
  * c_i rounded to fp32 moves c_i·P_i by at most u·|c_i|·M_i, so |ĉ_i·p̂_i − c_i·P_i| ≤ |c_i|·M_i·((1 + u)·γ_r + u);
  * the product ĉ·p̂ and the sum into the accumulator round twice, within (2u + u²)·A·(1 + η);

  δ32 = 1.01 · [ Σ_i |c_i|·M_i·(γ_{r_i} + 2u) + 3·n·u·A ]

where 1.01 ≥ 1 + η covers the second-order growth of the accumulator for any rank and LoRA count a file has.  The
fp64 evaluation here adds δ64 = 1.01·(max r_i + n + 2)·2^-53·A.

The LoRA files are read in the kohya layout (`lora_unet_*`, `lora_te_*`), with a name table of this module's own.
"""
from __future__ import annotations

from functools import lru_cache
from typing import Dict, List, Sequence, Tuple

import torch
import torch.nn as nn

U32 = 2.0 ** -24
U64 = 2.0 ** -53


@lru_cache(maxsize=None)
def _grid(dtype: torch.dtype) -> Tuple[torch.Tensor, torch.Tensor]:
    """(every finite value of the 16-bit `dtype` in increasing order as fp64, whether its last mantissa bit is 0)."""
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    vals = bits.view(dtype).to(torch.float64)
    keep = torch.isfinite(vals)
    vals, bits = vals[keep], bits[keep]
    order = torch.argsort(vals, stable=True)
    vals, bits = vals[order], bits[order]
    first = torch.ones_like(vals, dtype=torch.bool)
    first[1:] = vals[1:] != vals[:-1]                      # -0 and +0: one value, both even
    return vals[first], (bits[first] & 1) == 0


def round_to(x: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """fp64 `x` rounded to the nearest value of the 16-bit `dtype`, ties to even, as fp64 (the result of one
    correctly rounded conversion; torch's fp64 -> fp16 cast goes through fp32)."""
    vals, even = _grid(dtype)
    vals, even = vals.to(x.device), even.to(x.device)
    if not (x.abs() <= vals[-1]).all():
        raise AssertionError(f"a merged value overflows {dtype}")
    i = torch.searchsorted(vals, x.contiguous()).clamp(1, vals.numel() - 1)
    lo, hi = vals[i - 1], vals[i]
    d_lo, d_hi = x - lo, hi - x
    return torch.where((d_hi < d_lo) | ((d_hi == d_lo) & even[i]), hi, lo)


def kohya_terms(tensors: Dict[str, torch.Tensor], scale: float, unet: nn.Module,
                text_encoder: nn.Module) -> Dict[Tuple[str, str], Tuple[float, torch.Tensor, torch.Tensor]]:
    """{(model, module path): (c = scale·α/r, up, down)} of a kohya file's tensors; a missing alpha is α = r."""
    names = {}
    for model, prefix, net in (("unet", "lora_unet_", unet), ("text_encoder", "lora_te_", text_encoder)):
        for name, _ in net.named_modules():
            names[prefix + name.replace(".", "_")] = (model, name)
    out = {}
    for stem in {k.split(".", 1)[0] for k in tensors}:
        down, up = tensors[stem + ".lora_down.weight"], tensors[stem + ".lora_up.weight"]
        r = down.shape[0]
        alpha = float(tensors[stem + ".alpha"]) if stem + ".alpha" in tensors else float(r)
        out[names[stem]] = (scale * alpha / r, up, down)
    return out


def reference(w0: torch.Tensor, terms: Sequence[Tuple[float, torch.Tensor, torch.Tensor]]):
    """(v, δ) in fp64 on w0's device: the exact merged value and the bound of the module docstring."""
    dev = w0.device
    w = w0.to(torch.float64)
    v, cm, gam = w.clone(), torch.zeros_like(w), torch.zeros_like(w)
    r_max = 0
    for c, up, down in terms:
        r = down.shape[0]
        r_max = max(r_max, r)
        u = up.to(dev, torch.float64).reshape(w.shape[0], r)
        d = down.to(dev, torch.float64).reshape(r, -1)
        m = (u.abs() @ d.abs()).reshape(w.shape) * abs(c)
        v += c * (u @ d).reshape(w.shape)
        gamma = r * U32 / (1 - r * U32)
        cm += m
        gam += m * (gamma + 2 * U32)
    a = w.abs() + cm
    n = len(terms)
    delta = 1.01 * (gam + 3 * n * U32 * a) + 1.01 * (r_max + n + 2) * U64 * a
    return v, delta


def check_weight(out: torch.Tensor, v: torch.Tensor, delta: torch.Tensor) -> Tuple[int, int]:
    """(elements near a midpoint, elements) of one merged weight; AssertionError where an output is not a value the
    merge may produce."""
    o = out.detach().to(torch.float64)
    a, b = round_to(v - delta, out.dtype), round_to(v + delta, out.dtype)
    near = a != b
    ok = torch.where(near, (a <= o) & (o <= b), o == round_to(v, out.dtype))
    if not ok.all():
        i = int((~ok).flatten().nonzero()[0])
        raise AssertionError(f"{int((~ok).sum())} of {ok.numel()} outputs are not the rounded merge: first at flat "
                             f"index {i}, got {o.flatten()[i].item()!r}, exact {v.flatten()[i].item()!r} "
                             f"(δ {delta.flatten()[i].item():.3g})")
    return int(near.sum()), ok.numel()


def check_merge(unet: nn.Module, text_encoder: nn.Module, before: Dict[Tuple[str, str], torch.Tensor],
                files: List[Tuple[Dict[str, torch.Tensor], float]], max_near_fraction: float = 0.02) -> Tuple[int, int]:
    """Check every Linear and Conv2d weight of the models after a merge of the kohya `files` [(tensors, scale)] in
    order: a module no file names keeps `before`'s bits, every other passes `check_weight`, and the near-midpoint
    cases are at most `max_near_fraction` of the merged elements.  Returns (near-midpoint cases, merged elements)."""
    terms: Dict[Tuple[str, str], list] = {}
    for tensors, scale in files:
        for key, term in kohya_terms(tensors, scale, unet, text_encoder).items():
            terms.setdefault(key, []).append(term)
    near = total = 0
    for model, net in (("unet", unet), ("text_encoder", text_encoder)):
        for name, module in net.named_modules():
            if not isinstance(module, (nn.Linear, nn.Conv2d)):
                continue
            w0 = before[(model, name)]
            if (model, name) not in terms:
                assert torch.equal(module.weight, w0), f"{model} {name} changed but no LoRA names it"
                continue
            try:
                k, n = check_weight(module.weight, *reference(w0, terms[(model, name)]))
            except AssertionError as e:
                raise AssertionError(f"{model} {name}: {e}") from None
            near, total = near + k, total + n
    assert total == sum(before[k].numel() for k in terms), "a LoRA names a module the models do not have"
    assert near <= max_near_fraction * total, f"{near} of {total} outputs lie within δ of a rounding midpoint"
    return near, total


def weights(unet: nn.Module, text_encoder: nn.Module) -> Dict[Tuple[str, str], torch.Tensor]:
    """{(model, path): a copy of the weight} of every Linear and Conv2d: the `before` of `check_merge`."""
    return {(model, name): m.weight.detach().clone()
            for model, net in (("unet", unet), ("text_encoder", text_encoder))
            for name, m in net.named_modules() if isinstance(m, (nn.Linear, nn.Conv2d))}
