"""ORACLE (test infrastructure) — how far the native UNet body moves a seeded edit, against a noise floor.

The same seeded PnP edit (same weights, latents and keyframes) runs for a few steps in four arms:

  (a) native   channels_last body, GroupNorm sites and GEGLU on tf_group_norm_nhwc / tf_geglu;
  (b) aten_cl  channels_last body on the ATen ops (`ops._BODY_OPS = None`);
  (c) aten_nchw NCHW body on the ATen ops (`bench.py --no-channels-last`);
  (d) aten_fp32_stats  channels_last body on the ATen ops, but every GroupNorm site evaluated on the fp32-upcast
      input and rounded to fp16 once (no fp16 storage of the group mean and rstd): a more accurate GroupNorm, which
      differs from ATen's fp16 one only in last-bit rounding.

(b) and (c) could differ only through the convolution algorithms cuDNN picks for each layout.  On an H100 they
give bit-identical latents (rel-L2 0), so the layout is no noise floor.  rel-L2(b, d) is what a last-bit difference
of the GroupNorm sites alone, with nothing wrong on either side, does to the edit after that many steps.  A correct
native body sits at that floor, rel-L2(a, b) ~ rel-L2(b, d); a GroupNorm defect sits above it.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def _norm_act_fp32_stats(norm, x, bias=None, silu=True):
    """`sd_unet.norm_act` with the GroupNorm evaluated in fp32 and rounded once (the add and the SiLU stay fp16)."""
    if bias is not None:
        x = x + bias[:, :, None, None]
    y = F.group_norm(x.float(), norm.num_groups, norm.weight.float(), norm.bias.float(), norm.eps).to(x.dtype)
    return F.silu(y) if silu else y


def _rel(a: torch.Tensor, b: torch.Tensor) -> float:
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def body_drift(kind: str = "sd15", n_frames: int = 8, batch: int = 4, latent: int = 64, steps: int = 8,
               n_timesteps: int = 50, seed: int = 1) -> dict:
    """Run the four arms for `steps` denoising steps of an `n_timesteps` PnP schedule; return the final latents'
    pairwise relative L2 differences and whether every arm drew the same keyframes."""
    from tokenflow_b200 import ops as ops_module
    from tokenflow_b200 import sd_unet, tokenflow_utils as tfu
    from tokenflow_b200.editor import TokenFlowEditor, synthetic_inputs
    from tokenflow_b200.scheduler import DDIMScheduler

    device = torch.device("cuda")
    tfu._install_ops_for_testing(None)
    native_ops = ops_module.body_ops()
    assert native_ops is not None, "the native body needs the library and an sm_90 device"
    unet = sd_unet.build_unet(kind, seed=seed, device=device, dtype=torch.float16, init_on_device=True)
    x0, text, pnp, src = synthetic_inputs(n_frames, latent, unet.config.cross_attention_dim, n_timesteps, seed=seed,
                                          device=device, dtype=torch.float16)
    cfg = {"n_frames": n_frames, "batch_size": batch, "n_timesteps": n_timesteps, "guidance_scale": 7.5, "mode": "pnp",
           "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "start": 0.9, "fused_pass": True, "cuda_graph": False,
           "keyframe_seed": seed}
    arms = {"native": (torch.channels_last, native_ops), "aten_cl": (torch.channels_last, None),
            "aten_nchw": (torch.contiguous_format, None), "aten_fp32_stats": (torch.channels_last, None)}
    out, keyframes = {}, {}
    saved = ops_module._BODY_OPS, sd_unet.norm_act, tfu.norm_act
    try:
        for name, (fmt, body) in arms.items():
            ops_module._BODY_OPS = body
            sd_unet.norm_act = tfu.norm_act = _norm_act_fp32_stats if name == "aten_fp32_stats" else saved[1]
            unet.to(memory_format=fmt)
            ed = TokenFlowEditor(unet, DDIMScheduler(), tfu, dict(cfg), text, pnp, source_latents=lambda t: src[t])
            ed.init_method()
            x = x0.clone()
            with torch.no_grad():
                for i in range(steps):
                    x = ed.step_index(x, i)
            out[name] = x.float()
            keyframes[name] = ed.keyframe_log
    finally:
        ops_module._BODY_OPS, sd_unet.norm_act, tfu.norm_act = saved
    return {"kind": kind, "n_frames": n_frames, "batch": batch, "latent": latent, "steps": steps,
            "native_vs_aten_cl": _rel(out["native"], out["aten_cl"]),
            "aten_cl_vs_aten_nchw": _rel(out["aten_cl"], out["aten_nchw"]),
            "native_vs_aten_nchw": _rel(out["native"], out["aten_nchw"]),
            "aten_cl_vs_aten_fp32_stats": _rel(out["aten_cl"], out["aten_fp32_stats"]),
            "native_vs_aten_fp32_stats": _rel(out["native"], out["aten_fp32_stats"]),
            "native_vs_aten_cl_max_abs": (out["native"] - out["aten_cl"]).abs().max().item(),
            "absmax": out["aten_cl"].abs().max().item(),
            "keyframes_equal": all(k == keyframes["native"] for k in keyframes.values()),
            "finite": all(bool(torch.isfinite(v).all()) for v in out.values())}
