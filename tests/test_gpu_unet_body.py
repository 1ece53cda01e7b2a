"""GPU tier: the native UNet body (tf_group_norm_nhwc at every GroupNorm site, tf_geglu in every transformer block)
inside the full SD1.5 (latent 64) and SD2.1 (latent 96) UNets, fp16 channels_last, N = 2.

* Coverage: one forward makes exactly 61 `CudaOps.group_norm_nhwc` calls and 2 * 61 + 16 library launches, so no
  site falls back to ATen unnoticed.
* Real activations: every site's output passes `check_group_norm` on that site's own input (resnet norm1 + SiLU,
  temb add + norm2 + SiLU with the `time_emb_proj` bias, skip-connection concatenations whose groups straddle the
  two joined tensors, `Transformer2DModel.norm`, `conv_norm_out` + SiLU); the same input through the C ABI gives the
  same bits and a workspace that passes `check_group_norm_workspace`.
* Against fp32: the native fp16 body is as close to an fp32 run of the same weights as the ATen fp16 body.
* Drift: a seeded 8-step PnP edit moves no further from the ATen body than the ATen body moves when its GroupNorm
  sites are evaluated in fp32 and rounded once (`oracle/body_drift.py`).  The NCHW layout is run and reported too:
  on an H100 it leaves the ATen body's latents bit-identical, so it is no noise floor.
"""
import copy

import pytest
import torch

from oracle.body_drift import body_drift
from oracle.kernel_checks import check_group_norm, check_group_norm_workspace, guarded_group_norm
from tokenflow_b200 import ops as ops_module
from tokenflow_b200 import sd_unet

pytestmark = pytest.mark.gpu

SITES = 61                     # GroupNorm sites of one SD1.5 / SD2.1 forward
GEGLU_SITES = 16               # transformer blocks
# Calibrated on one H100 80GB HBM3 at a 400 W power limit.
# rel-L2(native, fp32) <= FP32_FACTOR * rel-L2(ATen, fp32); measured ratio 1.0000 (SD1.5) and 0.998 (SD2.1) in three runs
FP32_FACTOR = 1.05
# rel-L2(native, ATen) <= DRIFT_KAPPA * rel-L2(ATen, ATen with fp32 GroupNorm statistics); measured ratio 0.95-0.98 over
# seeds 1-4 at this size and 0.97 at C2
DRIFT_KAPPA = 1.25


@pytest.fixture(scope="module", params=[("sd15", 64), ("sd21", 96)], ids=["sd15", "sd21"])
def model(request):
    kind, latent = request.param
    unet = sd_unet.build_unet(kind, seed=1, device="cuda", dtype=torch.float16, init_on_device=True)
    unet = unet.to(memory_format=torch.channels_last)
    g = torch.Generator(device="cuda").manual_seed(0)
    sample = torch.randn(2, 4, latent, latent, device="cuda", generator=g).half()
    sample = sample.contiguous(memory_format=torch.channels_last)
    ctx = torch.randn(2, 77, unet.config.cross_attention_dim, device="cuda", generator=g).half()
    t = torch.tensor([501], device="cuda")
    yield kind, unet, (sample, t, ctx)
    del unet
    torch.cuda.empty_cache()


@pytest.fixture
def body_ops():
    ops = ops_module.body_ops()
    assert ops is not None, "the native body needs the library and an sm_90 device"
    return ops


def _forward(unet, inputs):
    sample, t, ctx = inputs
    with torch.no_grad():
        return unet(sample, t, encoder_hidden_states=ctx).sample


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def test_every_group_norm_site_runs_native_on_real_activations(model, body_ops, monkeypatch):
    kind, unet, inputs = model
    calls = []
    native = body_ops.group_norm_nhwc

    def record(x, norm, bias=None, silu=False):
        out = native(x, norm, bias, silu)
        calls.append((x.clone(), norm, None if bias is None else bias.clone(), silu, out.clone()))
        return out

    monkeypatch.setattr(body_ops, "group_norm_nhwc", record)
    before = body_ops.launch_count()
    _forward(unet, inputs)
    torch.cuda.synchronize()
    assert len(calls) == SITES, f"{kind}: {len(calls)} native GroupNorm calls, {SITES} sites"
    assert body_ops.launch_count() - before == 2 * SITES + GEGLU_SITES
    monkeypatch.undo()

    straddle = 0
    exempt_sites = []
    for i, (x, norm, bias, silu, out) in enumerate(calls):
        n, c, h, w = x.shape
        tag = f"{kind} site {i}: c={c} {h}x{w} G={norm.num_groups} bias={bias is not None} silu={silu}"
        # Each group is 1/64 of a site's tensor.  Where ATen's fp32 Welford itself misrounds a group's fp16 mean or
        # rstd, that group alone breaks the 99.9 % rule although the kernel is right; whether a real activation lands
        # on such a rounding boundary depends on the convolution algorithms cuDNN picks in that run.  Those groups are
        # left out of the fraction only: they meet the flip and fp64 bounds, and the workspace check below pins the
        # kernel's own statistics.
        st = check_group_norm(out, x, norm, bias, silu, tag, exempt_aten_misrounded=True)
        if st["exempt_groups"]:
            exempt_sites.append((i, st["exempt_groups"], round(st["within_1ulp_all"], 5)))
        again, ws = guarded_group_norm(body_ops.lib, x, norm, bias, silu)
        assert torch.equal(again, out), f"{tag}: the C-ABI call differs from the site's output"
        stats = check_group_norm_workspace(ws, x, bias, norm.num_groups, h * w, c, tag=tag)
        print(f"{tag}: workspace max rel err {stats['rel1']:.3g} / {stats['rel2']:.3g}")
        straddle += (c // norm.num_groups) % 8 != 0
    print(f"{kind}: sites with ATen-misrounded groups (site, groups, within 1 ulp with every group): {exempt_sites}")
    assert sum(b is not None for _, _, b, _, _ in calls) == 22                  # temb add at every resnet's norm2
    assert straddle > 0


def test_native_body_is_as_close_to_fp32_as_aten(model, body_ops, monkeypatch):
    kind, unet, (sample, t, ctx) = model
    native = _forward(unet, (sample, t, ctx)).float()
    with monkeypatch.context() as m:
        m.setattr(ops_module, "_BODY_OPS", None)
        aten = _forward(unet, (sample, t, ctx)).float()
    flags = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        ref_model = copy.deepcopy(unet).float()
        ref = _forward(ref_model, (sample.float(), t, ctx.float()))
        del ref_model
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = flags
    torch.cuda.empty_cache()
    rel_native, rel_aten = _rel(native, ref), _rel(aten, ref)
    print(f"{kind}: rel-L2 vs fp32: native {rel_native:.4g}, ATen {rel_aten:.4g}, ratio {rel_native / rel_aten:.4f}")
    assert torch.isfinite(native).all()
    assert rel_native <= FP32_FACTOR * rel_aten


def test_edit_drift_is_at_the_group_norm_rounding_noise_floor():
    """8 steps of a seeded SD1.5 PnP edit (8 frames, B = 4, latent 64) in the four arms of `body_drift`."""
    r = body_drift("sd15", n_frames=8, batch=4, latent=64, steps=8)
    print(f"drift: native vs ATen {r['native_vs_aten_cl']:.4g}, ATen vs ATen with fp32 GroupNorm statistics "
          f"{r['aten_cl_vs_aten_fp32_stats']:.4g}, ATen channels_last vs NCHW {r['aten_cl_vs_aten_nchw']:.4g}")
    assert r["keyframes_equal"] and r["finite"]
    assert r["native_vs_aten_cl"] <= DRIFT_KAPPA * r["aten_cl_vs_aten_fp32_stats"], r
