"""GPU tier (-m gpu): the ControlNet on the H100.

* inversion: `LatentInverter` with a ControlNet, graph-replayed against the same device path run eagerly, bit for bit,
  and against the reference's `controlnet_pred` loop (oracle/controlnet_inversion.py);
* editor: the CUDA-graphed fused step against the eager fused step, bit for bit, in PnP and SDEdit mode, on the tiny
  UNet and on SD1.5 channels_last (the ControlNet's GroupNorm and GEGLU sites on the library's kernels inside the
  captured step), with the Canny conditioning computed on the device by `preprocess.canny_cond`.
"""
import numpy as np
import pytest
import torch

from oracle import gen_canny_golden as gg
from oracle import controlnet_inversion as CI
from tokenflow_b200 import preprocess
from tokenflow_b200 import sd_unet
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.controlnet import build_controlnet
from tokenflow_b200.editor import TokenFlowEditor, synthetic_inputs
from tokenflow_b200.preprocess import LatentInverter
from tokenflow_b200.scheduler import DDIMScheduler

pytestmark = pytest.mark.gpu


def _cond(n, h, w, seed=5):
    rng = np.random.default_rng(seed)
    frames = torch.from_numpy(np.stack([gg.make_frame("smooth", h, w, rng) for _ in range(n)])).cuda()
    return preprocess.canny_cond(frames)


def _models(kind):
    tfu._install_ops_for_testing(None)
    on_dev = kind != "tiny"
    unet = sd_unet.build_unet(kind, seed=1, device="cuda", dtype=torch.float16, init_on_device=on_dev)
    cn = build_controlnet(kind, seed=3, device="cuda", dtype=torch.float16)
    if kind != "tiny":
        unet = unet.to(memory_format=torch.channels_last)
        cn = cn.to(memory_format=torch.channels_last)
    return unet, cn


def test_inversion_graph_replay_equals_eager_and_the_reference_loop():
    unet, cn = _models("sd15")
    g = torch.Generator().manual_seed(3)
    n = 4
    x0 = torch.randn(n, 4, 64, 64, generator=g).half().cuda()
    cond = torch.randn(1, 77, 768, generator=g).half().cuda()
    ccond = _cond(n, 512, 512)
    res = {}
    for graphed in (True, False):
        inv = LatentInverter(unet, DDIMScheduler(), 6, controlnet=cn, controlnet_cond=ccond)
        inv._use_graph = graphed
        xT = inv.ddim_inversion(cond, x0, None, batch_size=2)
        rec = inv.ddim_sample(xT, cond, batch_size=2)
        res[graphed] = (xT, rec, inv.saved_latents(), inv.scheduler)
    assert torch.isfinite(res[True][1]).all()
    assert torch.equal(res[True][0], res[False][0]) and torch.equal(res[True][1], res[False][1])
    for t in res[True][2]:
        assert torch.equal(res[True][2][t], res[False][2][t]), t
    sch = res[True][3]
    want_T, _ = CI.ddim_inversion(unet, cn, sch, cond, ccond, x0.clone(), 2)
    want_rec = CI.ddim_sample(unet, cn, sch, want_T.clone(), cond, ccond, 2)
    assert torch.equal(res[True][0], want_T), (res[True][0].float() - want_T.float()).abs().max().item()
    assert torch.equal(res[True][1], want_rec), (res[True][1].float() - want_rec.float()).abs().max().item()
    plain = LatentInverter(unet, DDIMScheduler(), 6)
    assert not torch.equal(plain.ddim_inversion(cond, x0, None, batch_size=2), res[True][0])


def _editor(kind, mode, steps, graph, n_frames=8, batch=2, latent=16):
    unet, cn = _models(kind)
    cfg = {"n_frames": n_frames, "batch_size": batch, "n_timesteps": steps, "guidance_scale": 7.5, "mode": mode,
           "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "start": 0.9, "fused_pass": True, "cuda_graph": graph,
           "keyframe_seed": 1, "controlnet_conditioning_scale": 0.8}
    x, text, pnp, src = synthetic_inputs(n_frames, latent, unet.config.cross_attention_dim, steps, seed=1,
                                         device="cuda", dtype=torch.float16, ctx_len=7)
    ed = TokenFlowEditor(unet, DDIMScheduler(), tfu, cfg, text, pnp, source_latents=lambda t: src[t],
                         controlnet=cn, controlnet_cond=_cond(n_frames, 8 * latent, 8 * latent))
    ed.init_method()
    return ed, x


@pytest.mark.parametrize("kind,mode,steps", [pytest.param("tiny", "pnp", 5, id="tiny-pnp-5"),
                                             pytest.param("tiny", "sdedit", 10, id="tiny-sdedit-10"),
                                             pytest.param("sd15", "pnp", 3, id="sd15-pnp-3"),
                                             pytest.param("sd15", "sdedit", 10, id="sd15-sdedit-10")])
def test_cuda_graph_step_identical_to_eager(kind, mode, steps):
    kw = {} if kind == "tiny" else dict(latent=64, batch=4)
    ed_e, x = _editor(kind, mode, steps, graph=False, **kw)
    want = ed_e.sample_loop(x.clone())
    ed_g, x = _editor(kind, mode, steps, graph=True, **kw)
    got = ed_g.sample_loop(x.clone())
    assert ed_g.keyframe_log == ed_e.keyframe_log
    assert all(e["replays"] >= 1 for e in ed_g._graphs.values())
    assert torch.isfinite(got).all()
    assert torch.equal(got, want), (got.float() - want.float()).abs().max().item()
