"""GPU tier (-m gpu, H100): single-file checkpoints run exactly what their diffusers folders run.

* a synthetic full-size SD1.5 single file (fp16 safetensors in the LDM layout, written by `oracle/ldm_layout.py`) and
  a Canny ControlNet `.pth` in lllyasviel's layout load as CUDA fp16 channels_last, equal to the diffusers folder's
  models;
* `pipeline.preprocess` + `pipeline.edit` on them (PnP with the ControlNet, C2's 40 frames of 512² and B = 8, a few
  steps, the CUDA-graphed fused step) give saved latents and uint8 frames equal bit for bit to the same calls on the
  diffusers folder;
* a step graph capture first frees the graphs of a dropped inverter, which its reference cycle keeps for the
  garbage collector: freed during a capture, they would make the capture fail (loading a second set of models
  in one process, as these tests do, drops one);
* an SD2.1-768 v single file (OpenCLIP text encoder, a Lightning `.ckpt`) passes the same check and its edit runs
  the v kernel of the fused CFG + DDIM step.
"""
import gc
import json
import os
import re
import weakref

import pytest
import torch

from oracle import ldm_layout
from tokenflow_b200 import checkpoint, pipeline, sd_unet
from tokenflow_b200 import synthetic_checkpoint as fx
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.controlnet import build_controlnet
from tokenflow_b200.preprocess import LatentInverter
from tokenflow_b200.vae import build_vae

pytestmark = pytest.mark.gpu

OPT = {"steps": 10, "batch_size": 40, "save_steps": 5, "inversion_prompt": "a woman running"}
PNP = {"prompt": "a marble sculpture of a woman", "negative_prompt": "ugly blurry", "guidance_scale": 7.5,
       "n_timesteps": 5, "batch_size": 8, "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "seed": 1}


def frames(n, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    base = torch.nn.functional.interpolate(torch.rand(n, 3, h // 16, w // 16, generator=g), size=(h, w),
                                           mode="bilinear", align_corners=False)
    return (base * 255).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def write_single_file(root, kind, model_dir, name, text_layout):
    """The same random-init models `write_checkpoint(kind, init_device="cuda")` saved, in the LDM layout, fp16."""
    from transformers import CLIPTextModel
    unet = sd_unet.build_unet(kind, seed=1, device="cuda", init_on_device=True)
    vae = build_vae("sd", seed=1, device="cuda", init_on_device=True)
    encoder = CLIPTextModel.from_pretrained(model_dir, subfolder="text_encoder", local_files_only=True)
    text = ldm_layout.ldm_clip(encoder) if text_layout == "clip" else ldm_layout.ldm_openclip(encoder)
    path = os.path.join(root, name)
    ldm_layout.save(path, {**ldm_layout.ldm_unet(unet), **ldm_layout.ldm_vae(vae), **text}, torch.float16)
    vae_tensors = {k: v.half().cpu() for k, v in ldm_layout.ldm_vae(vae).items()}
    del unet, vae
    torch.cuda.empty_cache()
    return path, vae_tensors


@pytest.fixture(scope="module")
def sd15(tmp_path_factory):
    """(diffusers folder, its ControlNet folder, the SD1.5 single file, the ControlNet .pth)."""
    root = str(tmp_path_factory.mktemp("sd15"))
    model_dir, cn_dir = fx.write_checkpoint(root, "sd15", controlnet=True, variant="fp16", dtype=torch.float16,
                                            init_device="cuda", deprecated_vae=True)
    weights, vae_tensors = write_single_file(root, "sd15", model_dir, "v1-5-pruned-emaonly.safetensors", "clip")
    pth = os.path.join(root, "control_sd15_canny.pth")
    # like lllyasviel's file, the ControlNet beside other SD tensors, which are not read
    ldm_layout.save(pth, {**ldm_layout.ldm_controlnet(build_controlnet("sd15", seed=3)), **vae_tensors},
                    torch.float16)
    torch.cuda.empty_cache()
    return model_dir, cn_dir, weights, pth


def _models(parts):
    return {"unet": parts.unet, "vae": parts.vae, "controlnet": parts.controlnet, "text_encoder": parts.text_encoder}


def test_sd15_file_and_controlnet_pth_load_cuda_fp16_channels_last(sd15):
    model_dir, cn_dir, weights, pth = sd15
    got = pipeline.load_parts(model_dir, "cuda", torch.float16, pth, weights=weights)
    want = pipeline.load_parts(model_dir, "cuda", torch.float16, cn_dir, variant="fp16")
    for name, net in _models(got).items():
        ref = _models(want)[name].state_dict()
        state = net.state_dict()
        assert list(state) == list(ref), name
        for k, p in state.items():
            assert p.is_cuda and torch.equal(p, ref[k]), (name, k)
            if p.is_floating_point():
                assert p.dtype == torch.float16, (name, k)
            if p.dim() == 4:
                assert p.is_contiguous(memory_format=torch.channels_last), (name, k)
    del got, want
    torch.cuda.empty_cache()


@torch.no_grad()
def run_arm(model_dir, frames_u8, opt, config, trace=None, **load):
    """preprocess + edit on freshly loaded parts; with `trace` (a chrome-trace path), also the kernel names of the
    edit."""
    parts = pipeline.load_parts(model_dir, "cuda", torch.float16, **load)
    saved, recon = pipeline.preprocess(parts, frames_u8, opt)
    torch.manual_seed(config["seed"])
    cfg = {**config, "inversion_prompt": opt["inversion_prompt"]}
    kernels = set()
    if trace:
        acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
        with torch.profiler.profile(activities=acts) as prof:
            out = pipeline.edit(parts, frames_u8, cfg, saved)
            torch.cuda.synchronize()
        prof.export_chrome_trace(trace)
        with open(trace) as f:
            kernels = {e["name"] for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"}
    else:
        out = pipeline.edit(parts, frames_u8, cfg, saved)
    saved = {t: v.clone() for t, v in saved.items()}
    del parts
    torch.cuda.empty_cache()
    return saved, recon, out, kernels


def assert_same_run(got, want):
    (saved, recon, out, _), (want_saved, want_recon, want_out, _) = got, want
    assert sorted(saved) == sorted(want_saved)
    for t in saved:
        assert torch.equal(saved[t], want_saved[t]), t
    assert recon.dtype == out.dtype == torch.uint8
    assert torch.equal(recon, want_recon) and torch.equal(out, want_out)
    assert 0 < out.float().std() and torch.isfinite(saved[max(saved)].float()).all()


def test_sd15_file_edits_bit_for_bit_as_its_folder(sd15):
    tfu._install_ops_for_testing(None)
    model_dir, cn_dir, weights, pth = sd15
    fr = frames(40, 512, 512)                                    # C2: 40 frames of 512², B = 8
    want = run_arm(model_dir, fr, OPT, PNP, controlnet_dir=cn_dir, variant="fp16")
    got = run_arm(model_dir, fr, OPT, PNP, controlnet_dir=pth, weights=weights)
    assert got[2].shape == (40, 512, 512, 3)
    assert_same_run(got, want)


def test_a_capture_frees_a_dropped_inverters_step_graph(sd15):
    tfu._install_ops_for_testing(None)
    model_dir = sd15[0]
    parts = pipeline.load_parts(model_dir, "cuda", torch.float16, variant="fp16")
    g = torch.Generator(device="cuda").manual_seed(0)
    latents = torch.randn(2, 4, 64, 64, device="cuda", generator=g).half()
    cond = checkpoint.text_embeds(parts.tokenizer, parts.text_encoder, "a woman running", "")[1:]

    def invert():
        inv = LatentInverter(parts.unet, checkpoint.load_scheduler(model_dir), 2)
        inv.ddim_inversion(cond, latents, None, batch_size=2, timesteps_to_save=[])
        return weakref.ref(inv)

    enabled = gc.isenabled()
    gc.disable()                    # only the capture's own collection may free the first inverter
    try:
        first = invert()
        second = invert()
        assert first() is None
    finally:
        if enabled:
            gc.enable()
    del parts, second
    gc.collect()
    torch.cuda.empty_cache()


def _pred(kernels, kernel):
    out = set()
    for k in kernels:
        m = re.search(r"(?<!\w)" + kernel + r"<([^>]*)>", k)
        if m:
            arg = m.group(1).strip()
            out.add("v" if arg.endswith("1") or "kV" in arg else "eps")
    return out


def test_sd21_768_v_file_edits_bit_for_bit_on_the_v_kernels(tmp_path):
    tfu._install_ops_for_testing(None)
    root = str(tmp_path)
    model_dir, _ = fx.write_checkpoint(root, "sd21", scheduler=fx.SD21_V_SCHEDULER, dtype=torch.float16,
                                       init_device="cuda")
    weights, _ = write_single_file(root, "sd21", model_dir, "v2-1_768-ema-pruned.ckpt", "openclip")
    with open(os.path.join(model_dir, "scheduler", "scheduler_config.json")) as f:
        assert json.load(f)["prediction_type"] == "v_prediction"
    opt = {**OPT, "batch_size": 8, "H": 768, "W": 704}
    fr = frames(8, 360, 640)
    want = run_arm(model_dir, fr, opt, PNP)
    got = run_arm(model_dir, fr, opt, PNP, trace=os.path.join(root, "edit.json"), weights=weights)
    assert got[2].shape == (8, 768, 704, 3) and all(v.shape == (8, 4, 96, 88) for v in got[0].values())
    assert_same_run(got, want)
    assert _pred(got[3], "cfg_ddim_kernel") == {"v"}, sorted(k for k in got[3] if "ddim" in k)
