"""GPU tier (-m gpu, H100): the pipeline on loaded checkpoints runs the native paths.

* a synthetic full-size SD1.5 checkpoint (random weights saved as the fp16 variant, the VAE's attention under the
  names the published VAE files use) loads as CUDA fp16 channels_last, with the saved values;
* `pipeline.preprocess` + `pipeline.edit` at 8 frames of 512², B = 4, a few steps, equal bit for bit the INTEGRATION.md
  §6 chain run by hand in the same process;
* a torch.profiler trace of each stage shows the library's kernels (GroupNorm in the UNet, with its time-embedding
  bias, and in the VAE, at 4 channels per group; extended attention, NN field, propagation, the CFG + DDIM and DDIM
  steps, the resize and the pixel conversions), no ATen GroupNorm kernel, and at least one CUDA-graph launch per
  inversion, reconstruction and edit step;
* an SD2.1-768 checkpoint with a v-prediction scheduler runs the v kernels and not the eps ones.
"""
import json
import os
import re

import pytest
import torch

from tokenflow_b200 import synthetic_checkpoint as fx

from tokenflow_b200 import checkpoint, pipeline, sd_unet
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.editor import TokenFlowEditor
from tokenflow_b200.preprocess import (LatentInverter, ddim_eps, decode_latents, encode_imgs,
                                       resize_frames)
from tokenflow_b200.scheduler import DDIMScheduler
from tokenflow_b200.vae import build_vae

pytestmark = pytest.mark.gpu

OPT = {"steps": 10, "batch_size": 8, "save_steps": 5, "inversion_prompt": "a woman running"}
PNP = {"prompt": "a marble sculpture of a woman", "negative_prompt": "ugly blurry", "guidance_scale": 7.5,
       "n_timesteps": 5, "batch_size": 4, "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "seed": 1}
SDEDIT = {"prompt": "a shiny silver robotic wolf", "negative_prompt": "ugly blurry", "guidance_scale": 7.5,
          "n_timesteps": 5, "batch_size": 4, "start": 0.9, "use_ddim_noise": True, "seed": 1}

# kernel name patterns of the library's entry points, as they appear in a trace (demangled, namespace tf::)
GN_UNET = r"gn_stats_kernel<true, 0>"           # tf_group_norm_nhwc with the time-embedding bias: UNet resnets
GN_VAE = r"gn_stats_kernel<false, 4>"           # tf_group_norm_nhwc at 4 channels per group: the VAE's 128-ch levels
ATEN_GN = r"GroupNorm|RowwiseMoments|ComputeFusedParams|group_norm"


@pytest.fixture(scope="module")
def sd15(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("sd15"))
    model_dir, _ = fx.write_checkpoint(root, "sd15", variant="fp16", dtype=torch.float16, init_device="cuda",
                                       deprecated_vae=True)         # the VAE's attention under its published names
    torch.cuda.empty_cache()
    return model_dir


def frames(n, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    base = torch.nn.functional.interpolate(torch.rand(n, 3, h // 16, w // 16, generator=g), size=(h, w),
                                           mode="bilinear", align_corners=False)
    return (base * 255).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def test_sd15_checkpoint_loads_cuda_fp16_channels_last(sd15):
    parts = pipeline.load_parts(sd15, "cuda", torch.float16, variant="fp16")
    for net in (parts.unet, parts.vae):
        for name, p in net.named_parameters():
            assert p.is_cuda and p.dtype == torch.float16, name
            if p.dim() == 4:
                assert p.is_contiguous(memory_format=torch.channels_last), name
    assert parts.text_encoder.dtype == torch.float16 and next(parts.text_encoder.parameters()).is_cuda
    want = sd_unet.build_unet("sd15", seed=1, device="cuda", init_on_device=True).half().state_dict()
    got = parts.unet.state_dict()
    assert list(got) == list(want)
    for k in want:
        assert torch.equal(got[k], want[k]), k
    vae = build_vae("sd", seed=1, device="cuda", init_on_device=True).half().state_dict()
    assert all(torch.equal(parts.vae.state_dict()[k], vae[k]) for k in vae)


def _trace(tmp_path, name, fn):
    """fn() under torch.profiler (CPU + CUDA); returns (result, kernel names, number of CUDA-graph launches)."""
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        out = fn()
        torch.cuda.synchronize()
    path = os.path.join(str(tmp_path), f"{name}.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        events = json.load(f)["traceEvents"]
    kernels = {e["name"] for e in events if e.get("cat") == "kernel"}
    launches = sum(1 for e in events if "GraphLaunch" in str(e.get("name")))
    return out, kernels, launches


def _ran(kernels, pattern):
    return any(re.search(pattern, k) for k in kernels)


def _pred(kernels, kernel):
    """The Pred template arguments (eps 0, v 1) of every instance of `kernel` that ran."""
    out = set()
    for k in kernels:
        m = re.search(r"(?<!\w)" + kernel + r"<([^>]*)>", k)
        if m:
            arg = m.group(1).strip()
            out.add("v" if arg.endswith("1") or "kV" in arg else "eps")
    return out


@torch.no_grad()
def hand_chain(model_dir, frames_u8, opt, config, variant):
    """INTEGRATION.md §6 stage by stage on freshly loaded models."""
    unet = checkpoint.load_unet(model_dir, "cuda", torch.float16, variant)
    vae = checkpoint.load_vae(model_dir, "cuda", torch.float16, variant)
    tok, enc = checkpoint.load_text_encoder(model_dir, "cuda", torch.float16)
    sched = checkpoint.read_config(os.path.join(model_dir, "scheduler"), "scheduler_config.json")
    fr = resize_frames(frames_u8.cuda(), 512 if frames_u8.shape[1] == frames_u8.shape[2] else (opt["H"], opt["W"]))
    latents = encode_imgs(vae, fr)
    toy = DDIMScheduler.from_config(sched)
    toy.set_timesteps(opt["save_steps"])
    inv = LatentInverter(unet, DDIMScheduler.from_config(sched), opt["steps"])
    cond = checkpoint.text_embeds(tok, enc, opt["inversion_prompt"], "")[1:]
    x_T = inv.ddim_inversion(cond, latents, None, batch_size=opt["batch_size"],
                             timesteps_to_save=toy.timesteps.tolist())
    recon = decode_latents(vae, inv.ddim_sample(x_T, cond, batch_size=opt["batch_size"]))
    saved = inv.saved_latents()
    torch.manual_seed(config["seed"])
    text = checkpoint.text_embeds(tok, enc, config["prompt"], config["negative_prompt"])
    pnp = checkpoint.text_embeds(tok, enc, opt["inversion_prompt"], opt["inversion_prompt"]).chunk(2)[0]
    mode = "pnp" if "pnp_attn_t" in config else "sdedit"
    cfg = {**config, "mode": mode, "fused_pass": True, "cuda_graph": True}
    editor = TokenFlowEditor(unet, DDIMScheduler.from_config(sched), tfu, cfg, text, pnp,
                             source_latents=saved.__getitem__)
    eps = ddim_eps(latents, saved, editor.scheduler)
    x = editor.scheduler.add_noise(latents, eps, editor.scheduler.timesteps[0])
    editor.init_method()
    return saved, recon, decode_latents(vae, editor.sample_loop(x))


def _run_traced(tmp_path, model_dir, frames_u8, opt, config, variant):
    parts = pipeline.load_parts(model_dir, "cuda", torch.float16, variant=variant)
    (saved, recon), k_pre, g_pre = _trace(tmp_path, "preprocess", lambda: pipeline.preprocess(parts, frames_u8, opt))
    torch.manual_seed(config["seed"])
    cfg = {**config, "inversion_prompt": opt["inversion_prompt"]}
    out, k_edit, g_edit = _trace(tmp_path, "edit", lambda: pipeline.edit(parts, frames_u8, cfg, saved))
    del parts
    torch.cuda.empty_cache()
    return (saved, recon, out), (k_pre, g_pre), (k_edit, g_edit)


def test_sd15_pipeline_equals_the_hand_chain_on_the_native_kernels(sd15, tmp_path):
    tfu._install_ops_for_testing(None)
    fr = frames(8, 480, 480)                                # square: edited at 512²
    (saved, recon, out), (k_pre, g_pre), (k_edit, g_edit) = _run_traced(tmp_path, sd15, fr, OPT, PNP, "fp16")
    want_saved, want_recon, want_out = hand_chain(sd15, fr, OPT, PNP, "fp16")
    assert sorted(saved) == sorted(want_saved)
    for t in saved:
        assert torch.equal(saved[t], want_saved[t]), t
    assert recon.shape == (8, 512, 512, 3) and torch.equal(recon, want_recon)
    assert out.shape == (8, 512, 512, 3) and torch.equal(out, want_out)
    assert 0 < out.float().std() and torch.isfinite(saved[max(saved)].float()).all()

    for what, kernels in (("preprocess", k_pre), ("edit", k_edit)):
        for pattern in (GN_UNET, GN_VAE, "resize_h_kernel", "resize_v_kernel", "frames_to_input_kernel",
                        "output_to_frames_kernel"):
            assert _ran(kernels, pattern), (what, pattern)
        assert not _ran(kernels, ATEN_GN), (what, sorted(k for k in kernels if re.search(ATEN_GN, k)))
    assert _pred(k_pre, "ddim_kernel") == {"eps"}
    for pattern in ("ext_attn_kernel", "nn_field_kernel", "propagate_kernel", "layernorm_rows_kernel"):
        assert _ran(k_edit, pattern), pattern
    assert _pred(k_edit, "cfg_ddim_kernel") == {"eps"}
    # a graph launch for every inversion and reconstruction step, and for every edit step
    assert g_pre >= 2 * OPT["steps"], g_pre
    assert g_edit >= PNP["n_timesteps"], g_edit


def test_sd21_768_v_checkpoint_runs_the_v_kernels(tmp_path):
    tfu._install_ops_for_testing(None)
    model_dir, _ = fx.write_checkpoint(str(tmp_path), "sd21", scheduler=fx.SD21_V_SCHEDULER, dtype=torch.float16,
                                       init_device="cuda")
    torch.cuda.empty_cache()
    opt = {**OPT, "H": 768, "W": 704}
    fr = frames(8, 360, 640)
    (saved, recon, out), (k_pre, g_pre), (k_edit, g_edit) = _run_traced(tmp_path, model_dir, fr, opt, SDEDIT, None)
    assert out.shape == (8, 768, 704, 3) and all(v.shape == (8, 4, 96, 88) for v in saved.values())
    assert torch.isfinite(saved[max(saved)].float()).all()
    assert _pred(k_pre, "ddim_kernel") == {"v"}
    assert _pred(k_edit, "cfg_ddim_kernel") == {"v"}
    for pattern in ("ext_attn_kernel", "nn_field_kernel", "propagate_kernel", GN_UNET, GN_VAE):
        assert _ran(k_edit, pattern), pattern
    assert not _ran(k_pre, ATEN_GN) and not _ran(k_edit, ATEN_GN)
    assert g_pre >= 2 * opt["steps"] and g_edit >= 3            # SDEdit from t = 0.9 * 1000: the last 3 of 5 steps
