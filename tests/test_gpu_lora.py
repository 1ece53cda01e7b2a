"""GPU tier (-m gpu, H100): LoRAs merged into CUDA fp16 channels_last models.

* a rank-64 kohya LoRA at every target (kohya's transformer and text-encoder sets and LoCon's convs) merged into
  SD 1.5 and SD 2.1 (random init, the text encoder included) passes `oracle/lora_merge.py`'s fp64 check, and two
  merges on the device are bit-identical;
* `load_parts(..., loras=)` and `load_parts` on a folder written from the merged models give the same saved latents,
  reconstruction and edited frames, bit for bit, on the graphed inversion and the graphed fused step: PnP and SDEdit,
  from the folder, from a single LDM file (`weights=`) and with a Canny ControlNet;
* a LoRA merged into models that already ran an edit (so their TokenFlow blocks hold a fused q/k/v weight and a
  captured graph) edits as the merged folder does;
* `run preprocess` + `run edit --lora` from a synthetic mp4 write the latents and frames the merged folder's runs
  write.
"""
import json
import os
import shutil

import pytest
import torch
from safetensors.torch import load_file

from oracle import ldm_layout, lora_merge
from tokenflow_b200 import lora, pipeline, run, sd_unet
from tokenflow_b200 import synthetic_checkpoint as fx
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.util import save_video
from tokenflow_b200.vae import build_vae

pytestmark = pytest.mark.gpu

ALL = ("transformer", "conv", "text_encoder")
OPT = {"steps": 10, "batch_size": 8, "save_steps": 5, "inversion_prompt": "a woman running"}
PNP = {"prompt": "a marble sculpture of a woman", "negative_prompt": "ugly blurry", "guidance_scale": 7.5,
       "n_timesteps": 5, "batch_size": 4, "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "seed": 1}
SDEDIT = {"prompt": "a shiny silver robotic woman", "negative_prompt": "ugly blurry", "guidance_scale": 7.5,
          "n_timesteps": 5, "batch_size": 4, "start": 0.9, "use_ddim_noise": True, "seed": 1}


def frames(n, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    base = torch.nn.functional.interpolate(torch.rand(n, 3, h // 16, w // 16, generator=g), size=(h, w),
                                           mode="bilinear", align_corners=False)
    return (base * 255).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def state(parts):
    return {f"{name}.{k}": v for name, net in (("unet", parts.unet), ("te", parts.text_encoder))
            for k, v in net.state_dict().items()}


@pytest.mark.parametrize("kind", ["sd15", "sd21"])
def test_rank64_kohya_merge_passes_the_fp64_check(tmp_path, kind):
    model_dir, _ = fx.write_checkpoint(str(tmp_path), kind, dtype=torch.float16, init_device="cuda")
    parts = pipeline.load_parts(model_dir, "cuda", torch.float16)
    assert parts.unet.down_blocks[0].resnets[0].conv1.weight.is_contiguous(memory_format=torch.channels_last)
    path = str(tmp_path / "lora.safetensors")
    targets = fx.write_lora(path, parts.unet, parts.text_encoder, "kohya", 64, ALL, 32, 1)
    assert sum(m == "unet" for m, _ in targets) > 192 and any(m == "text_encoder" for m, _ in targets)
    before = lora_merge.weights(parts.unet, parts.text_encoder)
    changed = lora.merge(parts.unet, parts.text_encoder, [(path, 0.8)])
    assert len(changed) == len(targets)
    # δ grows with the rank (the fp32 GEMM's worst case, γ_r·Σ|U||D|): at rank 64 about a tenth of the outputs are
    # not pinned to one value, against about 1 % at rank 8
    near, total = lora_merge.check_merge(parts.unet, parts.text_encoder, before, [(load_file(path), 0.8)],
                                         max_near_fraction=0.2)
    print(f"{kind}: {near} of {total} merged outputs within δ of a rounding midpoint")
    first = state(parts)
    del parts, before
    again = pipeline.load_parts(model_dir, "cuda", torch.float16, loras=[(path, 0.8)])
    for k, v in state(again).items():
        assert torch.equal(v, first[k]), k
    del again, first
    torch.cuda.empty_cache()


def write_merged_folder(parts, model_dir, dst, unet_config):
    """`model_dir` with the UNet and the text encoder replaced by `parts`' (merged) ones, fp16."""
    shutil.copytree(model_dir, dst)
    fx.write_model(os.path.join(dst, "unet"), parts.unet, unet_config)
    parts.text_encoder.save_pretrained(os.path.join(dst, "text_encoder"))
    return dst


@pytest.fixture(scope="module")
def sd15(tmp_path_factory):
    """(base folder, its ControlNet folder, a single LDM file of the base models, a rank-32 kohya LoRA, the folder of
    the models with the LoRA merged)."""
    root = str(tmp_path_factory.mktemp("sd15"))
    model_dir, cn_dir = fx.write_checkpoint(root, "sd15", controlnet=True, dtype=torch.float16, init_device="cuda")
    base = pipeline.load_parts(model_dir, "cuda", torch.float16)
    path = os.path.join(root, "style.safetensors")
    fx.write_lora(path, base.unet, base.text_encoder, "kohya", 32, ALL, 16, 1)
    weights = os.path.join(root, "v1-5.safetensors")
    unet = sd_unet.build_unet("sd15", seed=1, device="cuda", init_on_device=True)
    vae = build_vae("sd", seed=1, device="cuda", init_on_device=True)
    ldm_layout.save(weights, {**ldm_layout.ldm_unet(unet), **ldm_layout.ldm_vae(vae),
                              **ldm_layout.ldm_clip(base.text_encoder)}, torch.float16)
    del unet, vae
    lora.merge(base.unet, base.text_encoder, [(path, 0.8)])
    merged = write_merged_folder(base, model_dir, os.path.join(root, "merged"), fx.SD15_UNET)
    del base
    torch.cuda.empty_cache()
    return model_dir, cn_dir, weights, path, merged


@torch.no_grad()
def run_arm(parts, frames_u8, config):
    """preprocess + edit on `parts` (the graphed inversion and the graphed fused step)."""
    saved, recon = pipeline.preprocess(parts, frames_u8, OPT)
    torch.manual_seed(config["seed"])
    out = pipeline.edit(parts, frames_u8, {**config, "inversion_prompt": OPT["inversion_prompt"]}, saved)
    return {t: v.clone() for t, v in saved.items()}, recon, out


def assert_same_run(got, want):
    (saved, recon, out), (want_saved, want_recon, want_out) = got, want
    assert sorted(saved) == sorted(want_saved)
    for t in saved:
        assert torch.equal(saved[t], want_saved[t]), t
    assert torch.equal(recon, want_recon) and torch.equal(out, want_out)
    assert 0 < out.float().std() and torch.isfinite(saved[max(saved)].float()).all()


ARMS = {"pnp": (PNP, {}), "sdedit": (SDEDIT, {}), "pnp-weights": (PNP, {"weights": 2}),
        "pnp-controlnet": (PNP, {"controlnet_dir": 1})}


@pytest.mark.parametrize("arm", list(ARMS))
def test_loras_edit_bit_for_bit_as_the_merged_folder(sd15, arm):
    tfu._install_ops_for_testing(None)
    config, extra = ARMS[arm]
    model_dir, path, merged = sd15[0], sd15[3], sd15[4]
    load = {k: sd15[i] for k, i in extra.items()}
    fr = frames(8, 512, 512)
    want = run_arm(pipeline.load_parts(merged, "cuda", torch.float16,
                                       controlnet_dir=load.get("controlnet_dir")), fr, config)
    torch.cuda.empty_cache()
    got = run_arm(pipeline.load_parts(model_dir, "cuda", torch.float16, loras=[(path, 0.8)], **load), fr, config)
    assert_same_run(got, want)
    torch.cuda.empty_cache()


def test_a_merge_after_an_edit_edits_as_the_merged_folder(sd15):
    """The first edit caches each TokenFlow block's fused q/k/v weight and captures graphs; the merge bumps the
    weights' versions, and the next edit's new editor re-makes the fused weights and captures again."""
    tfu._install_ops_for_testing(None)
    model_dir, path, merged = sd15[0], sd15[3], sd15[4]
    fr = frames(8, 512, 512)
    saved, _, want = run_arm(pipeline.load_parts(merged, "cuda", torch.float16), fr, PNP)
    torch.cuda.empty_cache()
    cfg = {**PNP, "inversion_prompt": OPT["inversion_prompt"]}
    parts = pipeline.load_parts(model_dir, "cuda", torch.float16)
    with torch.no_grad():
        torch.manual_seed(PNP["seed"])
        base = pipeline.edit(parts, fr, cfg, saved)
        lora.merge(parts.unet, parts.text_encoder, [(path, 0.8)])
        torch.manual_seed(PNP["seed"])
        got = pipeline.edit(parts, fr, cfg, saved)
    assert torch.equal(got, want) and not torch.equal(base, want)
    del parts
    torch.cuda.empty_cache()


def test_cli_from_a_video_with_lora_writes_what_the_merged_folder_writes(sd15, tmp_path, monkeypatch):
    tfu._install_ops_for_testing(None)
    model_dir, path, merged = sd15[0], sd15[3], sd15[4]
    monkeypatch.chdir(tmp_path)
    os.makedirs("data")
    save_video(frames(8, 360, 640), "data/clip.mp4", fps=30)
    outputs = {}
    for arm, common in (("folder", ["--model_dir", merged]), ("lora", ["--model_dir", model_dir, "--lora",
                                                                       f"{path}:0.8"])):
        run.main(["preprocess", *common, "--data_path", "data/clip.mp4", "--sd_version", "1.5", "--save_dir", arm,
                  "--steps", "10", "--batch_size", "8", "--save_steps", "5", "--n_frames", "8",
                  "--inversion_prompt", OPT["inversion_prompt"]])
        config = {**PNP, "data_path": "data/clip", "latents_path": arm, "sd_version": "1.5", "n_inversion_steps": 10,
                  "n_frames": 8, "output_path": str(tmp_path / arm / "out")}
        with open(f"{arm}.yaml", "w") as f:
            json.dump(config, f)
        run.main(["edit", *common, "--config_path", f"{arm}.yaml"])
        lat = os.path.join(arm, "sd_1.5", "clip", "steps_10", "nframes_8")
        outputs[arm] = (run.read_latents(lat), run.read_frames(os.path.join(lat, "frames"), 8),
                        run.read_frames(str(tmp_path / arm / "out" / "img_ode"), 8))
        torch.cuda.empty_cache()
    (want_lat, want_recon, want_out), (got_lat, got_recon, got_out) = outputs["folder"], outputs["lora"]
    assert sorted(got_lat) == sorted(want_lat) and len(want_lat) == 6
    for t in want_lat:
        assert torch.equal(got_lat[t], want_lat[t]), t
    assert torch.equal(got_recon, want_recon) and torch.equal(got_out, want_out) and want_out.float().std() > 0
