"""CPU tier: single-file checkpoints in the original LDM layout (`checkpoint.load_single_file_models`,
`load_controlnet_file`, `run --weights`).

The files are written by `oracle/ldm_layout.py`, which names the tensors by LDM's own module grammar and shares no
table with the converters.

* a file of the tiny, SD1.5 and SD2.1 kinds (fp32 and fp16 safetensors, a Lightning `.ckpt`; the SD1.x text encoder
  with and without transformers' `text_model.` level, the SD2.x one in OpenCLIP's layout) loads, on the matching
  diffusers folder, to the builders' values;
* the EMA copy of the UNet is not read;
* an OpenCLIP text encoder with one resblock more than the folder's config gives the folder encoder's `text_embeds`,
  and one with fewer is refused;
* a cldm ControlNet file, alone or beside a whole SD model, loads to `build_controlnet`'s values;
* a missing prefix, an extra or missing key, a file of another family and a pickle `weights_only` rejects are refused
  with an error naming the prefix, the key or the remedy;
* `run preprocess` and `run edit` with `--weights` write what the same runs from the diffusers folder write.
"""
import argparse
import json
import os

import pytest
import torch

from oracle import ldm_layout
from oracle.oracle_ops import OracleOps
from tokenflow_b200 import checkpoint, run, sd_unet
from tokenflow_b200 import synthetic_checkpoint as fx
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.controlnet import build_controlnet
from tokenflow_b200.vae import build_vae

VAE_CONFIGS = {"tiny": fx.TINY_VAE, "sd15": fx.SD_VAE, "sd21": fx.SD_VAE}


def base_folder(root, kind, scheduler=fx.SD15_SCHEDULER, text_config=None):
    """A diffusers folder of `kind` without UNet or VAE weights: the configs, the scheduler and the text side, all a
    single file needs beside it."""
    model_dir = os.path.join(str(root), f"base-{kind}")
    for sub, config in (("unet", fx.UNET_CONFIGS[kind]), ("vae", VAE_CONFIGS[kind])):
        os.makedirs(os.path.join(model_dir, sub))
        with open(os.path.join(model_dir, sub, "config.json"), "w") as f:
            json.dump(config, f)
    os.makedirs(os.path.join(model_dir, "scheduler"))
    with open(os.path.join(model_dir, "scheduler", "scheduler_config.json"), "w") as f:
        json.dump(scheduler, f)
    fx.write_text_side(model_dir, fx.CONTEXT[kind], layers=1, heads=2 if kind == "tiny" else 8,
                       text_config=text_config)
    return model_dir


def builders(kind):
    """The random-init UNet and VAE `write_checkpoint` saves for `kind`."""
    return sd_unet.build_unet(kind, seed=1), build_vae("tiny" if kind == "tiny" else "sd", seed=1)


def folder_encoder(model_dir):
    from transformers import CLIPTextModel
    return CLIPTextModel.from_pretrained(model_dir, subfolder="text_encoder", local_files_only=True).eval()


def text_tensors(layout, encoder):
    return {"clip": lambda: ldm_layout.ldm_clip(encoder),
            "clip-legacy": lambda: ldm_layout.ldm_clip(encoder, text_model_level=False, position_ids=True),
            "openclip": lambda: ldm_layout.ldm_openclip(encoder)}[layout]()


def write_sd_file(path, unet, vae, encoder, layout="clip", dtype=None, ema=False):
    state = {**ldm_layout.ldm_unet(unet), **ldm_layout.ldm_vae(vae), **text_tensors(layout, encoder)}
    if ema:
        state.update(ldm_layout.ema_copy(state))
    ldm_layout.save(path, state, dtype)
    return path


def assert_equal_state(got, want, dtype=None):
    """`got`'s state dict is `want`'s (rounded through `dtype` when the file held that dtype)."""
    sg, sw = got.state_dict(), want.state_dict()
    assert list(sg) == list(sw)
    for k, v in sw.items():
        if dtype is not None and v.is_floating_point():
            v = v.to(dtype).to(v.dtype)
        assert sg[k].shape == v.shape and sg[k].dtype == v.dtype, k
        assert torch.equal(sg[k], v), k


@pytest.fixture(scope="module")
def sd21_file(tmp_path_factory):
    """An SD2.1-768 file in fp16 as a Lightning .ckpt, its text encoder in OpenCLIP's layout, and its base folder."""
    root = tmp_path_factory.mktemp("sd21")
    model_dir = base_folder(root, "sd21", fx.SD21_V_SCHEDULER)
    unet, vae = builders("sd21")
    path = write_sd_file(str(root / "v2-1_768.ckpt"), unet, vae, folder_encoder(model_dir), "openclip",
                         torch.float16)
    return model_dir, path


@pytest.fixture(scope="module")
def sd15_file(tmp_path_factory):
    """An SD1.5 file in fp16 safetensors and its base folder."""
    root = tmp_path_factory.mktemp("sd15")
    model_dir = base_folder(root, "sd15")
    unet, vae = builders("sd15")
    path = write_sd_file(str(root / "v1-5.safetensors"), unet, vae, folder_encoder(model_dir), "clip",
                         torch.float16)
    return model_dir, path


TINY_FORMS = {"fp32-safetensors": ("m.safetensors", None, "clip"),
              "fp16-safetensors": ("m.safetensors", torch.float16, "clip"),
              "ckpt-legacy-clip": ("m.ckpt", None, "clip-legacy")}


@pytest.mark.parametrize("form", list(TINY_FORMS))
def test_tiny_file_loads_the_builders_values(tmp_path, form):
    name, dtype, layout = TINY_FORMS[form]
    model_dir, _ = fx.write_checkpoint(str(tmp_path), "tiny")
    unet, vae = builders("tiny")
    encoder = folder_encoder(model_dir)
    path = write_sd_file(str(tmp_path / name), unet, vae, encoder, layout, dtype)
    if name.endswith(".ckpt"):
        stored = torch.load(path, weights_only=True)
        assert stored["global_step"] == 1 and "cond_stage_model.transformer.embeddings.position_ids" in stored[
            "state_dict"]
    got_unet, got_vae, tok, got_enc = checkpoint.load_single_file_models(path, model_dir)
    for got, want in ((got_unet, unet), (got_vae, vae), (got_enc, encoder)):
        assert not got.training and not any(t.is_meta for t in (*got.parameters(), *got.buffers()))
        assert_equal_state(got, want, dtype)
    assert tok.model_max_length == 77


@pytest.mark.parametrize("kind", ["sd15", "sd21"])
def test_full_size_file_loads_the_builders_values(request, kind):
    model_dir, path = request.getfixturevalue(f"{kind}_file")
    got_unet, got_vae, _, got_enc = checkpoint.load_single_file_models(path, model_dir)
    unet, vae = builders(kind)
    assert_equal_state(got_unet, unet, torch.float16)
    del got_unet, unet
    assert_equal_state(got_vae, vae, torch.float16)
    assert_equal_state(got_enc, folder_encoder(model_dir), torch.float16)


def test_the_ema_copy_is_not_read(tmp_path):
    model_dir, _ = fx.write_checkpoint(str(tmp_path), "tiny")
    unet, vae = builders("tiny")
    path = write_sd_file(str(tmp_path / "ema.safetensors"), unet, vae, folder_encoder(model_dir), ema=True)
    stored = checkpoint.load_single_file(path)
    assert torch.equal(stored["model_ema.diffusion_modelout2bias"], -unet.conv_out.bias.detach())
    got_unet, *_ = checkpoint.load_single_file_models(path, model_dir)
    assert_equal_state(got_unet, unet)


PROMPT, NEGATIVE = "a marble sculpture of a woman running", "ugly blurry low res"


def test_openclip_text_encoder_drops_the_last_block(tmp_path):
    """SD 2.x: the file has num_hidden_layers + 1 resblocks, q, k and v packed; the folder's encoder reads the
    penultimate layer, so the extra block is dropped and the prompts encode as the folder's encoder encodes them."""
    model_dir, _ = fx.write_checkpoint(str(tmp_path), "tiny", text_config={"num_hidden_layers": 2})
    unet, vae = builders("tiny")
    encoder = folder_encoder(model_dir)
    path = write_sd_file(str(tmp_path / "v2.safetensors"), unet, vae, encoder, "openclip")
    stored = checkpoint.load_single_file(path)
    assert "cond_stage_model.model.transformer.resblocks.2.attn.in_proj_weight" in stored
    _, _, tok, got = checkpoint.load_single_file_models(path, model_dir)
    assert_equal_state(got, encoder)
    want = checkpoint.text_embeds(tok, encoder, PROMPT, NEGATIVE)
    assert torch.equal(checkpoint.text_embeds(tok, got, PROMPT, NEGATIVE), want)
    state = {**ldm_layout.ldm_unet(unet), **ldm_layout.ldm_vae(vae), **ldm_layout.ldm_openclip(encoder, -1)}
    ldm_layout.save(str(tmp_path / "short.safetensors"), state)
    with pytest.raises(ValueError, match=r"1 resblocks.*num_hidden_layers=2"):
        checkpoint.load_single_file_models(str(tmp_path / "short.safetensors"), model_dir)


@pytest.mark.parametrize("with_sd", [False, True], ids=["control-only", "with-sd-model"])
def test_controlnet_file_loads_the_builders_values(tmp_path, sd15_file, with_sd):
    """lllyasviel's `control_sd15_canny.pth` holds `control_model.*` and a whole SD1.5 model; only the former is
    read, onto the Canny network `ControlNetModel` derives from the base folder's UNet config."""
    model_dir, sd_path = sd15_file
    want = build_controlnet("sd15", seed=3)
    state = ldm_layout.ldm_controlnet(want)
    if with_sd:
        state.update(checkpoint.load_single_file(sd_path))
        assert any(k.startswith("model.diffusion_model.input_blocks.1.0.") for k in state)
    path = str(tmp_path / "control_sd15_canny.pth")
    ldm_layout.save(path, state)
    got = checkpoint.load_controlnet_file(path, model_dir)
    assert not got.training
    assert_equal_state(got, want)


@pytest.mark.parametrize("prefix", [checkpoint.UNET_PREFIX, checkpoint.VAE_PREFIX, checkpoint.TEXT_PREFIX])
def test_a_missing_prefix_is_refused(tmp_path, prefix):
    model_dir, _ = fx.write_checkpoint(str(tmp_path), "tiny")
    unet, vae = builders("tiny")
    state = {**ldm_layout.ldm_unet(unet), **ldm_layout.ldm_vae(vae), **ldm_layout.ldm_clip(folder_encoder(model_dir))}
    ldm_layout.save(str(tmp_path / "m.safetensors"), {k: v for k, v in state.items() if not k.startswith(prefix)})
    with pytest.raises(ValueError, match=prefix.replace(".", r"\.")):
        checkpoint.load_single_file_models(str(tmp_path / "m.safetensors"), model_dir)
    ldm_layout.save(str(tmp_path / "cn.safetensors"), state)        # an SD file is not a ControlNet
    with pytest.raises(ValueError, match=r"control_model\."):
        checkpoint.load_controlnet_file(str(tmp_path / "cn.safetensors"), model_dir)


@pytest.mark.parametrize("edit,match", [
    ("extra", r'Unexpected key\(s\) in state_dict: "label_emb\.0\.0\.weight"'),
    ("missing", r'Missing key\(s\) in state_dict: "conv_out\.bias"'),
])
def test_an_extra_or_missing_key_is_refused(tmp_path, edit, match):
    model_dir, _ = fx.write_checkpoint(str(tmp_path), "tiny")
    unet, vae = builders("tiny")
    state = {**ldm_layout.ldm_unet(unet), **ldm_layout.ldm_vae(vae), **ldm_layout.ldm_clip(folder_encoder(model_dir))}
    if edit == "extra":                         # a class-conditional LDM's label embedding
        state["model.diffusion_model.label_emb.0.0.weight"] = torch.zeros(128, 32)
    else:
        del state["model.diffusion_model.out.2.bias"]
    ldm_layout.save(str(tmp_path / "m.safetensors"), state)
    with pytest.raises(RuntimeError, match=match):
        checkpoint.load_single_file_models(str(tmp_path / "m.safetensors"), model_dir)


def test_a_file_of_another_family_is_refused(tmp_path, sd21_file):
    """An SD2.1 file on an SD1.5 folder: the shapes differ (cross-attention width, linear projections)."""
    sd15_dir = base_folder(tmp_path, "sd15")
    with pytest.raises(RuntimeError, match=r"size mismatch for down_blocks\.0\.attentions\.0\.proj_in\.weight"):
        checkpoint.load_single_file_models(sd21_file[1], sd15_dir)


def test_a_pickle_weights_only_rejects_is_refused(tmp_path):
    model_dir, _ = fx.write_checkpoint(str(tmp_path), "tiny")
    unet, _ = builders("tiny")
    path = str(tmp_path / "lightning.ckpt")
    torch.save({"state_dict": ldm_layout.ldm_unet(unet), "hyper_parameters": argparse.Namespace(lr=1e-4)}, path)
    with pytest.raises(ValueError, match=r"lightning\.ckpt cannot be read with torch\.load\(weights_only=True\).*"
                                         r"convert it to \.safetensors"):
        checkpoint.load_single_file_models(path, model_dir)
    with pytest.raises(ValueError, match="weights_only"):
        checkpoint.load_controlnet_file(path, model_dir)


N, H, W = 8, 64, 96
PNP = {"prompt": "a marble sculpture of a woman", "negative_prompt": "ugly blurry", "guidance_scale": 7.5,
       "n_timesteps": 5, "batch_size": 4, "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "seed": 1}


def test_cli_with_weights_writes_what_the_folder_run_writes(tmp_path, monkeypatch):
    from PIL import Image
    tfu._install_ops_for_testing(OracleOps())
    model_dir, _ = fx.write_checkpoint(str(tmp_path), "tiny")
    unet, vae = builders("tiny")
    weights = write_sd_file(str(tmp_path / "model.ckpt"), unet, vae, folder_encoder(model_dir))
    g = torch.Generator().manual_seed(0)
    frames = torch.nn.functional.interpolate(torch.rand(N, 3, 6, 10, generator=g), size=(48, 80), mode="bilinear")
    frames = (frames * 255).round().to(torch.uint8).permute(0, 2, 3, 1).numpy()
    data = tmp_path / "data" / "clip"
    os.makedirs(data)
    for i, f in enumerate(frames):
        Image.fromarray(f).save(data / f"{i:05d}.png")
    monkeypatch.chdir(tmp_path)
    outputs = {}
    for arm, extra in (("folder", []), ("file", ["--weights", weights])):
        common = ["--model_dir", model_dir, "--device", "cpu", *extra]
        run.main(["preprocess", *common, "--data_path", str(data), "--H", str(H), "--W", str(W), "--save_dir", arm,
                  "--sd_version", "1.5", "--steps", "10", "--batch_size", "4", "--save_steps", "5",
                  "--n_frames", str(N), "--inversion_prompt", "a woman running"])
        config = {**PNP, "data_path": str(data), "latents_path": arm, "sd_version": "1.5", "n_inversion_steps": 10,
                  "n_frames": N, "output_path": str(tmp_path / arm / "out")}
        with open(tmp_path / f"{arm}.yaml", "w") as f:
            json.dump(config, f)
        run.main(["edit", *common, "--config_path", str(tmp_path / f"{arm}.yaml")])
        latents = run.read_latents(str(tmp_path / arm / "sd_1.5" / "clip" / "steps_10" / f"nframes_{N}"))
        outputs[arm] = latents, run.read_frames(str(tmp_path / arm / "out" / "img_ode"), N)
    (want_latents, want_frames), (got_latents, got_frames) = outputs["folder"], outputs["file"]
    assert sorted(got_latents) == sorted(want_latents) and len(want_latents) == 6
    for t in want_latents:
        assert torch.equal(got_latents[t], want_latents[t]), t
    assert torch.equal(got_frames, want_frames) and want_frames.float().std() > 0
