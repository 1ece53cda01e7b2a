"""CPU tier: loading diffusers model folders (tokenflow_b200/checkpoint.py) and the `from_config` of the restated models.

* the published SD1.5 / SD2.1 / VAE / Canny ControlNet configs give exactly the configs `build_*` uses;
* a loaded module has the keys, shapes and values of `build_*(kind)` after `load_state_dict`: tiny for values (fp32
  safetensors, the fp16 variant, a sharded index, .bin files), SD1.5 / SD2.1 / the Canny ControlNet on the meta device
  for keys and shapes;
* a VAE saved under the attention names of the published SD VAE files (query, key, value, proj_attn) loads with
  strict=True to the same values;
* `from_config` refuses SDXL-, depth- and inpainting-shaped configs and every other setting it does not compute, with
  a ValueError naming the key;
* `text_embeds` is the reference's `get_text_embeds`: direct CLIPTextModel calls in its order, the prompt truncated,
  the negative prompt not (a too long one raises the encoder's ValueError, as the reference's call does).
"""
import os

import pytest
import torch

from tokenflow_b200 import synthetic_checkpoint as fx

from tokenflow_b200 import checkpoint, sd_unet
from tokenflow_b200.controlnet import ControlNetModel, build_controlnet, sd15_canny_config
from tokenflow_b200.vae import AutoencoderKL, build_vae, sd_config


def test_published_configs_are_the_builders_configs():
    assert sd_unet.UNet2DConditionModel.from_config(fx.SD15_UNET).config == sd_unet.sd15_config()
    assert sd_unet.UNet2DConditionModel.from_config(fx.SD21_UNET).config == sd_unet.sd21_config()
    assert sd_unet.UNet2DConditionModel.from_config(fx.TINY_UNET).config == sd_unet.tiny_config()
    base = sd_unet.UNet2DConditionModel.from_config({**fx.SD21_UNET, "sample_size": 64, "upcast_attention": False})
    assert base.config.sample_size == 64 and base.config.num_heads == (5, 10, 20, 20)
    explicit = {**fx.SD21_UNET, "attention_head_dim": 64, "num_attention_heads": [5, 10, 20, 20]}
    assert sd_unet.UNet2DConditionModel.from_config(explicit).config == sd_unet.sd21_config()
    assert AutoencoderKL.from_config(fx.SD_VAE).config == sd_config()
    assert ControlNetModel.from_config(fx.SD15_CANNY).config == sd15_canny_config()


def _equal_state(a, b):
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb)
    for k in sa:
        assert sa[k].shape == sb[k].shape and sa[k].dtype == sb[k].dtype, k
        assert torch.equal(sa[k], sb[k]), k


@pytest.mark.parametrize("variant,fmt,shards", [(None, "safetensors", 1), ("fp16", "safetensors", 1),
                                                (None, "safetensors", 3), ("fp16", "safetensors", 2),
                                                (None, "bin", 1), (None, "bin", 2)])
def test_tiny_modules_load_the_builders_values(tmp_path, variant, fmt, shards):
    dtype = torch.float16 if variant == "fp16" else None
    model_dir, cn_dir = fx.write_checkpoint(str(tmp_path), "tiny", controlnet=True, variant=variant, dtype=dtype,
                                            fmt=fmt, shards=shards)
    want_unet = sd_unet.build_unet("tiny", seed=1)
    want_vae = build_vae("tiny", seed=1)
    want_cn = build_controlnet("tiny", seed=3)
    if dtype is not None:                       # the fp16 files hold the fp16 rounding of the same values
        with torch.no_grad():
            for m in (want_unet, want_vae, want_cn):
                for p in m.parameters():
                    p.copy_(p.half().float())
    unet = checkpoint.load_unet(model_dir, variant=variant)
    vae = checkpoint.load_vae(model_dir, variant=variant)
    cn = checkpoint.load_controlnet(cn_dir, variant=variant)
    for got, want in ((unet, want_unet), (vae, want_vae), (cn, want_cn)):
        assert not got.training
        assert not any(p.is_meta for p in got.parameters())
        _equal_state(got, want)
    half = checkpoint.load_unet(model_dir, dtype=torch.float16, variant=variant)
    assert all(p.dtype == torch.float16 for p in half.parameters())
    assert half.conv_in.weight.is_contiguous()          # channels_last only for CUDA fp16


@pytest.mark.parametrize("variant,shards", [(None, 1), ("fp16", 2)])
def test_vae_with_the_published_attention_names_loads(tmp_path, variant, shards):
    """The SD 1.x / 2.x VAE files keep diffusers' pre-0.14 names for the mid-block attentions (query, key, value,
    proj_attn); load_vae renames them, as diffusers does, and loads them with strict=True to the same values."""
    from tokenflow_b200.checkpoint import load_weights, renamed_vae_attention
    dtype = torch.float16 if variant else None
    model_dir, _ = fx.write_checkpoint(str(tmp_path), "tiny", variant=variant, dtype=dtype, shards=shards,
                                      deprecated_vae=True)
    stored = load_weights(os.path.join(model_dir, "vae"), variant)
    old = [k for k in stored if ".attentions.0." in k and not k.split(".attentions.0.")[1].startswith("group_norm")]
    assert sorted({k.split(".attentions.0.")[1] for k in old}) == [
        "key.bias", "key.weight", "proj_attn.bias", "proj_attn.weight", "query.bias", "query.weight", "value.bias",
        "value.weight"]
    assert len(old) == 16                                   # encoder and decoder mid blocks
    with pytest.raises(RuntimeError, match="query"):
        build_vae("tiny").load_state_dict(stored, strict=True)
    want = build_vae("tiny", seed=1)
    if dtype is not None:
        want = want.half().float()
    _equal_state(checkpoint.load_vae(model_dir, variant=variant), want)
    # today's names go through unchanged
    current = want.state_dict()
    assert renamed_vae_attention(current).keys() == current.keys()


def test_missing_weights_name_the_files(tmp_path):
    model_dir, _ = fx.write_checkpoint(str(tmp_path), "tiny")
    with pytest.raises(FileNotFoundError, match="diffusion_pytorch_model.fp16.safetensors"):
        checkpoint.load_unet(model_dir, variant="fp16")


def test_strict_load_refuses_a_mismatched_state(tmp_path):
    model_dir, _ = fx.write_checkpoint(str(tmp_path), "tiny")
    import json
    with open(os.path.join(model_dir, "unet", "config.json"), "w") as f:
        json.dump({**fx.TINY_UNET, "use_linear_projection": True}, f)
    with pytest.raises(RuntimeError):
        checkpoint.load_unet(model_dir)


@pytest.mark.parametrize("kind", ["sd15", "sd21"])
def test_full_size_configs_have_the_builders_keys_and_shapes(kind):
    with torch.device("meta"):
        got = sd_unet.UNet2DConditionModel.from_config(fx.UNET_CONFIGS[kind])
        want = sd_unet.UNet2DConditionModel({"sd15": sd_unet.sd15_config, "sd21": sd_unet.sd21_config}[kind]())
        pairs = [(got, want)]
        if kind == "sd15":
            pairs.append((AutoencoderKL.from_config(fx.SD_VAE), AutoencoderKL(sd_config())))
            pairs.append((ControlNetModel.from_config(fx.SD15_CANNY), ControlNetModel(sd15_canny_config())))
    for a, b in pairs:
        sa, sb = a.state_dict(), b.state_dict()
        assert list(sa) == list(sb)
        assert all(sa[k].shape == sb[k].shape for k in sa)
        b.load_state_dict(sa, strict=True, assign=True)


REFUSED_UNET = [
    ("in_channels", 5), ("in_channels", 9), ("out_channels", 8), ("addition_embed_type", "text_time"),
    ("transformer_layers_per_block", [1, 2, 10]), ("transformer_layers_per_block", 2), ("class_embed_type", "timestep"),
    ("num_class_embeds", 1000), ("time_cond_proj_dim", 256), ("mid_block_type", None),
    ("mid_block_type", "UNetMidBlock2DSimpleCrossAttn"), ("encoder_hid_dim", 1024), ("only_cross_attention", True),
    ("dual_cross_attention", True), ("center_input_sample", True), ("norm_eps", 1e-6), ("act_fn", "gelu"),
    ("resnet_time_scale_shift", "scale_shift"), ("conv_in_kernel", 7), ("time_embedding_type", "fourier"),
    ("flip_sin_to_cos", False), ("freq_shift", 1), ("layers_per_block", [2, 2, 2, 2]),
    ("cross_attention_dim", [768, 1024, 1024, 1024]),
    ("down_block_types", ["DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"]),
    ("down_block_types", ["CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D",
                          "SimpleCrossAttnDownBlock2D"]),
    ("up_block_types", ["UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "AttnUpBlock2D"]),
]


@pytest.mark.parametrize("key,value", REFUSED_UNET, ids=[f"{k}={v}" for k, v in REFUSED_UNET])
def test_unet_from_config_refuses_what_it_does_not_compute(key, value):
    with pytest.raises(ValueError, match=key):
        sd_unet.UNet2DConditionModel.from_config({**fx.SD15_UNET, key: value})


def test_sdxl_depth_and_inpainting_configs_are_refused():
    sdxl = {**fx.SD15_UNET, "addition_embed_type": "text_time", "addition_time_embed_dim": 256,
            "transformer_layers_per_block": [1, 2, 10], "block_out_channels": [320, 640, 1280],
            "down_block_types": ["DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"],
            "up_block_types": ["CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"], "cross_attention_dim": 2048,
            "projection_class_embeddings_input_dim": 2816}
    with pytest.raises(ValueError, match="addition_embed_type='text_time'"):
        sd_unet.UNet2DConditionModel.from_config(sdxl)
    with pytest.raises(ValueError, match="in_channels=5"):
        sd_unet.UNet2DConditionModel.from_config({**fx.SD21_UNET, "in_channels": 5})
    with pytest.raises(ValueError, match="in_channels=9"):
        sd_unet.UNet2DConditionModel.from_config({**fx.SD15_UNET, "in_channels": 9})
    with pytest.raises(ValueError, match="in_channels=9"):
        ControlNetModel.from_config({**fx.SD15_CANNY, "in_channels": 9})


@pytest.mark.parametrize("key,value", [("scaling_factor", 0.13025), ("latent_channels", 16), ("in_channels", 4),
                                       ("shift_factor", 0.1159), ("use_quant_conv", False),
                                       ("mid_block_add_attention", False), ("act_fn", "gelu"),
                                       ("down_block_types", ["DownEncoderBlock2D"] * 3 + ["AttnDownEncoderBlock2D"])])
def test_vae_from_config_refuses_what_it_does_not_compute(key, value):
    with pytest.raises(ValueError, match=key):
        AutoencoderKL.from_config({**fx.SD_VAE, key: value})


@pytest.mark.parametrize("key,value", [("controlnet_conditioning_channel_order", "bgr"),
                                       ("global_pool_conditions", True), ("class_embed_type", "projection"),
                                       ("transformer_layers_per_block", 2), ("addition_embed_type", "text_time")])
def test_controlnet_from_config_refuses_what_it_does_not_compute(key, value):
    with pytest.raises(ValueError, match=key):
        ControlNetModel.from_config({**fx.SD15_CANNY, key: value})


def test_scheduler_is_read_from_the_checkpoint(tmp_path):
    model_dir, _ = fx.write_checkpoint(str(tmp_path), "tiny", scheduler=fx.SD21_V_SCHEDULER)
    assert checkpoint.load_scheduler(model_dir).prediction_type == "v_prediction"
    model_dir, _ = fx.write_checkpoint(str(tmp_path / "eps"), "tiny")
    sched = checkpoint.load_scheduler(model_dir)
    assert sched.prediction_type == "epsilon" and sched.steps_offset == 1


PROMPT = "a marble sculpture of a woman running"
NEGATIVE = "ugly blurry low res"


def test_text_embeds_is_the_references_get_text_embeds(tmp_path):
    model_dir, _ = fx.write_checkpoint(str(tmp_path), "tiny")
    tok, enc = checkpoint.load_text_encoder(model_dir)
    assert tok.model_max_length == 77 and not enc.training
    ids = tok(PROMPT).input_ids
    assert len(ids) > len(PROMPT.split()) + 2                # every word is several tokens
    got = checkpoint.text_embeds(tok, enc, PROMPT, NEGATIVE)

    def direct(text, truncation):
        kw = dict(truncation=True) if truncation else {}
        ids = tok(text, padding="max_length", max_length=77, return_tensors="pt", **kw).input_ids
        return enc(ids)[0]

    with torch.no_grad():
        want = torch.cat([direct(NEGATIVE, False), direct(PROMPT, True)])
    assert got.shape == (2, 77, 32) and torch.equal(got, want)
    # inversion cond and PnP guidance, as the drivers take them
    with torch.no_grad():
        assert torch.equal(checkpoint.text_embeds(tok, enc, PROMPT, "")[1:], direct(PROMPT, True))
        assert torch.equal(checkpoint.text_embeds(tok, enc, PROMPT, PROMPT).chunk(2)[0], direct(PROMPT, False))


def test_long_prompts_behave_as_the_references_call(tmp_path):
    model_dir, _ = fx.write_checkpoint(str(tmp_path), "tiny")
    tok, enc = checkpoint.load_text_encoder(model_dir)
    long = " ".join(["abc"] * 40)                            # 120 tokens
    got = checkpoint.text_embeds(tok, enc, long, NEGATIVE)   # the prompt is truncated to 77
    with torch.no_grad():
        ids = tok(long, padding="max_length", max_length=77, truncation=True, return_tensors="pt").input_ids
        assert torch.equal(got[1], enc(ids)[0][0])
        # the negative prompt is not truncated: 122 positions, and the encoder refuses them
        with pytest.raises(ValueError, match="max_position_embeddings"):
            ids = tok(long, padding="max_length", max_length=77, return_tensors="pt").input_ids
            enc(ids)
    with pytest.raises(ValueError, match="max_position_embeddings"):
        checkpoint.text_embeds(tok, enc, PROMPT, long)
