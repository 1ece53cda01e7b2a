"""CPU tier: LoRA files merged into the UNet and the text encoder (`lora.read`, `lora.merge`, `load_parts(loras=)`,
`run --lora`).

* kohya names copied from published files map to the modules they name, and kohya's full target sets map completely
  (192 UNet and 72 text-encoder modules on SD 1.5, 192 and 138 on SD 2.x);
* every merged weight passes `oracle/lora_merge.py`'s fp64 check (correctly rounded, or within its bound δ of a
  rounding midpoint), which rejects each fault a merge could make, restated in plain torch;
* the kohya, diffusers, PEFT and attention-processor layouts, and 2-D and 1x1 LoRAs on 1x1 convs and linear
  projections, merge to the same bits; two LoRAs pass the check of their sum;
* each refusal raises before any weight changes;
* a model that already ran a TokenFlow edit edits after a merge as a fresh model holding the merged weights;
* `run preprocess` and `run edit` with `--lora` write what the same runs write on a folder of the merged models.
"""
import json
import os
import shutil

import pytest
import torch
from safetensors.torch import load_file, save_file

from oracle import lora_merge
from oracle.oracle_ops import OracleOps
from tokenflow_b200 import lora, pipeline, run, sd_unet
from tokenflow_b200 import synthetic_checkpoint as fx
from tokenflow_b200 import tokenflow_utils as tfu
from tokenflow_b200.editor import TokenFlowEditor, synthetic_inputs
from tokenflow_b200.scheduler import DDIMScheduler

# OpenCLIP ViT-H/14's text tower as SD 2.x's diffusers folders store it: the penultimate of 24 layers
OPENCLIP_H = {"hidden_size": 1024, "intermediate_size": 4096, "num_hidden_layers": 23, "num_attention_heads": 16,
              "hidden_act": "gelu", "projection_dim": 1024}
ALL = ("transformer", "conv", "text_encoder")


def meta_models(kind):
    from transformers import CLIPTextConfig, CLIPTextModel
    text = {**fx.CLIP_L, "hidden_act": "quick_gelu"} if kind == "sd15" else OPENCLIP_H
    with torch.device("meta"):
        unet = sd_unet.UNet2DConditionModel.from_config(fx.UNET_CONFIGS[kind])
        encoder = CLIPTextModel(CLIPTextConfig(**text))
    return unet, encoder


def kohya_state(unet, encoder, targets, rank=4, device="meta"):
    """A kohya LoRA's tensors of fitting shapes for `targets` [(model, path)]."""
    nets = {"unet": unet, "text_encoder": encoder}
    state = {}
    for model, name in targets:
        shape = nets[model].get_submodule(name).weight.shape
        stem = {"unet": "lora_unet_", "text_encoder": "lora_te_"}[model] + name.replace(".", "_")
        state[stem + ".lora_down.weight"] = torch.empty(rank, *shape[1:], device=device)
        state[stem + ".lora_up.weight"] = torch.empty(shape[0], rank, *([1, 1] if len(shape) == 4 else []),
                                                      device=device)
    return state


PUBLISHED = {
    "lora_unet_down_blocks_0_attentions_0_proj_in": "down_blocks.0.attentions.0.proj_in",
    "lora_unet_down_blocks_0_attentions_0_transformer_blocks_0_attn1_to_out_0":
        "down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_out.0",
    "lora_unet_down_blocks_0_attentions_0_transformer_blocks_0_ff_net_0_proj":
        "down_blocks.0.attentions.0.transformer_blocks.0.ff.net.0.proj",
    "lora_unet_mid_block_attentions_0_transformer_blocks_0_attn2_to_k":
        "mid_block.attentions.0.transformer_blocks.0.attn2.to_k",
    "lora_unet_up_blocks_3_attentions_2_proj_out": "up_blocks.3.attentions.2.proj_out",
    "lora_unet_down_blocks_1_resnets_0_conv1": "down_blocks.1.resnets.0.conv1",
    "lora_unet_down_blocks_1_downsamplers_0_conv": "down_blocks.1.downsamplers.0.conv",
    "lora_te_text_model_encoder_layers_11_mlp_fc2": "text_model.encoder.layers.11.mlp.fc2",
}


def test_published_kohya_names_map_to_the_modules_they_name():
    unet, encoder = meta_models("sd15")
    nets = {"lora_unet": unet, "lora_te": encoder}
    state = {}
    for key, path in PUBLISHED.items():
        shape = nets[key[:key.index("_", 5)]].get_submodule(path).weight.shape
        state[key + ".lora_down.weight"] = torch.empty(8, *shape[1:], device="meta")
        state[key + ".lora_up.weight"] = torch.empty(shape[0], 8, *([1, 1] if len(shape) == 4 else []), device="meta")
        state[key + ".alpha"] = torch.tensor(4.0)
    got = lora.resolve(unet, encoder, lora.parse(state))
    assert len(got) == len(PUBLISHED)
    for module, layer in got:
        net = nets[layer.key[:layer.key.index("_", 5)]]
        assert module is net.get_submodule(PUBLISHED[layer.key]) and layer.alpha == 4.0, layer.key


@pytest.mark.parametrize("kind,n_te", [("sd15", 72), ("sd21", 138)])
def test_a_full_kohya_target_set_maps_completely(kind, n_te):
    unet, encoder = meta_models(kind)
    targets = fx.lora_targets(unet, encoder, ("transformer", "text_encoder"))
    assert sum(m == "unet" for m, _ in targets) == 192 and sum(m == "text_encoder" for m, _ in targets) == n_te
    got = lora.resolve(unet, encoder, lora.parse(kohya_state(unet, encoder, targets)))
    nets = {"unet": unet, "text_encoder": encoder}
    assert [module for module, _ in got] == [nets[m].get_submodule(n) for m, n in targets]
    locon = fx.lora_targets(unet, encoder, ("conv",))
    assert len(lora.resolve(unet, encoder, lora.parse(kohya_state(unet, encoder, locon)))) == len(locon) > 0


@pytest.fixture(scope="module")
def tiny(tmp_path_factory):
    root = tmp_path_factory.mktemp("tiny")
    model_dir, _ = fx.write_checkpoint(str(root), "tiny")
    return root, model_dir


def fp16_parts(model_dir):
    return pipeline.load_parts(model_dir, "cpu", torch.float16)


def write(root, name, parts, layout="kohya", rank=8, targets=ALL, alpha=4, seed=1):
    path = str(root / name)
    fx.write_lora(path, parts.unet, parts.text_encoder, layout, rank, targets, alpha, seed)
    return path


def test_a_merge_passes_the_fp64_check(tiny):
    root, model_dir = tiny
    parts = fp16_parts(model_dir)
    path = write(root, "a.safetensors", parts)
    before = lora_merge.weights(parts.unet, parts.text_encoder)
    changed = lora.merge(parts.unet, parts.text_encoder, [(path, 0.7)])
    assert len(changed) == len(load_file(path)) // 3
    near, total = lora_merge.check_merge(parts.unet, parts.text_encoder, before, [(load_file(path), 0.7)])
    assert total > 5_000_000 and near < 0.02 * total


def plain_merge(parts, tensors, scale, coef=lambda s, a, r: s * a / r, missing_alpha=lambda r: r, fp16_add=False,
                product=lambda up, down: up @ down, flatten=lambda d: d.reshape(d.shape[0], -1), moved=None):
    """A merge of a kohya file restated in plain torch, with one of the faults a merge could make injected."""
    nets = {"unet": parts.unet, "text_encoder": parts.text_encoder}
    table = {}
    for model, prefix in (("unet", "lora_unet_"), ("text_encoder", "lora_te_")):
        for name, _ in nets[model].named_modules():
            table[prefix + name.replace(".", "_")] = (model, name)
    with torch.no_grad():
        for stem in {k.split(".", 1)[0] for k in tensors}:
            model, name = table[stem]
            w = nets[model].get_submodule((moved or {}).get(name, name)).weight
            down, up = tensors[stem + ".lora_down.weight"].float(), tensors[stem + ".lora_up.weight"].float()
            r = down.shape[0]
            alpha = float(tensors[stem + ".alpha"]) if stem + ".alpha" in tensors else missing_alpha(r)
            delta = coef(scale, alpha, r) * product(up.reshape(up.shape[0], r), flatten(down)).reshape(w.shape)
            w.copy_(w + delta.half() if fp16_add else w.float() + delta)


def _square(up, down):
    """up and down swapped where the product still fits (out = in = rank)."""
    return down @ up if up.shape[0] == up.shape[1] == down.shape[1] else up @ down


FAULTS = {
    "alpha-ignored": dict(coef=lambda s, a, r: s),
    "scale-twice": dict(coef=lambda s, a, r: s * s * a / r),
    "fp16-delta-added-in-fp16": dict(fp16_add=True),
    "up-down-swapped": dict(product=_square),
    "conv-kernel-flattened-channels-last": dict(
        flatten=lambda d: (d.permute(0, 2, 3, 1) if d.dim() == 4 else d).reshape(d.shape[0], -1)),
    "neighbouring-block": dict(moved={"down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_q":
                                      "down_blocks.0.attentions.1.transformer_blocks.0.attn1.to_q"}),
    "missing-alpha-read-as-1": dict(missing_alpha=lambda r: 1.0),
}


@pytest.mark.parametrize("fault", list(FAULTS))
def test_the_fp64_check_rejects_a_faulty_merge(tiny, fault):
    root, model_dir = tiny
    parts = fp16_parts(model_dir)
    rank, alpha = {"up-down-swapped": (32, 4), "missing-alpha-read-as-1": (8, None)}.get(fault, (8, 4))
    path = write(root, f"{fault}.safetensors", parts, rank=rank, alpha=alpha)
    files = [(load_file(path), 0.7)]
    before = lora_merge.weights(parts.unet, parts.text_encoder)
    plain_merge(parts, files[0][0], 0.7)                       # the restatement without a fault passes
    lora_merge.check_merge(parts.unet, parts.text_encoder, before, files)
    parts = fp16_parts(model_dir)
    plain_merge(parts, files[0][0], 0.7, **FAULTS[fault])
    with pytest.raises(AssertionError):
        lora_merge.check_merge(parts.unet, parts.text_encoder, before, files)


def merged_state(parts):
    return {**{"unet." + k: v for k, v in parts.unet.state_dict().items()},
            **{"te." + k: v for k, v in parts.text_encoder.state_dict().items()}}


def assert_same_state(got, want):
    assert list(got) == list(want)
    for k in want:
        assert torch.equal(got[k], want[k]), k


def test_every_layout_merges_the_same_bits(tiny):
    root, model_dir = tiny
    results = {}
    for layout, fmt, targets in (("kohya", "safetensors", ALL), ("diffusers", "bin", ALL), ("peft", "safetensors", ALL),
                                 ("kohya", "safetensors", ("attention",)), ("processor", "bin", ("attention",))):
        parts = fp16_parts(model_dir)
        path = write(root, f"{layout}-{len(targets)}.{fmt}", parts, layout, targets=targets)
        lora.merge(parts.unet, parts.text_encoder, [(path, 0.7)])
        results[(layout, targets)] = merged_state(parts)
    assert_same_state(results[("diffusers", ALL)], results[("kohya", ALL)])
    assert_same_state(results[("peft", ALL)], results[("kohya", ALL)])
    assert_same_state(results[("processor", ("attention",))], results[("kohya", ("attention",))])
    assert not torch.equal(results[("kohya", ALL)]["unet.down_blocks.0.resnets.0.conv1.weight"],
                           fp16_parts(model_dir).unet.down_blocks[0].resnets[0].conv1.weight)


def test_2d_and_1x1_loras_fit_1x1_convs_and_linear_projections(tiny):
    """SD 1.x's proj_in / proj_out are 1x1 convs, SD 2.x's linear layers: a LoRA saved either way fits both."""
    root, model_dir = tiny
    parts = fp16_parts(model_dir)
    path = write(root, "proj4d.safetensors", parts, targets=("transformer",))
    tensors = load_file(path)
    flat = {k: (v.flatten(1) if v.dim() == 4 else v) for k, v in tensors.items()}
    assert any(v.dim() == 4 for v in tensors.values()) and all(v.dim() <= 2 for v in flat.values())
    save_file(flat, str(root / "proj2d.safetensors"))
    conv = fp16_parts(model_dir)
    lora.merge(conv.unet, conv.text_encoder, [(str(root / "proj2d.safetensors"), 0.7)])
    lora.merge(parts.unet, parts.text_encoder, [(path, 0.7)])
    assert_same_state(merged_state(conv), merged_state(parts))
    with torch.device("meta"):
        linear = sd_unet.UNet2DConditionModel.from_config({**fx.TINY_UNET, "use_linear_projection": True})
    state = fp16_parts(model_dir).unet.state_dict()
    linear.load_state_dict({k: (v.flatten(1) if ".proj_" in k and v.dim() == 4 else v) for k, v in state.items()},
                           assign=True)
    lora.merge(linear, conv.text_encoder, [(path, 0.7)])
    for k, v in parts.unet.state_dict().items():
        assert torch.equal(linear.state_dict()[k], v.flatten(1) if ".proj_" in k and v.dim() == 4 else v), k


def test_two_loras_pass_the_fp64_check_of_their_sum(tiny):
    root, model_dir = tiny
    parts = fp16_parts(model_dir)
    a = write(root, "two-a.safetensors", parts, rank=8, alpha=4, seed=2)
    b = write(root, "two-b.safetensors", parts, rank=4, alpha=None, seed=3, targets=("attention", "text_encoder"))
    before = lora_merge.weights(parts.unet, parts.text_encoder)
    lora.merge(parts.unet, parts.text_encoder, [(a, 0.7), (lora.read(b), -0.5)])
    lora_merge.check_merge(parts.unet, parts.text_encoder, before, [(load_file(a), 0.7), (load_file(b), -0.5)])


ATTN = "down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_q"
KOHYA_ATTN = "lora_unet_" + ATTN.replace(".", "_")
REFUSALS = {
    "no-module": ({"lora_unet_down_blocks_9_attentions_0_proj_in.lora_down.weight": (4, 32),
                   "lora_unet_down_blocks_9_attentions_0_proj_in.lora_up.weight": (32, 4)}, None,
                  r"'lora_unet_down_blocks_9_attentions_0_proj_in' maps to no Linear or Conv2d module"),
    "not-linear-or-conv": ({"unet.down_blocks.0.attentions.0.norm.lora.down.weight": (4, 32),
                            "unet.down_blocks.0.attentions.0.norm.lora.up.weight": (32, 4)}, None,
                           r"'unet\.down_blocks\.0\.attentions\.0\.norm' targets .*GroupNorm"),
    "shape": ({"lora_unet_mid_block_attentions_0_transformer_blocks_0_attn2_to_k.lora_down.weight": (4, 48),
               "lora_unet_mid_block_attentions_0_transformer_blocks_0_attn2_to_k.lora_up.weight": (128, 4)}, None,
              r"attn2_to_k' \(down \[4, 48\], up \[128, 4\]\) does not fit the weight \[128, 32\]"),
    "twice": ({f"unet.{ATTN}.lora_A.weight": (4, 32), f"unet.{ATTN}.lora_B.weight": (32, 4)}, None,
              rf"'{KOHYA_ATTN}' and 'unet\.{ATTN}' target the same module"),
    "loha": ({f"{KOHYA_ATTN}.hada_w1_a": (32, 4)}, None, r"hada_w1_a.*LyCORIS"),
    "lokr": ({f"{KOHYA_ATTN}.lokr_w1": (4, 4)}, None, "LyCORIS"),
    "cp-conv": ({"lora_unet_down_blocks_1_resnets_0_conv1.lora_mid.weight": (4, 4, 3, 3)}, None, "LyCORIS"),
    "dora": ({f"{KOHYA_ATTN}.dora_scale": (1, 32)}, None, "LyCORIS"),
    "diff": ({"lora_unet_conv_in.diff": (32, 4, 3, 3)}, None, "LyCORIS"),
    "oft": ({f"{KOHYA_ATTN}.oft_blocks": (4, 8, 8)}, None, "LyCORIS"),
    "sdxl-te1": ({"lora_te1_text_model_encoder_layers_0_mlp_fc1.lora_down.weight": (4, 32)}, None, "SDXL"),
    "sdxl-te2": ({"lora_te2_text_model_encoder_layers_0_mlp_fc1.lora_down.weight": (4, 32)}, None, "SDXL"),
    "sdxl-diffusers": ({"text_encoder_2.text_model.encoder.layers.0.mlp.fc1.lora.down.weight": (4, 32)}, None,
                       "SDXL"),
    "sdxl-metadata": ({}, {"ss_base_model_version": "sdxl_base_v1-0"}, r"sdxl_base_v1-0.*SDXL"),
}


@pytest.mark.parametrize("case", list(REFUSALS))
def test_a_refusal_raises_before_any_weight_changes(tiny, case):
    root, model_dir = tiny
    parts = fp16_parts(model_dir)
    good = write(root, "good.safetensors", parts, targets=("attention",))
    extra, metadata, match = REFUSALS[case]
    tensors = load_file(good)                                   # valid layers come first in the file
    g = torch.Generator().manual_seed(0)
    tensors.update({k: torch.randn(shape, generator=g).half() for k, shape in extra.items()})
    bad = str(root / f"bad-{case}.safetensors")
    save_file(tensors, bad, metadata=metadata)
    want = merged_state(parts)
    with pytest.raises(ValueError, match=match):
        lora.merge(parts.unet, parts.text_encoder, [(good, 1.0), (bad, 1.0)])
    assert_same_state(merged_state(parts), want)


def _edit(unet, steps=2, n=4):
    cfg = {"n_frames": n, "batch_size": 2, "n_timesteps": steps, "guidance_scale": 7.5, "mode": "pnp",
           "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "fused_pass": True, "keyframe_seed": 1}
    x, text, pnp, src = synthetic_inputs(n, 16, unet.config.cross_attention_dim, steps, seed=1, ctx_len=7)
    ed = TokenFlowEditor(unet, DDIMScheduler(), tfu, cfg, text, pnp, source_latents=lambda t: src[t])
    ed.init_method()
    return ed.sample_loop(x)


def test_a_merge_after_a_tokenflow_edit_takes_effect(tiny):
    """The merge writes with copy_, which bumps each weight's version: the TokenFlow block's cached fused q/k/v
    weight is re-made, so the next edit runs the merged weights."""
    tfu._install_ops_for_testing(OracleOps())
    root, model_dir = tiny
    parts = pipeline.load_parts(model_dir, "cpu", torch.float32)
    path = write(root, "after.safetensors", parts, targets=("transformer",))
    unet = parts.unet
    attn = unet.down_blocks[0].attentions[0].transformer_blocks[0].attn1
    cached = tfu._fused_weight(attn, ("to_q", "to_k", "to_v"), torch.float16)
    _edit(unet)
    lora.merge(unet, parts.text_encoder, [(path, 0.7)])
    fresh = sd_unet.UNet2DConditionModel.from_config(fx.TINY_UNET).eval()
    fresh.load_state_dict(unet.state_dict())
    fused = tfu._fused_weight(attn, ("to_q", "to_k", "to_v"), torch.float16)
    assert not torch.equal(fused, cached)
    assert torch.equal(fused, torch.cat([attn.to_q.weight, attn.to_k.weight, attn.to_v.weight]).half())
    assert torch.equal(_edit(unet), _edit(fresh))


def test_cli_parses_lora_flags():
    assert run.parse_lora("a.safetensors:0.7") == ("a.safetensors", 0.7)
    assert run.parse_lora("b.safetensors") == ("b.safetensors", 1.0)
    assert run.parse_lora("C:\\loras\\c.safetensors") == ("C:\\loras\\c.safetensors", 1.0)
    assert run.parse_lora("d:e.pt:-0.5") == ("d:e.pt", -0.5)


N, H, W = 8, 64, 96
PNP = {"prompt": "a marble sculpture of a woman", "negative_prompt": "ugly blurry", "guidance_scale": 7.5,
       "n_timesteps": 5, "batch_size": 4, "pnp_attn_t": 0.5, "pnp_f_t": 0.8, "seed": 1}


def write_merged_folder(parts, model_dir, dst, unet_config):
    """`model_dir` with the UNet and the text encoder replaced by `parts`' (merged) ones."""
    shutil.copytree(model_dir, dst)
    fx.write_model(os.path.join(dst, "unet"), parts.unet, unet_config)
    parts.text_encoder.save_pretrained(os.path.join(dst, "text_encoder"))
    return dst


def test_cli_with_lora_writes_what_the_merged_folder_writes(tmp_path, monkeypatch):
    from PIL import Image
    tfu._install_ops_for_testing(OracleOps())
    model_dir, _ = fx.write_checkpoint(str(tmp_path), "tiny")
    base = pipeline.load_parts(model_dir, "cpu", torch.float32)
    a = str(tmp_path / "a.safetensors")
    b = str(tmp_path / "b.pt")
    fx.write_lora(a, base.unet, base.text_encoder, "kohya", 8, ALL, 4, 1)
    fx.write_lora(b, base.unet, base.text_encoder, "peft", 4, ("attention", "text_encoder"), None, 2)
    merged = pipeline.load_parts(model_dir, "cpu", torch.float32, loras=[(a, 0.7), (b, 1.0)])
    merged_dir = write_merged_folder(merged, model_dir, str(tmp_path / "merged"), fx.TINY_UNET)
    g = torch.Generator().manual_seed(0)
    frames = torch.nn.functional.interpolate(torch.rand(N, 3, 6, 10, generator=g), size=(48, 80), mode="bilinear")
    frames = (frames * 255).round().to(torch.uint8).permute(0, 2, 3, 1).numpy()
    data = tmp_path / "data" / "clip"
    os.makedirs(data)
    for i, f in enumerate(frames):
        Image.fromarray(f).save(data / f"{i:05d}.png")
    monkeypatch.chdir(tmp_path)
    outputs = {}
    for arm, common in (("folder", ["--model_dir", merged_dir]),
                        ("lora", ["--model_dir", model_dir, "--lora", f"{a}:0.7", "--lora", b])):
        common = [*common, "--device", "cpu"]
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
    (want_latents, want_frames), (got_latents, got_frames) = outputs["folder"], outputs["lora"]
    assert sorted(got_latents) == sorted(want_latents) and len(want_latents) == 6
    for t in want_latents:
        assert torch.equal(got_latents[t], want_latents[t]), t
    assert torch.equal(got_frames, want_frames) and want_frames.float().std() > 0
    import yaml
    with open(tmp_path / "lora" / "out" / "config.yaml") as f:
        assert yaml.safe_load(f)["loras"] == [{"path": a, "scale": 0.7}, {"path": b, "scale": 1.0}]
    with open(tmp_path / "folder" / "out" / "config.yaml") as f:
        assert "loras" not in yaml.safe_load(f)
