"""LoRA adapters merged into the UNet and the text encoder at load time, as diffusers' `load_lora_weights(file)`
followed by `fuse_lora(lora_scale=s)` merges them into a loaded model.

A LoRA file holds, for each adapted module, a down matrix D [r, in·kh·kw] (a conv LoRA stores it [r, in, kh, kw]), an
up matrix U [out, r] (or [out, r, 1, 1]) and optionally a scalar alpha.  Four key layouts are read:

    kohya-ss (LoCon convs too)       lora_unet_<path with _>  lora_te_<path with _>  .lora_down.weight / .lora_up.weight
    diffusers `save_lora_weights`    unet.<path>              text_encoder.<path>    .lora.down.weight / .lora.up.weight
    PEFT                             unet.<path>              text_encoder.<path>    .lora_A.weight / .lora_B.weight
    diffusers <= 0.16 attn. procs    [unet.]<...>.attn1.processor.to_q_lora         .down.weight / .up.weight
                                     (to_out_lora is to_out.0)

with an optional `<module key>.alpha`.  <path> is the module path in diffusers' names, which `sd_unet` and
transformers' CLIPTextModel both use.  A kohya name is looked up in a table built from the model's own
`named_modules()`: every nn.Linear and nn.Conv2d, its path with `.` replaced by `_`.

`merge` changes each targeted weight W [out, in, (kh, kw)] once:

    W <- round_to_dtype( float32(W) + sum_i s_i * (alpha_i / r_i) * (U_i @ D_i) )

with the product and the sum in fp32 on the model's device, TF32 off, the LoRAs added in the order given; a missing
alpha means alpha = r.  The down kernel is flattened as PyTorch stores a conv weight and the product reshaped back,
and a 2-D LoRA fits a 1x1 conv (SD 1.x's proj_in / proj_out) and a 1x1 conv LoRA a linear layer.  The weight is written in
place with `copy_` under no_grad, which bumps its version: the TokenFlow block's fused q/k/v weight
(`tokenflow_utils._fused_weight`) is re-made from it on the next forward.

Merge before a `TokenFlowEditor` or a `LatentInverter` is built: a captured CUDA graph holds the fused q/k/v weight it
was captured with.  LoRAs never touch the VAE or the ControlNet (diffusers does not apply them there either).

Refused with a ValueError naming the key, before any weight changes: a key that maps to no module, a module that is
neither Linear nor Conv2d, a shape that does not fit the module (both shapes named: an SD 1.5 LoRA on an SD 2.x model
fails here), one module given twice in one file, the LyCORIS types (LoHa `hada_*`, LoKr `lokr_*`, CP-decomposed
`lora_mid`, DoRA `dora_scale`, `.diff`, OFT `oft_*`), and SDXL files (`lora_te1_` / `lora_te2_` / `text_encoder_2.`
keys, or kohya's `ss_base_model_version` metadata naming sdxl).
"""
from __future__ import annotations

import contextlib
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch
import torch.nn as nn

from .checkpoint import _read_file

# (suffix, part); the bare ".down.weight" / ".up.weight" only under an attention processor
_PARTS = ((".lora_down.weight", "down"), (".lora_up.weight", "up"),
          (".lora.down.weight", "down"), (".lora.up.weight", "up"),
          (".lora_A.weight", "down"), (".lora_B.weight", "up"),
          (".down.weight", "down"), (".up.weight", "up"),
          (".alpha", "alpha"))
_LYCORIS = ("hada_", "lokr_", "lora_mid", "dora_scale", ".diff", "oft_")
_SDXL = ("lora_te1_", "lora_te2_", "text_encoder_2.")
_KOHYA = {"lora_unet_": "unet", "lora_te_": "text_encoder"}
_DIFFUSERS = {"unet.": "unet", "text_encoder.": "text_encoder"}


@dataclass
class Layer:
    """One adapted module of a file: `key` is the file's key stem (for messages), `model` "unet" or "text_encoder",
    `name` the module path, or kohya's underscore name when `kohya`."""
    key: str
    model: str
    name: str
    kohya: bool
    down: torch.Tensor
    up: torch.Tensor
    alpha: Optional[float]

    @property
    def rank(self) -> int:
        return self.down.shape[0]


@dataclass
class LoRA:
    path: str
    layers: List[Layer]


def _target(stem: str) -> Tuple[str, str, bool]:
    """(model, module name, kohya) of a key stem."""
    for prefix, model in _KOHYA.items():
        if stem.startswith(prefix):
            return model, stem[len(prefix):], True
    model = "unet"
    for prefix, m in _DIFFUSERS.items():
        if stem.startswith(prefix):
            model, stem = m, stem[len(prefix):]
            break
    else:
        if ".processor." not in stem:              # only the attention-processor layout may omit the "unet." prefix
            raise ValueError(f"LoRA key {stem!r} is in none of the kohya, diffusers, PEFT or attention-processor "
                             f"layouts")
    if ".processor." in stem:
        head, proc = stem.split(".processor.", 1)
        if model != "unet" or not proc.endswith("_lora"):
            raise ValueError(f"LoRA key {stem!r} is not an attention processor's <name>_lora")
        name = proc[:-len("_lora")]
        stem = f"{head}.{'to_out.0' if name == 'to_out' else name}"
    return model, stem, False


def parse(tensors: Dict[str, torch.Tensor], metadata: Optional[Dict[str, str]] = None, path: str = "<memory>") -> LoRA:
    """The LoRA of a file's tensors (and safetensors metadata), validated as far as it can be without the models."""
    base = (metadata or {}).get("ss_base_model_version", "")
    if base.lower().startswith("sdxl"):
        raise ValueError(f"{path}: ss_base_model_version={base!r}: SDXL LoRAs are not supported (SD 1.x / 2.x only)")
    groups: Dict[str, Dict[str, torch.Tensor]] = {}
    for key, value in tensors.items():
        if key.startswith(_SDXL):
            raise ValueError(f"{path}: LoRA key {key!r} is SDXL's second text encoder or its layout: SDXL LoRAs are "
                             f"not supported (SD 1.x / 2.x only)")
        if any(t in key for t in _LYCORIS):
            raise ValueError(f"{path}: LoRA key {key!r} is a LyCORIS type (LoHa, LoKr, CP-decomposed conv, DoRA, "
                             f"diff or OFT), not a LoRA: it is not supported")
        for suffix, part in _PARTS:
            if suffix in (".down.weight", ".up.weight") and ".processor." not in key:
                continue
            if key.endswith(suffix):
                groups.setdefault(key[:-len(suffix)], {})[part] = value
                break
        else:
            raise ValueError(f"{path}: LoRA key {key!r} is no down, up or alpha tensor of a LoRA layout")
    layers = []
    for stem, parts in groups.items():
        if "down" not in parts or "up" not in parts:
            missing = "down" if "down" not in parts else "up"
            raise ValueError(f"{path}: LoRA key {stem!r} has no {missing} weight")
        alpha = parts.get("alpha")
        if alpha is not None and alpha.numel() != 1:
            raise ValueError(f"{path}: LoRA key {stem + '.alpha'!r} has {alpha.numel()} elements, not 1")
        model, name, kohya = _target(stem)
        layers.append(Layer(stem, model, name, kohya, parts["down"], parts["up"],
                            None if alpha is None else float(alpha.reshape(()).item())))
    return LoRA(path, layers)


def read(path: str) -> LoRA:
    """The LoRA of a `.safetensors` file, or a `.pt` / `.ckpt` / `.bin` read with `torch.load(weights_only=True)`:
    parsed and validated as far as it can be without the models; nothing is applied."""
    metadata = None
    if path.endswith(".safetensors"):
        from safetensors import safe_open
        with safe_open(path, framework="pt") as f:
            metadata = f.metadata()
    return parse(_read_file(path), metadata, path)


def kohya_names(net: nn.Module) -> Dict[str, Tuple[str, nn.Module]]:
    """{path with `.` replaced by `_`: (path, module)} over every nn.Linear and nn.Conv2d of `net`; a name two modules
    share is refused."""
    table: Dict[str, Tuple[str, nn.Module]] = {}
    for name, module in net.named_modules():
        if isinstance(module, (nn.Linear, nn.Conv2d)):
            key = name.replace(".", "_")
            if key in table:
                raise ValueError(f"modules {table[key][0]!r} and {name!r} have the same kohya name {key!r}")
            table[key] = (name, module)
    return table


def _core(shape) -> tuple:
    """A shape with a trailing 1x1 kernel dropped."""
    shape = tuple(shape)
    return shape[:2] if len(shape) == 4 and shape[2:] == (1, 1) else shape


def resolve(unet: nn.Module, text_encoder: nn.Module, lora: LoRA) -> List[Tuple[nn.Module, Layer]]:
    """(module, layer) for every layer of `lora`, each module checked to be Linear or Conv2d, to fit the layer's
    shapes, and to be named once in the file."""
    models = {"unet": unet, "text_encoder": text_encoder}
    tables: Dict[str, Dict[str, Tuple[str, nn.Module]]] = {}
    out, seen = [], {}
    for layer in lora.layers:
        net = models[layer.model]
        if layer.kohya:
            if layer.model not in tables:
                tables[layer.model] = kohya_names(net)
            hit = tables[layer.model].get(layer.name)
            if hit is None:
                raise ValueError(f"{lora.path}: LoRA key {layer.key!r} maps to no Linear or Conv2d module of the "
                                 f"{layer.model}")
            module = hit[1]
        else:
            try:
                module = net.get_submodule(layer.name)
            except AttributeError:
                raise ValueError(f"{lora.path}: LoRA key {layer.key!r} maps to no module of the {layer.model} "
                                 f"({layer.name!r})") from None
            if not isinstance(module, (nn.Linear, nn.Conv2d)):
                raise ValueError(f"{lora.path}: LoRA key {layer.key!r} targets {layer.name!r}, a "
                                 f"{type(module).__name__}: only Linear and Conv2d take a LoRA")
        if id(module) in seen:
            raise ValueError(f"{lora.path}: LoRA keys {seen[id(module)]!r} and {layer.key!r} target the same module")
        seen[id(module)] = layer.key
        w, d, u = _core(module.weight.shape), _core(layer.down.shape), _core(layer.up.shape)
        if not (len(u) == 2 and u[1] == d[0] and u[0] == w[0] and d[1:] == w[1:]):
            raise ValueError(f"{lora.path}: LoRA key {layer.key!r} (down {list(layer.down.shape)}, up "
                             f"{list(layer.up.shape)}) does not fit the weight {list(module.weight.shape)} of "
                             f"{layer.model} module {type(module).__name__}")
        out.append((module, layer))
    return out


@contextlib.contextmanager
def _fp32_matmul():
    """fp32 GEMMs in full fp32 (TF32 off) for the duration."""
    previous = torch.get_float32_matmul_precision()
    torch.set_float32_matmul_precision("highest")
    try:
        yield
    finally:
        torch.set_float32_matmul_precision(previous)


def merge(unet: nn.Module, text_encoder: nn.Module,
          loras: Sequence[Tuple[Union[LoRA, str], float]]) -> List[nn.Module]:
    """Merge `[(LoRA or path, scale), ...]` into the UNet's and the text encoder's weights, in place, and return the
    modules changed.  Every file is read and every key resolved and checked before any weight changes.

    Merge before a `TokenFlowEditor` or a `LatentInverter` is built on these models: a captured CUDA graph holds the
    fused q/k/v weight of the model it was captured on."""
    plan: Dict[int, Tuple[nn.Module, list]] = {}
    for item, scale in loras:
        lora = read(item) if isinstance(item, str) else item
        for module, layer in resolve(unet, text_encoder, lora):
            alpha = layer.rank if layer.alpha is None else layer.alpha
            plan.setdefault(id(module), (module, []))[1].append((float(scale) * alpha / layer.rank, layer))
    with torch.no_grad(), _fp32_matmul():
        for module, terms in plan.values():
            w = module.weight
            acc = w.detach().to(torch.float32, copy=True)
            for c, layer in terms:
                up = layer.up.to(device=w.device, dtype=torch.float32).reshape(w.shape[0], -1)
                down = layer.down.to(device=w.device, dtype=torch.float32).reshape(layer.rank, -1)
                acc.add_((up @ down).reshape(w.shape), alpha=c)
            w.copy_(acc)
    return [module for module, _ in plan.values()]
