"""LoRA adapters for FLUX and SD3: read an adapter file and map its factors onto the engine's reference-named weights.

An adapter stores, per upstream module (the names the BFL FLUX / Stability SD3 checkpoints use, model_io.py), a
low-rank update ΔW = (alpha / rank) · up @ down.  Two encodings are read:
  kohya  `lora_unet_<module with . -> _>.lora_down.weight` / `.lora_up.weight` / `.alpha`
  PEFT   `<module>.lora_A.weight` (down) / `.lora_B.weight` (up) / optional `.alpha`, optionally behind
         `diffusion_model.` (FLUX) or `model.diffusion_model.` (SD3)
A kohya name is resolved against the module names enumerated from the config (underscores are ambiguous:
`img_attn`, `adaLN_modulation`), never by splitting it.

The fused upstream modules split exactly as the checkpoint loader splits their weights: `qkv` and `linear1` split the
up rows into q / k / v (/ fc1), `linear2` splits the down columns into o_proj / fc2.  The k projection's weight takes
its share (only the k bias is dropped, quirk Q3).  MMDiT.apply_lora merges the result into the packed weights.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple, Union

import torch

from . import model_io
from .config import MMDiTConfig
from .weights import mmdit_param_specs

Tensor = torch.Tensor

_REJECTED = ("hada_", "lokr_", "dora_scale")                     # LyCORIS LoHa / LoKr and DoRA
_SKIPPED = ("lora_te", "text_encoder")                           # text-encoder adapters: not part of this model
_PEFT_PREFIXES = ("model.diffusion_model.", "diffusion_model.")
_KOHYA = "lora_unet_"
_SUFFIXES = {
    ".lora_down.weight": "down", ".lora_up.weight": "up", ".lora_A.weight": "down", ".lora_B.weight": "up",
    ".alpha": "alpha",
}


@dataclass
class LoRA:
    """A parsed adapter.  `targets` maps a reference-named weight (e.g.
    `unified_transformer_blocks.3.transformer_block.mlp.fc1.weight`) to fp32 CPU factors (up [out, r], down [r, in])
    with ΔW = up @ down; `alpha / rank` is folded into `up`.  Conv weights (SD3 `x_embedder.proj`) have their down
    factor in the engine's (kh, kw, cin) column order.  `skipped` lists the keys of modules this model does not have."""

    name: str
    targets: Dict[str, Tuple[Tensor, Tensor]]
    skipped: List[str] = field(default_factory=list)


def module_table(config: MMDiTConfig) -> Dict[str, Tuple[int, List[str]]]:
    """upstream module name -> (axis the factors split along: 0 = up rows, 1 = down columns, reference weight names)"""
    c = config
    table: Dict[str, Tuple[int, List[str]]] = {}

    def lin(up, ref, axis=0):
        table[up] = (axis, [f"{r}.weight" for r in ([ref] if isinstance(ref, str) else ref)])

    def qkv(up, base, extra=()):
        lin(up, [f"{base}.attn.{n}_proj" for n in "qkv"] + list(extra))

    if c.depth_unified > 0:                                          # BFL FLUX layout
        for i in range(c.depth_multimodal):
            for s, stream in (("img", "image_transformer_block"), ("txt", "text_transformer_block")):
                b, u = f"multimodal_transformer_blocks.{i}.{stream}", f"double_blocks.{i}.{s}"
                qkv(f"{u}_attn.qkv", b)
                lin(f"{u}_attn.proj", b + ".attn.o_proj")
                lin(f"{u}_mlp.0", b + ".mlp.fc1")
                lin(f"{u}_mlp.2", b + ".mlp.fc2")
                lin(f"{u}_mod.lin", b + ".adaLN_modulation.layers.1")
        for i in range(c.depth_unified):
            b, u = f"unified_transformer_blocks.{i}.transformer_block", f"single_blocks.{i}"
            qkv(u + ".linear1", b, [b + ".mlp.fc1"])
            lin(u + ".linear2", [b + ".attn.o_proj", b + ".mlp.fc2"], axis=1)
            lin(u + ".modulation.lin", b + ".adaLN_modulation.layers.1")
        embed = {"img_in": "x_embedder.proj", "txt_in": "context_embedder",
                 "time_in.in_layer": "t_embedder.mlp.layers.0", "time_in.out_layer": "t_embedder.mlp.layers.2",
                 "vector_in.in_layer": "y_embedder.mlp.layers.0", "vector_in.out_layer": "y_embedder.mlp.layers.2",
                 "final_layer.linear": "final_layer.linear",
                 "final_layer.adaLN_modulation.1": "final_layer.adaLN_modulation.layers.1"}
        if c.guidance_embed:                                         # FLUX.1-dev's guidance embedder
            embed.update({"guidance_in.in_layer": "guidance_in.mlp.layers.0",
                          "guidance_in.out_layer": "guidance_in.mlp.layers.2"})
    else:                                                            # Stability SD3 / SD3.5 layout
        for i in range(c.depth_multimodal):
            skip_text = i == c.depth_multimodal - 1                  # the last context block has no post-attention
            for blk, stream in (("x_block", "image_transformer_block"), ("context_block", "text_transformer_block")):
                b, u = f"multimodal_transformer_blocks.{i}.{stream}", f"joint_blocks.{i}.{blk}"
                qkv(f"{u}.attn.qkv", b)
                if not (skip_text and blk == "context_block"):
                    lin(f"{u}.attn.proj", b + ".attn.o_proj")
                    lin(f"{u}.mlp.fc1", b + ".mlp.fc1")
                    lin(f"{u}.mlp.fc2", b + ".mlp.fc2")
                lin(f"{u}.adaLN_modulation.1", b + ".adaLN_modulation.layers.1")
            if i in c.x_block_self_attn_layers:                      # SD3.5 Medium's MMDiT-X second attention
                b, u = f"multimodal_transformer_blocks.{i}.image_transformer_block", f"joint_blocks.{i}.x_block"
                lin(f"{u}.attn2.qkv", [f"{b}.attn2.{n}_proj" for n in "qkv"])
                lin(f"{u}.attn2.proj", b + ".attn2.o_proj")
        embed = {"x_embedder.proj": "x_embedder.proj", "context_embedder": "context_embedder",
                 "t_embedder.mlp.0": "t_embedder.mlp.layers.0", "t_embedder.mlp.2": "t_embedder.mlp.layers.2",
                 "y_embedder.mlp.0": "y_embedder.mlp.layers.0", "y_embedder.mlp.2": "y_embedder.mlp.layers.2",
                 "final_layer.linear": "final_layer.linear",
                 "final_layer.adaLN_modulation.1": "final_layer.adaLN_modulation.layers.1"}
    for up, ref in embed.items():
        lin(up, ref)
    return table


def _is_skipped(module: str) -> bool:
    # FLUX.1-dev's guidance embedder on a model without one (quirk Q1); with one, module_table lists it
    return module.startswith(("guidance_in.", "guidance_in_"))


def _split_key(key: str, kohya: Dict[str, str], table) -> Tuple[str, str]:
    """key -> (upstream module, "up" | "down" | "alpha"); module "" = a key of a module this model does not have"""
    for suffix, part in _SUFFIXES.items():
        if key.endswith(suffix):
            stem = key[: -len(suffix)]
            break
    else:
        raise KeyError(f"LoRA key {key!r} is neither a LoRA up / down factor nor an alpha")
    if stem.startswith(_KOHYA):
        flat = stem[len(_KOHYA):]
        if flat in kohya:
            return kohya[flat], part
        if _is_skipped(flat):
            return "", part
    else:
        for p in _PEFT_PREFIXES:
            if stem.startswith(p):
                stem = stem[len(p):]
                break
        if stem in table:
            return stem, part
        if _is_skipped(stem):
            return "", part
    raise KeyError(f"LoRA key {key!r} names no module of this model")


def _as_matrix(t: Tensor, what: str, key: str) -> Tensor:
    """fp32 CPU 2-D factor; a conv factor's (kh, kw, cin) columns in the engine's order (model_io OIHW -> OHWI)"""
    t = t.detach().to("cpu", torch.float32)
    if t.dim() == 4:
        if what == "up":
            if t.shape[2:] != (1, 1):
                raise ValueError(f"{key}: a conv LoRA up factor must be 1x1, got {tuple(t.shape)}")
            return t.reshape(t.shape[0], t.shape[1])
        return model_io._conv_oihw_to_ohwi(t).reshape(t.shape[0], -1)
    if t.dim() != 2:
        raise ValueError(f"{key}: expected a 2-D (or conv 4-D) factor, got shape {tuple(t.shape)}")
    return t.contiguous()


def load_lora(path_or_state_dict: Union[str, os.PathLike, Dict[str, Tensor]], config: MMDiTConfig,
              name: Optional[str] = None) -> LoRA:
    """Parse a kohya or PEFT LoRA (.safetensors path or state dict) for the model `config` describes.

    Raises ValueError for LyCORIS / DoRA keys, incomplete modules and shapes that do not match the model, and KeyError
    naming the first key that matches no module of the model.  Text-encoder keys, and guidance-embedder keys when the
    config has no guidance embedder (`guidance_embed`), are skipped and listed in `LoRA.skipped`."""
    if isinstance(path_or_state_dict, (str, os.PathLike)):
        path = os.fspath(path_or_state_dict)
        sd = model_io.load_safetensors(path)
        if name is None:
            name = os.path.splitext(os.path.basename(path))[0]
    else:
        sd = dict(path_or_state_dict)
    if name is None:
        name = "adapter"
    rejected = [k for k in sd if any(r in k for r in _REJECTED)]
    if rejected:
        raise ValueError(f"LoRA key {rejected[0]!r}: LyCORIS (LoHa / LoKr) and DoRA adapters are not supported")
    table = module_table(config)
    kohya = {m.replace(".", "_"): m for m in table}
    shapes = {n: s for n, s, _ in mmdit_param_specs(config)}
    factors: Dict[str, Dict[str, Tensor]] = {}
    skipped: List[str] = []
    for key, v in sd.items():
        if key.startswith(_SKIPPED):
            skipped.append(key)
            continue
        module, part = _split_key(key, kohya, table)
        if not module:
            skipped.append(key)
            continue
        factors.setdefault(module, {})[part] = v

    targets: Dict[str, Tuple[Tensor, Tensor]] = {}
    for module, f in factors.items():
        if "up" not in f or "down" not in f:
            raise ValueError(f"LoRA module {module!r} lacks its {'up' if 'up' not in f else 'down'} factor")
        up, down = _as_matrix(f["up"], "up", module), _as_matrix(f["down"], "down", module)
        rank = down.shape[0]
        axis, refs = table[module]
        outs = [shapes[r][0] for r in refs]
        ins = [math.prod(shapes[r][1:]) for r in refs]
        want_up = (sum(outs) if axis == 0 else outs[0], rank)
        want_down = (rank, ins[0] if axis == 0 else sum(ins))
        if tuple(up.shape) != want_up or tuple(down.shape) != want_down:
            raise ValueError(f"LoRA module {module!r}: up {tuple(up.shape)} / down {tuple(down.shape)} do not match "
                             f"the model's weight (expected up {want_up}, down {want_down})")
        alpha = float(f["alpha"]) if "alpha" in f else float(rank)
        up = up * (alpha / rank)
        if axis == 0:
            for ref, u in zip(refs, torch.split(up, outs, dim=0)):
                targets[ref] = (u.contiguous(), down)
        else:
            for ref, d in zip(refs, torch.split(down, ins, dim=1)):
                targets[ref] = (up, d.contiguous())
    return LoRA(name=name, targets=targets, skipped=skipped)
