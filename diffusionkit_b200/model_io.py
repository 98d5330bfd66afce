"""Checkpoint key remapping: upstream (BFL FLUX / Stability SD3 / LDM VAE) safetensors layouts -> the parameter tree
this engine consumes (the reference's module-tree names, SURVEY.md App. C).

Restates the rules of the reference loaders (python/src/diffusionkit/mlx/model_io.py):
  flux_state_dict_adjustments        :130-311
  mmdit_state_dict_adjustments       :314-408
  vae_decoder_state_dict_adjustments :411-486, vae_encoder_state_dict_adjustments :489-571
as table-driven converters over torch tensors.  SURVEY.md §8 "next" row f1.  Downloading (huggingface_hub) is out of
scope — callers pass a local .safetensors path (the reference's `local_ckpt`).
"""
from __future__ import annotations

import re
from typing import Callable, Dict, Iterable, List, Optional, Tuple

import torch

Tensor = torch.Tensor


def load_safetensors(path: str) -> Dict[str, Tensor]:
    from safetensors.torch import load_file

    return load_file(path)


def _conv_oihw_to_ohwi(w: Tensor) -> Tensor:
    """PyTorch conv weight (O, I, kh, kw) -> mlx nn.Conv2d weight (O, kh, kw, I)"""
    return w.permute(0, 2, 3, 1).contiguous()


# ------------------------------------------------------------------------------------------------ FLUX (BFL layout)
_FLUX_STREAM = {"img": "image_transformer_block", "txt": "text_transformer_block"}


_FLUX_GUIDANCE_KEYS = {f"guidance_in.{layer}.{leaf}": f"guidance_in.mlp.layers.{idx}.{leaf}"
                       for layer, idx in (("in_layer", 0), ("out_layer", 2)) for leaf in ("weight", "bias")}


def flux_checkpoint_to_params(sd: Dict[str, Tensor], hidden_size: int = 3072, mlp_ratio: int = 4, *,
                              guidance_embed: bool = False, cond_channels: int = 0) -> Dict[str, Tensor]:
    """BFL `flux1-*.safetensors` -> MMDiT parameter tree (reference model_io.py:130-311).

    double_blocks.i.{img,txt}_attn.qkv        -> split 3 (rows)  -> ...{image,text}_transformer_block.attn.{q,k,v}_proj
    double_blocks.i.{img,txt}_attn.proj       -> ...attn.o_proj
    double_blocks.i.{img,txt}_attn.norm.*     -> ...qk_norm.{q,k}_norm.weight
    double_blocks.i.{img,txt}_mlp.{0,2}       -> ...mlp.{fc1,fc2}
    double_blocks.i.{img,txt}_mod.lin         -> ...adaLN_modulation.layers.1
    single_blocks.i.linear1                   -> split rows [h, h, h, r*h] -> attn.{q,k,v}_proj, mlp.fc1
    single_blocks.i.linear2.weight            -> split cols [h, r*h]       -> attn.o_proj.weight, mlp.fc2.weight
    single_blocks.i.linear2.bias              -> attn.o_proj.bias (and mlp.fc2.bias, which the forward zeroes, mmdit.py:742)
    img_in / txt_in / time_in / vector_in / final_layer.adaLN_modulation.1 -> embedders / final layer
    guidance_in.{in,out}_layer                -> guidance_in.mlp.layers.{0,2}  (guidance_embed only)
    The K-projection bias is dropped (quirk Q3).  Without `guidance_embed` guidance_in.* is ignored, as the reference
    does (quirk Q1); with it, FLUX.1-dev's guidance embedder is loaded and must be present.
    `cond_channels` (MMDiTConfig.x_embedder_cond_channels): img_in.weight must have 64 + cond_channels columns, 384 for
    FLUX.1 Fill's `flux1-fill-dev.safetensors` (DESIGN.md §18), 128 for `flux1-canny-dev.safetensors` and
    `flux1-depth-dev.safetensors` (cond_channels 64, DESIGN.md §19); a ValueError names the key otherwise.
    """
    h = hidden_size
    out: Dict[str, Tensor] = {}
    for key, v in sd.items():
        m = re.fullmatch(r"double_blocks\.(\d+)\.(img|txt)_(attn|mlp|mod)\.(.+)", key)
        if m:
            i, stream, part, rest = m.groups()
            base = f"multimodal_transformer_blocks.{i}.{_FLUX_STREAM[stream]}"
            if part == "attn":
                if rest.startswith("qkv."):
                    leaf = rest[4:]
                    for name, chunk in zip("qkv", v.chunk(3, dim=0)):
                        if name == "k" and leaf == "bias":
                            continue
                        out[f"{base}.attn.{name}_proj.{leaf}"] = chunk.contiguous()
                elif rest.startswith("proj."):
                    out[f"{base}.attn.o_proj.{rest[5:]}"] = v
                elif rest == "norm.query_norm.scale":
                    out[f"{base}.qk_norm.q_norm.weight"] = v
                elif rest == "norm.key_norm.scale":
                    out[f"{base}.qk_norm.k_norm.weight"] = v
                else:
                    raise KeyError(f"unrecognised FLUX key {key}")
            elif part == "mlp":
                idx, leaf = rest.split(".", 1)
                out[f"{base}.mlp.{'fc1' if idx == '0' else 'fc2'}.{leaf}"] = v
            else:  # mod.lin.{weight,bias}
                out[f"{base}.adaLN_modulation.layers.1.{rest.split('.', 1)[1]}"] = v
            continue
        m = re.fullmatch(r"single_blocks\.(\d+)\.(.+)", key)
        if m:
            i, rest = m.groups()
            base = f"unified_transformer_blocks.{i}.transformer_block"
            if rest.startswith("linear1."):
                leaf = rest[8:]
                q, k, vv, fc1 = torch.split(v, [h, h, h, mlp_ratio * h], dim=0)
                out[f"{base}.attn.q_proj.{leaf}"] = q.contiguous()
                if leaf != "bias":
                    out[f"{base}.attn.k_proj.{leaf}"] = k.contiguous()
                out[f"{base}.attn.v_proj.{leaf}"] = vv.contiguous()
                out[f"{base}.mlp.fc1.{leaf}"] = fc1.contiguous()
            elif rest == "linear2.weight":
                o, fc2 = torch.split(v, [h, mlp_ratio * h], dim=1)
                out[f"{base}.attn.o_proj.weight"] = o.contiguous()
                out[f"{base}.mlp.fc2.weight"] = fc2.contiguous()
            elif rest == "linear2.bias":
                out[f"{base}.attn.o_proj.bias"] = v
                out[f"{base}.mlp.fc2.bias"] = v
            elif rest.startswith("modulation.lin."):
                out[f"{base}.adaLN_modulation.layers.1.{rest[15:]}"] = v
            elif rest == "norm.query_norm.scale":
                out[f"{base}.qk_norm.q_norm.weight"] = v
            elif rest == "norm.key_norm.scale":
                out[f"{base}.qk_norm.k_norm.weight"] = v
            else:
                raise KeyError(f"unrecognised FLUX key {key}")
            continue
        if key.startswith("img_in."):
            leaf = key[7:]
            if leaf == "weight" and v.shape[1] != 64 + cond_channels:
                kind = {0: "a plain FLUX", 64: "a FLUX.1 Canny / Depth"}.get(cond_channels, "a FLUX.1 Fill")
                raise ValueError(f"{key} has {v.shape[1]} input columns, {kind} config takes {64 + cond_channels} "
                                 f"(x_embedder_cond_channels = {cond_channels})")
            out[f"x_embedder.proj.{leaf}"] = v.reshape(v.shape[0], 1, 1, v.shape[1]).contiguous() if leaf == "weight" else v
        elif key.startswith("txt_in."):
            out["context_embedder." + key[7:]] = v
        elif key.startswith(("time_in.", "vector_in.")):
            emb = "t_embedder" if key.startswith("time_in.") else "y_embedder"
            _, layer, leaf = key.split(".")
            out[f"{emb}.mlp.layers.{0 if layer == 'in_layer' else 2}.{leaf}"] = v
        elif key.startswith("final_layer.adaLN_modulation.1."):
            out["final_layer.adaLN_modulation.layers.1." + key.rsplit(".", 1)[1]] = v
        elif key.startswith("final_layer.linear."):
            out[key] = v
        elif key.startswith("guidance_in."):
            if not guidance_embed:
                continue  # quirk Q1: the reference ignores the guidance embedder (model_io.py:756,783)
            if key not in _FLUX_GUIDANCE_KEYS:
                raise KeyError(f"unrecognised FLUX key {key}")
            out[_FLUX_GUIDANCE_KEYS[key]] = v
        else:
            raise KeyError(f"unrecognised FLUX key {key}")
    if guidance_embed:
        missing = sorted(k for k in _FLUX_GUIDANCE_KEYS if k not in sd)
        if missing:
            raise ValueError(f"the config has a guidance embedder (FLUX.1-dev) but the checkpoint lacks {missing}")
    return out


# ------------------------------------------------------------------------------------------------ SD3 (SAI layout)
def sd3_checkpoint_to_params(sd: Dict[str, Tensor], prefix: str = "model.diffusion_model.", *,
                             k_bias: bool = False) -> Dict[str, Tensor]:
    """Stability `sd3_medium.safetensors` / `sd3.5_*.safetensors` -> MMDiT parameter tree (reference
    model_io.py:314-408).  VAE (`first_stage_model.` / `decoder.` / `encoder.`) and `teacher_model.` tensors are
    skipped here.  SD3.5 Medium's x-block second attention (MMDiT-X) maps as the first one does:
    attn2.qkv -> attn2.{q,k,v}_proj, attn2.proj -> attn2.o_proj, attn2.ln_{q,k} -> qk_norm2.{q,k}_norm.
    The k bias of every qkv is dropped (quirk Q3) unless `k_bias` (MMDiTConfig.attn_k_bias) keeps it."""
    out: Dict[str, Tensor] = {}
    for key, v in sd.items():
        if "decoder." in key or "encoder." in key or "teacher_model." in key:
            continue
        if key.startswith(prefix):
            key = key[len(prefix):]
        m = re.fullmatch(r"joint_blocks\.(\d+)\.(context_block|x_block)\.(.+)", key)
        if m:
            i, blk, rest = m.groups()
            stream = "text_transformer_block" if blk == "context_block" else "image_transformer_block"
            base = f"multimodal_transformer_blocks.{i}.{stream}"
            a = re.fullmatch(r"(attn2?)\.(qkv|proj|ln_q|ln_k)\.(.+)", rest)
            if a:
                attn, part, leaf = a.groups()
                norm = "qk_norm" if attn == "attn" else "qk_norm2"
                if part == "qkv":
                    for name, chunk in zip("qkv", v.chunk(3, dim=0)):
                        if name == "k" and leaf == "bias" and not k_bias:
                            continue                 # model_io.py:389-390
                        out[f"{base}.{attn}.{name}_proj.{leaf}"] = chunk.contiguous()
                elif part == "proj":
                    out[f"{base}.{attn}.o_proj.{leaf}"] = v
                else:
                    out[f"{base}.{norm}.{part[-1]}_norm.{leaf}"] = v
            elif rest.startswith("adaLN_modulation."):
                out[f"{base}.adaLN_modulation.layers.{rest[17:]}"] = v
            else:                                    # mlp.fc1 / mlp.fc2 keep their names
                out[f"{base}.{rest}"] = v
            continue
        if key == "pos_embed":
            out["x_pos_embedder.pos_embed.weight"] = v[0].contiguous()       # (1, N, h) buffer -> (N, h) table
        elif key == "x_embedder.proj.weight":
            out[key] = _conv_oihw_to_ohwi(v)
        elif key.startswith(("y_embedder.mlp.", "t_embedder.mlp.")):
            emb, _, idx, leaf = key.split(".")
            out[f"{emb}.mlp.layers.{idx}.{leaf}"] = v
        elif key.startswith("final_layer.adaLN_modulation."):
            out["final_layer.adaLN_modulation.layers." + key[len("final_layer.adaLN_modulation."):]] = v
        elif key.startswith(("x_embedder.", "context_embedder.", "final_layer.linear.")):
            out[key] = v
        else:
            raise KeyError(f"unrecognised SD3 key {key}")
    return out


# ------------------------------------------------------------------------------------------------ VAE (LDM layout)
def _vae_checkpoint_to_params(sd: Dict[str, Tensor], prefix: str, side: str) -> Dict[str, Tensor]:
    """LDM autoencoder `<prefix>*` -> VAEDecoder / VAEEncoder parameter tree.  side = "up" (decoder: up.N.block.M,
    up.N.upsample.conv) or "down" (encoder: down.N.block.M, down.N.downsample.conv)."""
    blocks, sample = f"{side}_blocks", f"{side}sample"
    out: Dict[str, Tensor] = {}
    for key, v in sd.items():
        pos = key.find(prefix)
        if pos < 0 or "diffusion_model." in key:
            continue
        k = key[pos + len(prefix):]
        leaf = k.rsplit(".", 1)[1]
        m = re.fullmatch(side + r"\.(\d+)\.block\.(\d+)\.(norm1|conv1|norm2|conv2|nin_shortcut)\.(weight|bias)", k)
        if m:
            j, l, mod, _ = m.groups()
            if mod == "nin_shortcut":
                name, val = f"{blocks}.{j}.resnets.{l}.conv_shortcut.{leaf}", (v[:, :, 0, 0].contiguous() if leaf == "weight" else v)
            elif mod.startswith("conv"):
                name, val = f"{blocks}.{j}.resnets.{l}.{mod}.{leaf}", (_conv_oihw_to_ohwi(v) if leaf == "weight" else v)
            else:
                name, val = f"{blocks}.{j}.resnets.{l}.{mod}.{leaf}", v
            out[name] = val
            continue
        m = re.fullmatch(side + r"\.(\d+)\." + sample + r"\.conv\.(weight|bias)", k)
        if m:
            out[f"{blocks}.{m.group(1)}.{sample}.{leaf}"] = _conv_oihw_to_ohwi(v) if leaf == "weight" else v
            continue
        m = re.fullmatch(r"mid\.block_(1|2)\.(norm1|conv1|norm2|conv2)\.(weight|bias)", k)
        if m:
            idx = 0 if m.group(1) == "1" else 2
            mod = m.group(2)
            out[f"mid_blocks.{idx}.{mod}.{leaf}"] = _conv_oihw_to_ohwi(v) if (mod.startswith("conv") and leaf == "weight") else v
            continue
        m = re.fullmatch(r"mid\.attn_1\.(norm|q|k|v|proj_out)\.(weight|bias)", k)
        if m:
            mod = {"norm": "group_norm", "q": "query_proj", "k": "key_proj", "v": "value_proj",
                   "proj_out": "out_proj"}[m.group(1)]
            val = v[:, :, 0, 0].contiguous() if (leaf == "weight" and v.dim() == 4) else v
            out[f"mid_blocks.1.{mod}.{leaf}"] = val
            continue
        if k.startswith(("conv_in.", "conv_out.")):
            out[k] = _conv_oihw_to_ohwi(v) if leaf == "weight" else v
        elif k.startswith("norm_out."):
            out["conv_norm_out." + leaf] = v
        else:
            raise KeyError(f"unrecognised VAE {'decoder' if side == 'up' else 'encoder'} key {key}")
    return out


def vae_decoder_checkpoint_to_params(sd: Dict[str, Tensor], prefix: str = "decoder.") -> Dict[str, Tensor]:
    """LDM autoencoder `decoder.*` -> VAEDecoder parameter tree (reference model_io.py:411-486).
    `prefix` may sit behind another prefix (e.g. `first_stage_model.decoder.`): everything up to and including the first
    occurrence of `prefix` is stripped."""
    return _vae_checkpoint_to_params(sd, prefix, "up")


def vae_encoder_checkpoint_to_params(sd: Dict[str, Tensor], prefix: str = "encoder.") -> Dict[str, Tensor]:
    """LDM autoencoder `encoder.*` -> VAEEncoder parameter tree (reference model_io.py:489-571)."""
    return _vae_checkpoint_to_params(sd, prefix, "down")


# ------------------------------------------------------------------------------------------------ text encoders
def clip_checkpoint_to_params(sd: Dict[str, Tensor]) -> Dict[str, Tensor]:
    """HF CLIPTextModel(WithProjection) safetensors -> CLIPTextModel parameter tree
    (reference map_clip_text_encoder_weights, model_io.py:611-636)."""
    out: Dict[str, Tensor] = {}
    for key, v in sd.items():
        k = key
        for pre in ("text_model.", "embeddings.", "encoder."):
            if k.startswith(pre):
                k = k[len(pre):]
        if k == "position_ids":
            continue                                      # a buffer older checkpoints carry; not a parameter
        k = k.replace("self_attn.", "attention.")
        k = k.replace("q_proj.", "query_proj.").replace("k_proj.", "key_proj.").replace("v_proj.", "value_proj.")
        k = k.replace("mlp.fc1", "linear1").replace("mlp.fc2", "linear2")
        out[k] = v
    return out


def t5_checkpoint_to_params(sd: Dict[str, Tensor], prefix: str = "") -> Dict[str, Tensor]:
    """HF T5EncoderModel (t5xxl.safetensors) -> SD3T5Encoder parameter tree
    (reference t5_encoder_state_dict_adjustments, model_io.py:565-608)."""
    out: Dict[str, Tensor] = {}
    attn = {"q": "query_proj", "k": "key_proj", "v": "value_proj", "o": "out_proj"}
    for key, v in sd.items():
        k = key[len(prefix):] if prefix and key.startswith(prefix) else key
        if k in ("shared.weight",):
            continue                                      # same tensor as encoder.embed_tokens.weight (:601-603)
        if k == "encoder.embed_tokens.weight":
            out["wte.weight"] = v
        elif k == "encoder.final_layer_norm.weight":
            out["encoder.ln.weight"] = v
        elif k == "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight":
            out["encoder.relative_attention_bias.embeddings.weight"] = v
        else:
            m = re.fullmatch(r"encoder\.block\.(\d+)\.layer\.(0|1)\.(.+)", k)
            if not m:
                raise KeyError(f"unrecognised T5 key {key}")
            i, sub, rest = m.groups()
            base = f"encoder.layers.{i}."
            if rest == "layer_norm.weight":
                out[base + f"ln{int(sub) + 1}.weight"] = v
            elif rest.startswith("SelfAttention."):
                out[base + f"attention.{attn[rest.split('.')[1]]}.weight"] = v
            elif rest.startswith("DenseReluDense."):
                out[base + "dense." + rest[len("DenseReluDense."):]] = v
            else:
                raise KeyError(f"unrecognised T5 key {key}")
    if "wte.weight" not in out and "shared.weight" in sd:
        out["wte.weight"] = sd["shared.weight"]
    return out


# ------------------------------------------------------------------------------------------------ 4-bit variants
def is_q4_checkpoint(sd: Dict[str, Tensor]) -> bool:
    return any(k.endswith(".scales") for k in sd)


def preadjusted_checkpoint_to_params(sd: Dict[str, Tensor], prefix: str = "") -> Dict[str, Tensor]:
    """The `*-4bit-quantized` checkpoints were saved from the reference's own module tree, so their keys already are
    the App. C names (behind `prefix` for the single-file SD3.5 checkpoint): keep the keys that contain the prefix and
    strip it (reference model_io.py:733-734, 772-775 "4-bit ckpt already adjusted")."""
    if not prefix:
        return dict(sd)
    return {k.replace(prefix, ""): v for k, v in sd.items() if prefix in k}


def dequantize_q4_params(sd: Dict[str, Tensor], device, dtype: torch.dtype, group_size: int = 64) -> Dict[str, Tensor]:
    """MLX QuantizedLinear triples (`X.weight` uint32 [N, K/8], `X.scales`, `X.biases` [N, K/64]) -> dense 16-bit
    `X.weight` [N, K] on `device` (dk_dequant_q4).  The denoise GEMMs are tensor-pipe bound at M >= 1024 rows and the dense
    FLUX weights (23.8 GB) fit HBM, so the 4-bit form is expanded once at load instead of inside every GEMM.  Every other tensor is passed through (cast to `dtype` like the reference, :736-738)."""
    from . import ops

    out: Dict[str, Tensor] = {}
    for k, v in sd.items():
        if k.endswith((".scales", ".biases")) and (k.rsplit(".", 1)[0] + ".weight") in sd:
            continue
        base = k[:-7] if k.endswith(".weight") else None
        if base is not None and (base + ".scales") in sd:
            if v.dtype not in (torch.uint32, torch.int32):
                raise ValueError(f"{k}: quantised weight must be uint32, got {v.dtype}")
            wq = v.contiguous().view(torch.int32).to(device)
            sc = sd[base + ".scales"].to(device=device, dtype=dtype).contiguous()
            bi = sd[base + ".biases"].to(device=device, dtype=dtype).contiguous()
            out[k] = ops.dequant_q4(wq, sc, bi, group_size)
        else:
            out[k] = v.to(device=device, dtype=dtype) if v.is_floating_point() else v.to(device)
    return out


def check_against_specs(params: Dict[str, Tensor], specs: Iterable[Tuple[str, Tuple[int, ...], str]],
                        allow_extra: Iterable[str] = ()) -> None:
    """Raise if the converted tree does not match the engine's parameter specs (names and shapes)."""
    want = {n: tuple(s) for n, s, _ in specs}
    missing = sorted(set(want) - set(params))
    extra = sorted(k for k in set(params) - set(want) if not any(k.endswith(a) for a in allow_extra))
    bad = sorted(n for n in want if n in params and tuple(params[n].shape) != want[n])
    if missing or extra or bad:
        raise ValueError(f"checkpoint does not match the model: missing {missing[:5]} (+{max(0, len(missing) - 5)}), "
                         f"unexpected {extra[:5]} (+{max(0, len(extra) - 5)}), wrong shape {bad[:5]}")


# ------------------------------------------------------------------------------------------------ FLUX.1 Redux
_SIGLIP_DROPPED = ("text_model.", "logit_scale", "logit_bias", "vision_model.head.", "head.")


def siglip_checkpoint_to_params(sd: Dict[str, Tensor], config=None) -> Dict[str, Tensor]:
    """Hugging Face SigLIP safetensors -> the engine's SiglipVisionModel tree (image_encoders.pack_siglip_params).
    Takes the full SiglipModel file (`vision_model.*` beside `text_model.*`, `logit_scale`, `logit_bias`) or a
    vision-only export (with or without the `vision_model.` prefix).  The text tower, the logit scalars and the pooling
    head (`vision_model.head.*`, not part of last_hidden_state) are dropped; the `position_ids` buffer older exports carry
    is skipped.  A missing key, an unexpected one or a wrong shape raises ValueError naming it.  config: a
    SiglipVisionConfig (default google/siglip-so400m-patch14-384)."""
    from .config import SIGLIP_SO400M_PATCH14_384
    from .image_encoders import pack_siglip_params, siglip_param_specs

    cfg = config if config is not None else SIGLIP_SO400M_PATCH14_384
    out: Dict[str, Tensor] = {}
    for key, v in sd.items():
        if key.startswith(_SIGLIP_DROPPED) or key.endswith("position_ids"):
            continue
        out[key[len("vision_model."):] if key.startswith("vision_model.") else key] = v
    want = {n: tuple(s) for n, s, _ in siglip_param_specs(cfg)}
    for n, s in want.items():
        if n not in out:
            raise ValueError(f"SigLIP checkpoint: missing vision_model.{n}")
        if tuple(out[n].shape) != s:
            raise ValueError(f"SigLIP checkpoint: vision_model.{n} has shape {tuple(out[n].shape)}, expected {s}")
    extra = sorted(set(out) - set(want))
    if extra:
        raise ValueError(f"SigLIP checkpoint: unexpected keys {extra[:5]} (+{max(0, len(extra) - 5)})")
    return pack_siglip_params(out, cfg)


def redux_checkpoint_to_params(sd: Dict[str, Tensor], token_level_text_embed_dim: int = 4096,
                               siglip_hidden: int = 1152) -> Dict[str, Tensor]:
    """BFL `flux1-redux-dev.safetensors` (redux_up / redux_down .weight / .bias) -> ReduxImageEncoder's tree, the same
    names.  Shapes are checked against the FLUX config's token_level_text_embed_dim and the SigLIP width; a missing,
    unexpected or misshaped key raises ValueError naming it."""
    from .image_encoders import redux_param_specs

    want = {n: tuple(s) for n, s, _ in redux_param_specs(siglip_hidden, token_level_text_embed_dim)}
    for n, s in want.items():
        if n not in sd:
            raise ValueError(f"Redux checkpoint: missing {n}")
        if tuple(sd[n].shape) != s:
            raise ValueError(f"Redux checkpoint: {n} has shape {tuple(sd[n].shape)}, expected {s}")
    extra = sorted(set(sd) - set(want))
    if extra:
        raise ValueError(f"Redux checkpoint: unexpected keys {extra}")
    return {n: sd[n] for n in want}


# ------------------------------------------------------------------------------------------------ FLUX.1 Depth
def depth_anything_config(config_json: dict):
    """a transformers DepthAnything `config.json` (as a dict) -> DepthAnythingConfig.  The backbone's MLP width is
    hidden_size * mlp_ratio (Dinov2Config); its stages come from out_indices, or from out_features ("stageN")."""
    from .config import DepthAnythingConfig

    bb = config_json.get("backbone_config") or {}
    D = int(bb.get("hidden_size", 1024))
    if "out_indices" in bb and bb["out_indices"] is not None:
        out_indices = tuple(int(i) for i in bb["out_indices"])
    elif bb.get("out_features"):
        out_indices = tuple(int(str(f).replace("stage", "")) for f in bb["out_features"])
    else:
        out_indices = DepthAnythingConfig.out_indices
    rh = config_json.get("reassemble_hidden_size", D)
    if rh != D:
        raise ValueError(f"Depth Anything config: reassemble_hidden_size {rh} differs from the backbone width {D}")
    return DepthAnythingConfig(
        hidden_size=D, num_attention_heads=int(bb.get("num_attention_heads", 16)),
        intermediate_size=int(D * bb.get("mlp_ratio", 4)), num_hidden_layers=int(bb.get("num_hidden_layers", 24)),
        patch_size=int(bb.get("patch_size", 14)), image_size=int(bb.get("image_size", 518)),
        layer_norm_eps=float(bb.get("layer_norm_eps", 1e-6)), hidden_act=bb.get("hidden_act", "gelu"),
        out_indices=out_indices,
        neck_hidden_sizes=tuple(int(c) for c in config_json.get("neck_hidden_sizes", (256, 512, 1024, 1024))),
        reassemble_factors=tuple(config_json.get("reassemble_factors", (4, 2, 1, 0.5))),
        fusion_hidden_size=int(config_json.get("fusion_hidden_size", 256)),
        head_hidden_size=int(config_json.get("head_hidden_size", 32)),
        depth_estimation_type=config_json.get("depth_estimation_type", "relative"))


_DEPTH_DROPPED = ("backbone.embeddings.mask_token", "neck.fusion_stage.layers.0.residual_layer1.")


def depth_anything_checkpoint_to_params(sd: Dict[str, Tensor], config=None) -> Dict[str, Tensor]:
    """transformers DepthAnythingForDepthEstimation safetensors (`backbone.*`, `neck.*`, `head.*`) -> the engine's
    DepthAnythingModel tree (depth.pack_depth_params, fp32).  backbone.embeddings.mask_token and the unused
    neck.fusion_stage.layers.0.residual_layer1.* are dropped.  A missing key, an unexpected one or a wrong shape raises
    ValueError naming it, as does a configuration the kernels cannot run.  config: a DepthAnythingConfig (default
    LiheYoung/depth-anything-large-hf)."""
    from .config import DEPTH_ANYTHING_LARGE
    from .depth import check_config, depth_param_specs, pack_depth_params

    cfg = config if config is not None else DEPTH_ANYTHING_LARGE
    check_config(cfg)
    out = {k: v for k, v in sd.items() if not k.startswith(_DEPTH_DROPPED)}
    want = {n: tuple(s) for n, s, _ in depth_param_specs(cfg)}
    for n, s in want.items():
        if n not in out:
            raise ValueError(f"Depth Anything checkpoint: missing {n}")
        if tuple(out[n].shape) != s:
            raise ValueError(f"Depth Anything checkpoint: {n} has shape {tuple(out[n].shape)}, expected {s}")
    extra = sorted(set(out) - set(want))
    if extra:
        raise ValueError(f"Depth Anything checkpoint: unexpected keys {extra[:5]} (+{max(0, len(extra) - 5)})")
    return pack_depth_params(out, cfg)
