"""FLUX.1 Redux image prompts (DESIGN.md §15): the SigLIP vision encoder (transformers' SiglipVisionModel,
`last_hidden_state`) and BFL's Redux projector, on the engine's kernels.

SigLIP: the 14 x 14 stride-14 patch convolution is dk_image_patches + one wgmma GEMM (bias in the epilogue, the position
table added as a residual broadcast over the batch); 27 pre-LN layers of LayerNorm, packed QKV GEMM, dk_attention_fwd,
o-proj GEMM with an in-place residual, LayerNorm, fc1 with tanh-GELU, fc2 with residual; then post_layernorm.  The
pooling head is not part of `last_hidden_state` and is neither loaded nor computed.

SigLIP's head dim is 72 and dk_attention_fwd takes 64 or 128, so at load every head of the packed [q | k | v] weight and
bias gets zero rows up to 128, and the out_proj weight zero columns to match.  Zero q / k columns add nothing to a score;
zero v columns give output columns that the zero out_proj columns ignore: the padding is exact.  The softmax scale stays
72^-0.5.

Parameter trees.  `siglip_param_specs` / `redux_param_specs` describe the upstream layouts (transformers'
`vision_model.*` names without that prefix; BFL's `redux_{up,down}`), which the synthetic initialiser and the checkpoint
loaders (model_io.siglip_checkpoint_to_params / redux_checkpoint_to_params) start from.  `pack_siglip_params` turns the
SigLIP tree into the engine's: the patch weight permuted OIHW -> (O, kh, kw, c) and zero-padded to a multiple of 8
columns (patch_weight_kp), q / k / v packed as `self_attn.qkv_proj` with padded heads, out_proj padded.  SiglipVisionModel
takes the engine's tree.
"""
from __future__ import annotations

from typing import Dict, List

import torch

from . import ops
from ._lib import ACT_GELU_TANH, ACT_SILU, dtype_code, ptr
from .config import SiglipVisionConfig
from .text_encoders import _device_params

Spec = tuple


def patch_weight_kp(cfg: SiglipVisionConfig) -> int:
    """columns of a patch row: 3 p^2 rounded up to a multiple of 8 (the GEMM's K % 8 == 0): 588 -> 592"""
    return -(-3 * cfg.patch_size ** 2 // 8) * 8


def padded_head_dim(cfg: SiglipVisionConfig) -> int:
    """the head dim dk_attention_fwd runs SigLIP's heads at: 72 -> 128, 64 stays"""
    d = cfg.head_dim
    if cfg.hidden_size != cfg.num_attention_heads * d or d not in (64, 72):
        raise ValueError(f"SigLIP: hidden size {cfg.hidden_size} must be heads ({cfg.num_attention_heads}) x a head dim "
                         "of 72 (so400m) or 64")
    return 128 if d == 72 else 64


def siglip_param_specs(cfg: SiglipVisionConfig) -> List[Spec]:
    """transformers' SiglipVisionTransformer tree without the pooling head (`head.*`), names without `vision_model.`"""
    D, F, p = cfg.hidden_size, cfg.intermediate_size, cfg.patch_size
    specs: List[Spec] = [("embeddings.patch_embedding.weight", (D, 3, p, p), "w"),
                         ("embeddings.patch_embedding.bias", (D,), "b"),
                         ("embeddings.position_embedding.weight", (cfg.num_patches, D), "e")]

    def lin(name, cout, cin):
        specs.append((name + ".weight", (cout, cin), "w"))
        specs.append((name + ".bias", (cout,), "b"))

    def ln(name):
        specs.append((name + ".weight", (D,), "g"))
        specs.append((name + ".bias", (D,), "b"))

    for i in range(cfg.num_hidden_layers):
        l = f"encoder.layers.{i}."
        ln(l + "layer_norm1")
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            lin(l + "self_attn." + n, D, D)
        ln(l + "layer_norm2")
        lin(l + "mlp.fc1", F, D)
        lin(l + "mlp.fc2", D, F)
    ln("post_layernorm")
    return specs


def redux_param_specs(siglip_hidden: int = 1152, txt_dim: int = 4096) -> List[Spec]:
    """BFL's ReduxImageEncoder: redux_up (siglip_hidden -> 3 txt_dim), redux_down (3 txt_dim -> txt_dim)"""
    return [("redux_up.weight", (3 * txt_dim, siglip_hidden), "w"), ("redux_up.bias", (3 * txt_dim,), "b"),
            ("redux_down.weight", (txt_dim, 3 * txt_dim), "w"), ("redux_down.bias", (txt_dim,), "b")]


def _pad_heads(t: torch.Tensor, heads: int, d: int, dp: int, dim: int) -> torch.Tensor:
    """t with each of its `heads` blocks of d rows (dim 0) or columns (dim 1) zero-padded to dp"""
    if dim == 0:
        blocks = t.reshape(heads, d, *t.shape[1:])
        return torch.cat([blocks, blocks.new_zeros((heads, dp - d, *t.shape[1:]))], 1).reshape(heads * dp, *t.shape[1:])
    blocks = t.reshape(t.shape[0], heads, d)
    return torch.cat([blocks, blocks.new_zeros((t.shape[0], heads, dp - d))], 2).reshape(t.shape[0], heads * dp)


def pack_siglip_params(params: Dict[str, torch.Tensor], cfg: SiglipVisionConfig) -> Dict[str, torch.Tensor]:
    """upstream-layout SigLIP tree (siglip_param_specs) -> the engine's: patch weight (D, kp) in (kh, kw, c) column
    order with zero columns 3p^2..kp, `self_attn.qkv_proj` [q | k | v] (3 heads dp, D) with each head's rows zero-padded
    from d to dp, out_proj (D, heads dp) with zero columns to match; every other tensor as it is"""
    H, d, dp = cfg.num_attention_heads, cfg.head_dim, padded_head_dim(cfg)
    out: Dict[str, torch.Tensor] = {}
    for k, v in params.items():
        if k == "embeddings.patch_embedding.weight":
            w = v.permute(0, 2, 3, 1).reshape(v.shape[0], -1)
            out[k] = torch.cat([w, w.new_zeros((w.shape[0], patch_weight_kp(cfg) - w.shape[1]))], 1).contiguous()
        elif ".self_attn.q_proj." in k:
            base, leaf = k.split(".q_proj.")
            out[f"{base}.qkv_proj.{leaf}"] = torch.cat(
                [_pad_heads(params[f"{base}.{n}_proj.{leaf}"], H, d, dp, 0) for n in "qkv"]).contiguous()
        elif ".self_attn.k_proj." in k or ".self_attn.v_proj." in k:
            continue
        elif k.endswith(".self_attn.out_proj.weight"):
            out[k] = _pad_heads(v, H, d, dp, 1).contiguous()
        else:
            out[k] = v
    return out


def engine_siglip_shapes(cfg: SiglipVisionConfig) -> Dict[str, tuple]:
    """names and shapes of the engine's SigLIP tree (pack_siglip_params of siglip_param_specs)"""
    dp = padded_head_dim(cfg)
    D, H = cfg.hidden_size, cfg.num_attention_heads
    shapes = {n: tuple(s) for n, s, _ in siglip_param_specs(cfg) if ".k_proj." not in n and ".v_proj." not in n}
    shapes["embeddings.patch_embedding.weight"] = (D, patch_weight_kp(cfg))
    for i in range(cfg.num_hidden_layers):
        a = f"encoder.layers.{i}.self_attn."
        del shapes[a + "q_proj.weight"], shapes[a + "q_proj.bias"]
        shapes[a + "qkv_proj.weight"], shapes[a + "qkv_proj.bias"] = (3 * H * dp, D), (3 * H * dp,)
        shapes[a + "out_proj.weight"] = (D, H * dp)
    return shapes


def init_siglip_params(cfg: SiglipVisionConfig, seed: int = 0, dtype: torch.dtype = torch.bfloat16,
                       device="cpu") -> Dict[str, torch.Tensor]:
    """deterministic synthetic SigLIP weights (weights.init_params of siglip_param_specs) in the engine's layout"""
    from .weights import init_params

    return pack_siglip_params(init_params(siglip_param_specs(cfg), seed=seed, dtype=dtype, device=device), cfg)


def image_patches(img_u8, dtype, p: int, kp: int, out=None):
    """dk_image_patches: uint8 NHWC [B, H, W, >=3] -> 16-bit patch rows [B * (H // p) * (W // p), kp] of a stride-p
    p x p convolution, columns (kh, kw, c) normalised like ops.image_pre, columns 3p^2.. zero (the last H % p rows and
    W % p columns dropped).  Kept beside its one caller rather than in ops: the launch census of the shipped models
    requires a reference for every launching op there, and this one runs only under an image prompt, whose GPU test
    runs a census of its own that wraps it."""
    assert img_u8.dtype == torch.uint8 and img_u8.is_contiguous() and img_u8.dim() == 4 and img_u8.is_cuda
    B, H, W, Cs = img_u8.shape
    rows = B * (H // p) * (W // p)
    if out is None:
        out = torch.empty((rows, kp), dtype=dtype, device=img_u8.device)
    assert out.dtype == dtype and out.is_contiguous() and tuple(out.shape) == (rows, kp)
    c = ops.ctx(img_u8.device.index)
    c.call("dk_image_patches", dtype_code(dtype), ptr(img_u8), ptr(out), B, H, W, Cs, p, kp)
    return out


def _check_shapes(params, want: Dict[str, tuple], who: str):
    missing = sorted(set(want) - set(params))
    bad = sorted(k for k in want if k in params and tuple(params[k].shape) != want[k])
    if missing or bad:
        raise ValueError(f"{who}: missing {missing[:5]}, wrong shape "
                         f"{[(k, tuple(params[k].shape), want[k]) for k in bad[:5]]}")


class SiglipVisionModel:
    """SigLIP's vision transformer -> last_hidden_state (transformers SiglipVisionModel), on the device.
    params: the engine's tree (pack_siglip_params), 16-bit."""

    def __init__(self, params: Dict[str, torch.Tensor], config: SiglipVisionConfig, device=None):
        if config.hidden_act != "gelu_pytorch_tanh":
            raise ValueError(f"SigLIP: only the gelu_pytorch_tanh activation is implemented, got {config.hidden_act}")
        self.dp = padded_head_dim(config)
        _check_shapes(params, engine_siglip_shapes(config), "SiglipVisionModel")
        self.device, self.dtype, self.p = _device_params(params, device, "SiglipVisionModel")
        self.config = config
        self.kp = patch_weight_kp(config)

    def __call__(self, images: torch.Tensor) -> torch.Tensor:
        """images: uint8 (n, S, S, >=3) on the device, S = config.image_size -> (n, tokens, hidden) in the weight
        dtype"""
        c, p = self.config, self.p
        n, Hs, Ws = images.shape[:3]
        if (Hs, Ws) != (c.image_size, c.image_size):
            raise ValueError(f"SigLIP takes {c.image_size}x{c.image_size} images, got {Hs}x{Ws}")
        P, D, H = c.num_patches, c.hidden_size, c.num_attention_heads
        x = image_patches(images, self.dtype, c.patch_size, self.kp)
        h = ops.gemm(x, p["embeddings.patch_embedding.weight"], bias=p["embeddings.patch_embedding.bias"],
                     res=p["embeddings.position_embedding.weight"], rows_per_batch=P, out_batch_rows=P,
                     res_batch_rows=0)
        att = torch.empty((n * P, H * self.dp), dtype=self.dtype, device=self.device)
        scale = c.head_dim ** -0.5                      # the real head dim, not the padded one
        eps = c.layer_norm_eps
        for i in range(c.num_hidden_layers):
            l = f"encoder.layers.{i}."
            y = ops.layernorm(h, p[l + "layer_norm1.weight"], p[l + "layer_norm1.bias"], eps)
            qkv = ops.gemm(y, p[l + "self_attn.qkv_proj.weight"], bias=p[l + "self_attn.qkv_proj.bias"])
            ops.attention(qkv, n, P, H, self.dp, att, scale=scale)
            ops.gemm(att, p[l + "self_attn.out_proj.weight"], bias=p[l + "self_attn.out_proj.bias"], res=h, out=h)
            y = ops.layernorm(h, p[l + "layer_norm2.weight"], p[l + "layer_norm2.bias"], eps)
            y = ops.gemm(y, p[l + "mlp.fc1.weight"], bias=p[l + "mlp.fc1.bias"], act=ACT_GELU_TANH)
            ops.gemm(y, p[l + "mlp.fc2.weight"], bias=p[l + "mlp.fc2.bias"], res=h, out=h)
        return ops.layernorm(h, p["post_layernorm.weight"], p["post_layernorm.bias"], eps).reshape(n, P, D)


class ReduxImageEncoder:
    """BFL's Redux projector: redux_down(silu(redux_up(x))), siglip_hidden -> 3 txt_dim -> txt_dim."""

    def __init__(self, params: Dict[str, torch.Tensor], device=None):
        if set(params) != {n for n, _, _ in redux_param_specs()}:
            raise ValueError(f"ReduxImageEncoder: expected redux_{{up,down}}.{{weight,bias}}, got {sorted(params)}")
        self.device, self.dtype, self.p = _device_params(params, device, "ReduxImageEncoder")
        self.txt_dim = self.p["redux_down.weight"].shape[0]
        self.siglip_hidden = self.p["redux_up.weight"].shape[1]
        _check_shapes(self.p, {n: s for n, s, _ in redux_param_specs(self.siglip_hidden, self.txt_dim)},
                      "ReduxImageEncoder")

    def __call__(self, x: torch.Tensor, tokens: int, out=None, out_seq_rows: int = 0, out_row_off: int = 0):
        """x: [n * tokens, siglip_hidden] -> [n * tokens, txt_dim]; with `out` (a 2-D view of a [.., txt_dim] buffer)
        the tokens of image i go to rows i * out_seq_rows + out_row_off + [0, tokens) of it (the GEMM's row map)"""
        p = self.p
        u = ops.gemm(x, p["redux_up.weight"], bias=p["redux_up.bias"], act=ACT_SILU)
        if out is None:
            return ops.gemm(u, p["redux_down.weight"], bias=p["redux_down.bias"])
        return ops.gemm(u, p["redux_down.weight"], bias=p["redux_down.bias"], out=out, rows_per_batch=tokens,
                        out_batch_rows=out_seq_rows, out_row_off=out_row_off)
