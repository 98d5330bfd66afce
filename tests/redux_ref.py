"""CPU fp32 oracle of FLUX.1 Redux image prompts (DESIGN.md §15): SigLIP's vision transformer (last_hidden_state) on
the engine's parameter tree, BFL's Redux projector, and the oracle pipeline on the concatenated conditioning.  Kept
beside the tests, like tests/kontext_ref.py, so no file under oracle/ changes.  tests/test_redux_cpu.py pins it against
transformers' SiglipVisionModel and a transcription of BFL's ReduxImageEncoder.

The oracle runs on the packed tree as the engine does (patch weight in (kh, kw, c) order padded to kp columns, q / k / v
heads zero-padded from 72 to 128, out_proj columns to match): the zero rows and columns contribute exact zeros in fp32,
so what it checks against transformers is the loader's permutation and padding together with the forward.
"""
from __future__ import annotations

from typing import Dict, Sequence

import torch
import torch.nn.functional as F

from diffusionkit_b200._lib import ACT_GELU_TANH
from diffusionkit_b200.config import SiglipVisionConfig
from diffusionkit_b200.image_encoders import padded_head_dim, patch_weight_kp


def gelu_tanh(x: torch.Tensor) -> torch.Tensor:
    """0.5 x (1 + tanh(sqrt(2 / pi) (x + 0.044715 x^3))), transformers' gelu_pytorch_tanh written out"""
    return 0.5 * x * (1.0 + torch.tanh(0.7978845608028654 * (x + 0.044715 * x.pow(3))))


# ------------------------------------------------------------------------------------------------ per-launch references
def ref_image_patches(img_u8, dtype, p, kp):
    """uint8 NHWC -> patch rows [B * (H // p) * (W // p), kp] of a stride-p p x p convolution in `dtype`: (kh, kw, c)
    columns of u8 / 255 * 2 - 1 (on the CPU, like tests/kernel_checks.ref_image_pre: torch's CUDA division by a scalar
    multiplies by the reciprocal, the kernel divides), columns 3p^2.. zero, the last H % p rows and W % p columns
    dropped"""
    B, H, W, _ = img_u8.shape
    hp, wp = H // p, W // p
    x = img_u8.cpu()[:, :hp * p, :wp * p, :3].float() / 255 * 2 - 1.0
    x = x.reshape(B, hp, p, wp, p, 3).permute(0, 1, 3, 2, 4, 5).reshape(B * hp * wp, 3 * p * p)
    return F.pad(x, (0, kp - 3 * p * p)).to(dtype).to(img_u8.device)


def with_gelu_tanh(ref_gemm):
    """tests/kernel_checks.ref_gemm extended by DK_ACT_GELU_TANH, the activation SigLIP's fc1 uses (no gate, no
    residual there); every other call goes to ref_gemm unchanged"""
    def ref(A, W, bias=None, act=0, gate=None, res=None, **kw):
        if act != ACT_GELU_TANH:
            return ref_gemm(A, W, bias, act, gate, res, **kw)
        assert gate is None and res is None, "the tanh-GELU reference covers bias + activation"
        return F.gelu(ref_gemm(A, W, bias, 0, **kw), approximate="tanh")
    return ref


def ref_attention(qkv, B, S, heads, d, scale):
    """softmax(scale q k^T) v in fp32 for a packed [B * S, 3 * heads * d] qkv -> [B * S, heads * d], one head at a
    time; SigLIP's padded heads run at d = 128 with scale 72^-0.5"""
    x = qkv.reshape(B, S, 3, heads, d)
    ref = torch.empty((B, S, heads * d), dtype=torch.float32, device=qkv.device)
    for b in range(B):
        for hd in range(heads):
            q, k, v = x[b, :, 0, hd].float(), x[b, :, 1, hd].float(), x[b, :, 2, hd].float()
            ref[b, :, hd * d:(hd + 1) * d] = torch.softmax(q @ k.t() * scale, dim=-1) @ v
    return ref.reshape(B * S, heads * d)


class SiglipVisionRef:
    """fp32 SigLIP vision transformer -> last_hidden_state (n, tokens, hidden), from the engine's packed tree"""

    def __init__(self, params: Dict[str, torch.Tensor], cfg: SiglipVisionConfig):
        self.p = {k: v.float().cpu() for k, v in params.items()}
        self.cfg = cfg

    def __call__(self, images_u8: torch.Tensor) -> torch.Tensor:
        c, p = self.cfg, self.p
        n = images_u8.shape[0]
        P, D, H, dp = c.num_patches, c.hidden_size, c.num_attention_heads, padded_head_dim(c)
        x = ref_image_patches(images_u8.cpu(), torch.float32, c.patch_size, patch_weight_kp(c))
        h = x @ p["embeddings.patch_embedding.weight"].t() + p["embeddings.patch_embedding.bias"]
        h = (h.reshape(n, P, D) + p["embeddings.position_embedding.weight"]).reshape(n * P, D)
        eps = c.layer_norm_eps

        def ln(t, name):
            return F.layer_norm(t, (D,), p[name + ".weight"], p[name + ".bias"], eps)

        for i in range(c.num_hidden_layers):
            l = f"encoder.layers.{i}."
            qkv = ln(h, l + "layer_norm1") @ p[l + "self_attn.qkv_proj.weight"].t() + p[l + "self_attn.qkv_proj.bias"]
            q, k, v = (t.reshape(n, P, H, dp).transpose(1, 2) for t in qkv.split(H * dp, dim=1))
            s = torch.softmax((q @ k.transpose(-1, -2)) * c.head_dim ** -0.5, dim=-1)
            att = (s @ v).transpose(1, 2).reshape(n * P, H * dp)
            h = h + att @ p[l + "self_attn.out_proj.weight"].t() + p[l + "self_attn.out_proj.bias"]
            y = gelu_tanh(ln(h, l + "layer_norm2") @ p[l + "mlp.fc1.weight"].t() + p[l + "mlp.fc1.bias"])
            h = h + y @ p[l + "mlp.fc2.weight"].t() + p[l + "mlp.fc2.bias"]
        return ln(h, "post_layernorm").reshape(n, P, D)


def redux_project(params: Dict[str, torch.Tensor], x: torch.Tensor) -> torch.Tensor:
    """redux_down(silu(redux_up(x))) in fp32"""
    p = {k: v.float().cpu() for k, v in params.items()}
    u = F.silu(x.float() @ p["redux_up.weight"].t() + p["redux_up.bias"])
    return u @ p["redux_down.weight"].t() + p["redux_down.bias"]


def redux_tokens(siglip_params, redux_params, cfg: SiglipVisionConfig, images_u8: torch.Tensor) -> torch.Tensor:
    """uint8 (n, S, S, 3) -> fp32 Redux tokens (n, tokens, txt_dim)"""
    return redux_project(redux_params, SiglipVisionRef(siglip_params, cfg)(images_u8))


def redux_pipeline_latents(mmdit_ref, sample, sigmas, x0s, cond, pooled, tokens: Sequence[torch.Tensor], guidance,
                           act_dtype) -> torch.Tensor:
    """The oracle pipeline on the concatenated conditioning: image i denoises with cat(cond[i], tokens[i]) (its T5 rows,
    then its (tokens, txt_dim) image tokens, rounded to the activation dtype as the engine's conditioning is), through
    tests/kontext_ref.kontext_pipeline_latents without a reference.  No CFG (Redux runs without it)."""
    from tests.kontext_ref import kontext_pipeline_latents

    n = len(x0s)
    cat = torch.stack([torch.cat([cond[i].float(), tokens[i].to(act_dtype).float()]) for i in range(n)])
    return kontext_pipeline_latents(mmdit_ref, sample, sigmas, x0s, cat, pooled, [None] * n, guidance, 0.0, act_dtype)
