"""Text encoders on H100 (SURVEY.md §8 row f2) — host-side mirrors of the reference CLIPTextModel
(python/src/diffusionkit/mlx/clip.py:27-120) and SD3T5Encoder (mlx/t5.py:198-243, 316-325).

Same parameter names as the reference module trees.  Kernels: every projection / MLP on the wgmma GEMM (packed QKV,
bias / quick-GELU / GELU / residual fused in the epilogue); embedding lookup, LayerNorm, T5 RMSNorm over the fp32
residual stream, gated-GELU product and the short-sequence attention (causal mask or relative-position bias) in
csrc/text.cu.

Deliberate differences (DESIGN.md §7): T5's feed-forward runs with 16-bit GEMM inputs and fp32 accumulation (the
reference's type promotion makes it fp32 x 16-bit weights, t5.py:214-224); the residual stream itself stays fp32 like
the reference's.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional

import numpy as np
import torch

from . import ops
from ._lib import ACT_GELU_ERF, ACT_QUICK_GELU, DkError
from .config import CLIPTextModelConfig, T5EncoderConfig

Spec = tuple


def clip_param_specs(cfg: CLIPTextModelConfig) -> List[Spec]:
    d = cfg.model_dims
    specs: List[Spec] = [("token_embedding.weight", (cfg.vocab_size, d), "e"),
                         ("position_embedding.weight", (cfg.max_length, d), "e")]

    def lin(name, cout, cin, bias=True):
        specs.append((name + ".weight", (cout, cin), "w"))
        if bias:
            specs.append((name + ".bias", (cout,), "b"))

    def ln(name):
        specs.append((name + ".weight", (d,), "g"))
        specs.append((name + ".bias", (d,), "b"))

    for i in range(cfg.num_layers):
        p = f"layers.{i}"
        ln(p + ".layer_norm1")
        ln(p + ".layer_norm2")
        for n in ("query_proj", "key_proj", "value_proj", "out_proj"):
            lin(f"{p}.attention.{n}", d, d)
        lin(p + ".linear1", 4 * d, d)
        lin(p + ".linear2", d, 4 * d)
    ln("final_layer_norm")
    if cfg.projection_dim is not None:
        lin("text_projection", cfg.projection_dim, d, bias=False)
    return specs


def t5_param_specs(cfg: T5EncoderConfig) -> List[Spec]:
    d, inner = cfg.d_model, cfg.d_kv * cfg.num_heads
    specs: List[Spec] = [("wte.weight", (cfg.vocab_size, d), "e")]
    for i in range(cfg.num_layers):
        p = f"encoder.layers.{i}"
        for n in ("query_proj", "key_proj", "value_proj"):
            specs.append((f"{p}.attention.{n}.weight", (inner, d), "w"))
        specs.append((f"{p}.attention.out_proj.weight", (d, inner), "w"))
        specs.append((p + ".ln1.weight", (d,), "g"))
        specs.append((p + ".ln2.weight", (d,), "g"))
        specs.append((p + ".dense.wi_0.weight", (cfg.d_ff, d), "w"))
        specs.append((p + ".dense.wi_1.weight", (cfg.d_ff, d), "w"))
        specs.append((p + ".dense.wo.weight", (d, cfg.d_ff), "w"))
    specs.append(("encoder.ln.weight", (d,), "g"))
    specs.append(("encoder.relative_attention_bias.embeddings.weight",
                  (cfg.relative_attention_num_buckets, cfg.num_heads), "e"))
    return specs


@dataclass
class CLIPOutput:
    """reference mlx/clip.py:14-24"""

    pooled_output: Optional[torch.Tensor] = None
    last_hidden_state: Optional[torch.Tensor] = None
    hidden_states: Optional[List[torch.Tensor]] = None


def _device_params(params, device, who):
    any_p = next(iter(params.values()))
    dev = torch.device(device) if device is not None else any_p.device
    if dev.type != "cuda":
        raise DkError(f"{who}: parameters must live on a CUDA device (no CPU fallback)")
    dt = any_p.dtype
    if dt not in (torch.bfloat16, torch.float16):
        raise DkError(f"{who}: weights must be bf16 or fp16, got {dt}")
    return dev, dt, {k: v.to(device=dev, dtype=dt).contiguous() for k, v in params.items()}


class CLIPTextModel:
    """Implements the text encoder transformer from CLIP (reference mlx/clip.py:63-120)."""

    def __init__(self, params: Dict[str, torch.Tensor], config: CLIPTextModelConfig, device=None):
        self.device, self.dtype, p = _device_params(params, device, "CLIPTextModel")
        self.config = config
        self.max_length = config.max_length
        if config.model_dims % config.num_heads or config.model_dims // config.num_heads != 64:
            raise DkError("CLIPTextModel: head dim must be 64 (CLIP-L/14 and OpenCLIP bigG both are)")
        if config.hidden_act not in ("quick_gelu", "gelu"):
            raise ValueError(f"unknown CLIP activation {config.hidden_act}")
        self.act = ACT_QUICK_GELU if config.hidden_act == "quick_gelu" else ACT_GELU_ERF
        self.p = p
        self.layers = []
        for i in range(config.num_layers):
            a = f"layers.{i}.attention."
            w_qkv = torch.cat([p[a + "query_proj.weight"], p[a + "key_proj.weight"], p[a + "value_proj.weight"]]).contiguous()
            b_qkv = torch.cat([p[a + "query_proj.bias"], p[a + "key_proj.bias"], p[a + "value_proj.bias"]]).contiguous()
            self.layers.append((w_qkv, b_qkv))

    def __call__(self, x: torch.Tensor) -> CLIPOutput:
        """x: integer token ids (B, N), N <= max_length"""
        cfg, p = self.config, self.p
        ids = torch.as_tensor(x)
        B, N = ids.shape
        if N > cfg.max_length:
            raise ValueError(f"CLIPTextModel: {N} tokens exceed max_length {cfg.max_length}")
        eos_tokens = ids.argmax(-1).to(self.device)                          # clip.py:94 (EOS has the largest id)
        ids32 = ids.to(device=self.device, dtype=torch.int32).contiguous()
        h = ops.embedding(p["token_embedding.weight"], ids32, pos=p["position_embedding.weight"][:N].contiguous())
        heads = cfg.num_heads
        scale = math.sqrt(1.0 / 64)
        hidden_states = []
        for i, (w_qkv, b_qkv) in enumerate(self.layers):
            l = f"layers.{i}."
            y = ops.layernorm(h, p[l + "layer_norm1.weight"], p[l + "layer_norm1.bias"], 1e-5)
            qkv = ops.gemm(y, w_qkv, bias=b_qkv)
            att = ops.attention_small(qkv, B, N, heads, scale, causal=True)   # mask: clip.py:84-90
            h = ops.gemm(att, p[l + "attention.out_proj.weight"], bias=p[l + "attention.out_proj.bias"], res=h)
            y = ops.layernorm(h, p[l + "layer_norm2.weight"], p[l + "layer_norm2.bias"], 1e-5)
            y = ops.gemm(y, p[l + "linear1.weight"], bias=p[l + "linear1.bias"], act=self.act)
            h = ops.gemm(y, p[l + "linear2.weight"], bias=p[l + "linear2.bias"], res=h)
            hidden_states.append(h.reshape(B, N, -1))
        last = ops.layernorm(h, p["final_layer_norm.weight"], p["final_layer_norm.bias"], 1e-5).reshape(B, N, -1)
        pooled = last[torch.arange(B, device=self.device), eos_tokens].contiguous()
        if "text_projection.weight" in p:
            pooled = ops.gemm(pooled, p["text_projection.weight"])
        return CLIPOutput(pooled_output=pooled, last_hidden_state=last, hidden_states=hidden_states)


def relative_position_bucket(relative_position: np.ndarray, bidirectional: bool = True, num_buckets: int = 32,
                             max_distance: int = 128) -> np.ndarray:
    """reference mlx/t5.py:21-64 (the int16 truncation and the fp32 `log(n / max_exact) * scale` order included)"""
    rel = np.asarray(relative_position, dtype=np.int64)
    buckets = np.zeros_like(rel)
    if bidirectional:
        num_buckets //= 2
        buckets += (rel > 0).astype(np.int64) * num_buckets
        rel = np.abs(rel)
    else:
        rel = -np.minimum(rel, 0)
    max_exact = num_buckets // 2
    is_small = rel < max_exact
    scale = np.float32((num_buckets - max_exact) / np.log(max_distance / max_exact))
    with np.errstate(divide="ignore"):
        val = np.log(rel.astype(np.float32) / np.float32(max_exact)) * scale
    large = max_exact + np.where(is_small, 0, np.trunc(np.where(is_small, 0.0, val))).astype(np.int64)
    large = np.minimum(large, num_buckets - 1)
    return buckets + np.where(is_small, rel, large)


class SD3T5Encoder:
    """wte + TransformerEncoder (reference mlx/t5.py:226-243, 316-325)."""

    def __init__(self, params: Dict[str, torch.Tensor], config: T5EncoderConfig = T5EncoderConfig(), device=None,
                 low_memory_mode: bool = True):
        self.device, self.dtype, p = _device_params(params, device, "SD3T5Encoder")
        self.config = config
        self.model_dim = config.d_model
        if config.d_kv != 64:
            raise DkError("SD3T5Encoder: d_kv must be 64")
        if config.feed_forward_proj != "gated-gelu":
            raise DkError("SD3T5Encoder: only the gated-gelu feed-forward of t5-v1_1 is implemented")
        self.p = p
        self.layers = []
        for i in range(config.num_layers):
            l = f"encoder.layers.{i}."
            w_qkv = torch.cat([p[l + "attention.query_proj.weight"], p[l + "attention.key_proj.weight"],
                               p[l + "attention.value_proj.weight"]]).contiguous()
            w_in = torch.cat([p[l + "dense.wi_0.weight"], p[l + "dense.wi_1.weight"]]).contiguous()
            self.layers.append((w_qkv, w_in))
        self._bias_cache: Dict[int, torch.Tensor] = {}

    def relative_bias(self, L: int) -> torch.Tensor:
        """[heads, 2L-1] table: entry (h, j - i + L - 1) is the bias of key j for query i (t5.py:79-102)"""
        if L not in self._bias_cache:
            c = self.config
            rel = np.arange(-(L - 1), L)
            b = relative_position_bucket(rel, True, c.relative_attention_num_buckets, c.relative_attention_max_distance)
            emb = self.p["encoder.relative_attention_bias.embeddings.weight"]              # [buckets, heads]
            self._bias_cache[L] = emb[torch.from_numpy(b).to(self.device)].t().contiguous()
        return self._bias_cache[L]

    def __call__(self, inputs: torch.Tensor) -> torch.Tensor:
        """inputs: integer token ids (B, L), L <= 512 -> (B, L, d_model) in the weight dtype"""
        c, p = self.config, self.p
        ids = torch.as_tensor(inputs)
        B, L = ids.shape
        ids32 = ids.to(device=self.device, dtype=torch.int32).contiguous()
        x = ops.cast_to_f32(ops.embedding(p["wte.weight"], ids32))           # residual stream in fp32 (t5.py:214-221)
        bias = self.relative_bias(L)
        eps = c.layer_norm_epsilon
        for i, (w_qkv, w_in) in enumerate(self.layers):
            l = f"encoder.layers.{i}."
            y = ops.rmsnorm_f32(x, p[l + "ln1.weight"], eps)
            qkv = ops.gemm(y, w_qkv)
            att = ops.attention_small(qkv, B, L, c.num_heads, 1.0, rel_bias=bias)      # no 1/sqrt(d) in T5
            ops.add_f32_16(x, ops.gemm(att, p[l + "attention.out_proj.weight"]))
            y = ops.rmsnorm_f32(x, p[l + "ln2.weight"], eps)
            g = ops.glu_gelu(ops.gemm(y, w_in))
            ops.add_f32_16(x, ops.gemm(g, p[l + "dense.wo.weight"]))
        return ops.rmsnorm_f32(x, p["encoder.ln.weight"], eps).reshape(B, L, c.d_model)
