"""Parameter trees (names/shapes exactly as the reference's module tree after its checkpoint remapping,
SURVEY.md App. C; reference mlx/mmdit.py module attributes, mlx/vae.py:349-384) and the deterministic synthetic
initialiser used by tests and benchmarks (there are no checkpoints in the sandbox; SURVEY.md §8d).

Initialiser: Linear/Conv weight ~ N(0, 1/fan_in); biases ~ N(0, 0.02^2); RMSNorm/GroupNorm weight = 1 + N(0, 0.02^2);
GroupNorm bias, position table ~ N(0, 0.02^2).  One torch.Generator per tensor, seeded from (seed, index), so any
subset of tensors can be generated independently and on either device.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import torch

from .config import MMDiTConfig, PositionalEncoding, VAEDecoderConfig, VAEEncoderConfig

# kind: "w" matrix/conv weight (fan_in = prod(shape[1:])), "b" bias, "g" norm gain, "e" embedding table
Spec = Tuple[str, Tuple[int, ...], str]


def mmdit_param_specs(cfg: MMDiTConfig) -> List[Spec]:
    h = cfg.hidden_size
    d = cfg.head_dim
    p = cfg.patch_size
    specs: List[Spec] = []

    def lin(name, out_f, in_f, bias=True):
        specs.append((name + ".weight", (out_f, in_f), "w"))
        if bias:
            specs.append((name + ".bias", (out_f,), "b"))

    if cfg.patchify_via_reshape:
        specs.append(("x_embedder.proj.weight", (h, 1, 1, cfg.vae_latent_dim * p * p + cfg.x_embedder_cond_channels),
                      "w"))
    else:
        specs.append(("x_embedder.proj.weight", (h, p, p, cfg.vae_latent_dim), "w"))
    specs.append(("x_embedder.proj.bias", (h,), "b"))
    if cfg.pos_embed_type == PositionalEncoding.LearnedInputEmbedding:
        specs.append(("x_pos_embedder.pos_embed.weight", (cfg.max_latent_resolution ** 2, h), "e"))
    lin("y_embedder.mlp.layers.0", h, cfg.pooled_text_embed_dim)
    lin("y_embedder.mlp.layers.2", h, h)
    lin("t_embedder.mlp.layers.0", h, cfg.frequency_embed_dim)
    lin("t_embedder.mlp.layers.2", h, h)
    lin("context_embedder", h, cfg.token_level_text_embed_dim)

    def block(prefix, n_mod, skip_post=False):
        lin(prefix + ".attn.q_proj", h, h)
        lin(prefix + ".attn.k_proj", h, h, bias=False)
        lin(prefix + ".attn.v_proj", h, h)
        if not skip_post:
            lin(prefix + ".attn.o_proj", h, h)
            lin(prefix + ".mlp.fc1", cfg.mlp_ratio * h, h)
            lin(prefix + ".mlp.fc2", h, cfg.mlp_ratio * h)
        lin(prefix + ".adaLN_modulation.layers.1", n_mod * h, h)
        if cfg.use_qk_norm:
            specs.append((prefix + ".qk_norm.q_norm.weight", (d,), "g"))
            specs.append((prefix + ".qk_norm.k_norm.weight", (d,), "g"))

    x_layers = set(cfg.x_block_self_attn_layers)
    for i in range(cfg.depth_multimodal):
        skip_text = (i == cfg.depth_multimodal - 1) and (cfg.depth_unified < 1)
        block(f"multimodal_transformer_blocks.{i}.image_transformer_block", 9 if i in x_layers else 6)
        block(f"multimodal_transformer_blocks.{i}.text_transformer_block", 2 if skip_text else 6, skip_post=skip_text)
    for i in range(cfg.depth_unified):
        block(f"unified_transformer_blocks.{i}.transformer_block", 3 if cfg.parallel_mlp_for_unified_blocks else 6)
    lin("final_layer.linear", p * p * cfg.vae_latent_dim, h)
    lin("final_layer.adaLN_modulation.layers.1", 2 * h, h)
    if cfg.guidance_embed:
        # FLUX.1-dev's guidance MLPEmbedder (reference mlx/mmdit.py:31-34, 945-955).  Last, so that init_params (seeded
        # by spec index) gives every other tensor the values it has without the embedder.
        lin("guidance_in.mlp.layers.0", h, cfg.frequency_embed_dim)
        lin("guidance_in.mlp.layers.2", h, h)
    # MMDiT-X (SD3.5 Medium) and the kept k bias, appended for the same reason
    for i in sorted(x_layers):
        prefix = f"multimodal_transformer_blocks.{i}.image_transformer_block"
        for n in "qkvo":
            lin(f"{prefix}.attn2.{n}_proj", h, h, bias=n != "k" or cfg.attn_k_bias)
        specs.append((prefix + ".qk_norm2.q_norm.weight", (d,), "g"))
        specs.append((prefix + ".qk_norm2.k_norm.weight", (d,), "g"))
    if cfg.attn_k_bias:
        for name, _, _ in list(specs):
            if name.endswith(".attn.k_proj.weight"):
                specs.append((name[:-len("weight")] + "bias", (h,), "b"))
    return specs


class _VaeSpecBuilder:
    def __init__(self):
        self.specs: List[Spec] = []

    def conv(self, name, cout, cin):
        self.specs.append((name + ".weight", (cout, 3, 3, cin), "w"))
        self.specs.append((name + ".bias", (cout,), "b"))

    def gn(self, name, c):
        self.specs.append((name + ".weight", (c,), "g"))
        self.specs.append((name + ".bias", (c,), "b"))

    def lin(self, name, cout, cin):
        self.specs.append((name + ".weight", (cout, cin), "w"))
        self.specs.append((name + ".bias", (cout,), "b"))

    def resnet(self, name, cin, cout):
        self.gn(name + ".norm1", cin)
        self.conv(name + ".conv1", cout, cin)
        self.gn(name + ".norm2", cout)
        self.conv(name + ".conv2", cout, cout)
        if cin != cout:
            self.lin(name + ".conv_shortcut", cout, cin)

    def mid(self, top):
        self.resnet("mid_blocks.0", top, top)
        self.gn("mid_blocks.1.group_norm", top)
        for n in ("query_proj", "key_proj", "value_proj", "out_proj"):
            self.lin("mid_blocks.1." + n, top, top)
        self.resnet("mid_blocks.2", top, top)


def vae_encoder_param_specs(cfg: VAEEncoderConfig = VAEEncoderConfig()) -> List[Spec]:
    """reference VAEEncoder module tree (mlx/vae.py:404-451)"""
    b = _VaeSpecBuilder()
    boc = list(cfg.block_out_channels)
    b.conv("conv_in", boc[0], cfg.in_channels)
    channels = [boc[0]] + boc
    for i, (cin, cout) in enumerate(zip(channels, channels[1:])):
        for l in range(cfg.layers_per_block):
            b.resnet(f"down_blocks.{i}.resnets.{l}", cin if l == 0 else cout, cout)
        if i < len(boc) - 1:
            b.conv(f"down_blocks.{i}.downsample", cout, cout)
    b.mid(boc[-1])
    b.gn("conv_norm_out", boc[-1])
    b.conv("conv_out", cfg.out_channels, boc[-1])
    return b.specs


def vae_decoder_param_specs(cfg: VAEDecoderConfig = VAEDecoderConfig()) -> List[Spec]:
    b = _VaeSpecBuilder()
    specs = b.specs
    conv, gn, resnet = b.conv, b.gn, b.resnet
    boc = list(cfg.block_out_channels)
    top = boc[-1]
    conv("conv_in", top, cfg.in_channels)
    b.mid(top)
    channels = list(reversed(boc))
    channels = [channels[0]] + channels
    n_blocks = len(boc)
    # up_blocks list is built with insert(0, ...) (vae.py:367-379): the i-th constructed block lands at index n-1-i
    for i, (cin, cout) in enumerate(zip(channels, channels[1:])):
        j = n_blocks - 1 - i
        for l in range(cfg.layers_per_block):
            resnet(f"up_blocks.{j}.resnets.{l}", cin if l == 0 else cout, cout)
        if i < n_blocks - 1:
            conv(f"up_blocks.{j}.upsample", cout, cout)
    gn("conv_norm_out", boc[0])
    conv("conv_out", cfg.out_channels, boc[0])
    return specs


def init_params(specs: List[Spec], seed: int = 0, dtype: torch.dtype = torch.bfloat16,
                device: str | torch.device = "cpu") -> Dict[str, torch.Tensor]:
    """Deterministic synthetic parameters.  Values are generated in fp32 on `device` and cast to `dtype`."""
    out: Dict[str, torch.Tensor] = {}
    dev = torch.device(device)
    for idx, (name, shape, kind) in enumerate(specs):
        g = torch.Generator(device=dev)
        g.manual_seed(seed * 1000003 + idx)
        t = torch.randn(shape, generator=g, device=dev, dtype=torch.float32)
        if kind == "w":
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            t = t * (1.0 / fan_in ** 0.5)
        elif kind == "g":
            t = 1.0 + 0.02 * t
        else:  # "b", "e"
            t = 0.02 * t
        out[name] = t.to(dtype)
    return out


def param_count(specs: List[Spec]) -> int:
    n = 0
    for _, shape, _ in specs:
        k = 1
        for s in shape:
            k *= s
        n += k
    return n
