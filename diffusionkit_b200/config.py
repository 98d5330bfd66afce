"""Model hyper-parameters — same field names and preset names as the reference
(python/src/diffusionkit/mlx/config.py:19-111, 126-132), with torch dtypes instead of mx dtypes."""
from dataclasses import dataclass, field, replace
from enum import Enum
from typing import List, Optional, Tuple

import torch


class PositionalEncoding(Enum):
    LearnedInputEmbedding = 1
    PreSDPARope = 2


@dataclass
class MMDiTConfig:
    """Multi-modal Diffusion Transformer configuration (reference mlx/config.py:19-71)."""

    num_heads: int = 24
    depth_multimodal: int = 24
    depth_unified: int = 0
    parallel_mlp_for_unified_blocks: bool = True
    mlp_ratio: int = 4
    vae_latent_dim: int = 16
    layer_norm_eps: float = 1e-6
    pos_embed_type: PositionalEncoding = PositionalEncoding.LearnedInputEmbedding
    rope_axes_dim: Optional[Tuple[int, ...]] = None
    use_qk_norm: bool = False
    upcast_multimodal_blocks: Optional[List[int]] = None
    upcast_unified_blocks: Optional[List[int]] = None
    hidden_size_override: Optional[int] = None

    @property
    def hidden_size(self) -> int:
        return self.hidden_size_override or (64 * self.depth_multimodal)

    max_latent_resolution: int = 192
    patch_size: int = 2
    patchify_via_reshape: bool = False
    pooled_text_embed_dim: int = 2048
    token_level_text_embed_dim: int = 4096
    frequency_embed_dim: int = 256
    max_period: int = 10000
    dtype: torch.dtype = torch.bfloat16
    float16_dtype: torch.dtype = torch.bfloat16
    low_memory_mode: bool = True
    guidance_embed: bool = False
    # MMDiT-X (SD3.5 Medium): the joint blocks whose image stream has a second self-attention, attn2, over the image
    # tokens only, with its own adaLN shift, scale and gate (Stability's field name)
    x_block_self_attn_layers: Tuple[int, ...] = ()
    # keep the k bias of the q/k/v projections; False drops it (quirk Q3), which SD3.5 Medium cannot: with QK-RMSNorm
    # the bias enters before the norm and changes the output
    attn_k_bias: bool = False
    # FLUX.1 Fill: input channels of the x-embedder beyond the packed latent's, the masked-image latent (64) and the
    # mask (256) of every token (DESIGN.md §18); 0 for every other model
    x_embedder_cond_channels: int = 0
    # FLUX.1 Canny / Depth [dev]: "canny" or "depth" names the control image's preprocessing and the default guidance
    # (DESIGN.md §19); None for every other model
    control: Optional[str] = None

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_heads


SD3_8b = MMDiTConfig(depth_multimodal=38, num_heads=38, upcast_multimodal_blocks=[35], use_qk_norm=True)

SD3_2b = MMDiTConfig(depth_multimodal=24, num_heads=24, float16_dtype=torch.float16, dtype=torch.float16)

FLUX_SCHNELL = MMDiTConfig(
    num_heads=24,
    depth_multimodal=19,
    depth_unified=38,
    parallel_mlp_for_unified_blocks=True,
    hidden_size_override=3072,
    patchify_via_reshape=True,
    pos_embed_type=PositionalEncoding.PreSDPARope,
    rope_axes_dim=(16, 56, 56),
    pooled_text_embed_dim=768,
    use_qk_norm=True,
    float16_dtype=torch.bfloat16,
    dtype=torch.bfloat16,
)

# Stability's SD3.5 Medium: SD3-medium's width and depth with QK-RMSNorm, a 384^2 position table, attn2 in joint
# blocks 0-12 (MMDiT-X) and the k bias kept (DESIGN.md §13)
SD35_MEDIUM = replace(SD3_2b, use_qk_norm=True, max_latent_resolution=384, x_block_self_attn_layers=tuple(range(13)),
                      attn_k_bias=True)

# Defined by the reference but never used: FLUX.1-dev is loaded with FLUX_SCHNELL (mlx/model_io.py:109,756; quirk Q1).
# Here mmdit_config=FLUX_DEV opts in to the guidance embedder (DESIGN.md §12); MODEL_CONFIGS keeps the quirk.
FLUX_DEV = replace(FLUX_SCHNELL, guidance_embed=True)

# FLUX.1 Fill [dev]: FLUX.1-dev with 320 conditioning channels per token in the x-embedder input (DESIGN.md §18)
FLUX_FILL_DEV = replace(FLUX_DEV, x_embedder_cond_channels=320)

# FLUX.1 Canny [dev] and FLUX.1 Depth [dev]: FLUX.1-dev with the control image's 64 latent channels per token in the
# x-embedder input (DESIGN.md §19)
FLUX_CANNY_DEV = replace(FLUX_DEV, x_embedder_cond_channels=64, control="canny")
FLUX_DEPTH_DEV = replace(FLUX_DEV, x_embedder_cond_channels=64, control="depth")


@dataclass
class VAEDecoderConfig:
    """reference mlx/config.py:126-132"""

    in_channels: int = 16
    out_channels: int = 3
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: int = 3
    resnet_groups: int = 32


@dataclass
class VAEEncoderConfig:
    """reference mlx/config.py:135-141"""

    in_channels: int = 3
    out_channels: int = 32
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: int = 2
    resnet_groups: int = 32


# model_version -> config, as the reference's loader resolves it (mlx/model_io.py:105-112)
MODEL_CONFIGS = {
    "argmaxinc/mlx-stable-diffusion-3-medium": SD3_2b,
    "argmaxinc/mlx-FLUX.1-schnell": FLUX_SCHNELL,
    "argmaxinc/mlx-FLUX.1-schnell-4bit-quantized": FLUX_SCHNELL,
    "argmaxinc/mlx-FLUX.1-dev": FLUX_SCHNELL,  # quirk Q1
    "argmaxinc/mlx-stable-diffusion-3.5-large": SD3_8b,
    "argmaxinc/mlx-stable-diffusion-3.5-large-4bit-quantized": SD3_8b,
    "stabilityai/stable-diffusion-3.5-medium": SD35_MEDIUM,
    # FLUX.1 Kontext [dev]: FLUX.1-dev's architecture and guidance embedder, run with reference tokens (DESIGN.md §14)
    "black-forest-labs/FLUX.1-Kontext-dev": FLUX_DEV,
    # FLUX.1 Fill [dev]: masked-image and mask channels in the x-embedder input (DESIGN.md §18)
    "black-forest-labs/FLUX.1-Fill-dev": FLUX_FILL_DEV,
}

# model_version -> config of the structural-control models (DESIGN.md §19), resolved like MODEL_CONFIGS; a table of
# their own because FLUX.1 Fill is the only model of MODEL_CONFIGS with conditioning channels in the x-embedder
CONTROL_MODEL_CONFIGS = {
    "black-forest-labs/FLUX.1-Canny-dev": FLUX_CANNY_DEV,
    "black-forest-labs/FLUX.1-Depth-dev": FLUX_DEPTH_DEV,
}

# T5 sequence lengths (mlx/__init__.py:46-53)
T5_MAX_LENGTH = {
    "argmaxinc/mlx-stable-diffusion-3-medium": 512,
    "argmaxinc/mlx-stable-diffusion-3.5-large": 512,
    "argmaxinc/mlx-stable-diffusion-3.5-large-4bit-quantized": 512,
    "argmaxinc/mlx-FLUX.1-schnell": 256,
    "argmaxinc/mlx-FLUX.1-schnell-4bit-quantized": 256,
    "argmaxinc/mlx-FLUX.1-dev": 512,
    "stabilityai/stable-diffusion-3.5-medium": 512,
    "black-forest-labs/FLUX.1-Kontext-dev": 512,
    "black-forest-labs/FLUX.1-Fill-dev": 512,
    "black-forest-labs/FLUX.1-Canny-dev": 512,
    "black-forest-labs/FLUX.1-Depth-dev": 512,
}


def tiny_sd35_config(hidden: int = 128, heads: int = 2, depth: int = 2) -> MMDiTConfig:
    """Small SD3.5-shaped config for tests: learned positional embedding + QK-RMSNorm, head dim 64, bf16 sinusoid
    (SD3_8b keeps the dataclass default dtype, mlx/config.py:74-76)."""
    return MMDiTConfig(num_heads=heads, depth_multimodal=depth, hidden_size_override=hidden, use_qk_norm=True,
                       upcast_multimodal_blocks=[depth - 1], max_latent_resolution=24, pooled_text_embed_dim=64,
                       token_level_text_embed_dim=128)


def tiny_sd35_medium_config() -> MMDiTConfig:
    """Small SD3.5-Medium-shaped config for tests: MMDiT-X blocks 0 and 1 of 3, QK-RMSNorm, k bias, fp16."""
    return replace(tiny_sd3_config(), use_qk_norm=True, x_block_self_attn_layers=(0, 1), attn_k_bias=True)


def tiny_flux_config(hidden: int = 256, heads: int = 2, depth_mm: int = 2, depth_uni: int = 2) -> MMDiTConfig:
    """Small FLUX-shaped config for tests (head dim 128 like the real model)."""
    d = hidden // heads
    assert d in (64, 128)
    axes = (16, 56, 56) if d == 128 else (8, 28, 28)
    return replace(FLUX_SCHNELL, num_heads=heads, depth_multimodal=depth_mm, depth_unified=depth_uni,
                   hidden_size_override=hidden, rope_axes_dim=axes, pooled_text_embed_dim=64,
                   token_level_text_embed_dim=128)


def tiny_sd3_config(hidden: int = 128, heads: int = 2, depth_mm: int = 3) -> MMDiTConfig:
    """Small SD3-shaped config for tests (head dim 64 like the real model)."""
    assert hidden // heads == 64
    return replace(SD3_2b, num_heads=heads, depth_multimodal=depth_mm, hidden_size_override=hidden,
                   max_latent_resolution=24, pooled_text_embed_dim=64, token_level_text_embed_dim=128)


@dataclass
class CLIPTextModelConfig:
    """reference mlx/config.py:144-152 (defaults are the reference's; CLIP_L / CLIP_G below are the values of the
    config.json files the reference downloads, model_io.py:799-816)"""

    num_layers: int = 23
    model_dims: int = 1024
    num_heads: int = 16
    max_length: int = 77
    vocab_size: int = 49408
    projection_dim: Optional[int] = None
    hidden_act: str = "quick_gelu"


CLIP_L = CLIPTextModelConfig(num_layers=12, model_dims=768, num_heads=12, projection_dim=None, hidden_act="quick_gelu")
CLIP_G = CLIPTextModelConfig(num_layers=32, model_dims=1280, num_heads=20, projection_dim=1280, hidden_act="gelu")


@dataclass
class T5EncoderConfig:
    """The fields of transformers.T5Config the reference reads (mlx/t5.py), with google/t5-v1_1-xxl's values
    (reference model_io.py:928, T5Config.from_pretrained("google/t5-v1_1-xxl"))."""

    vocab_size: int = 32128
    d_model: int = 4096
    d_kv: int = 64
    d_ff: int = 10240
    num_layers: int = 24
    num_heads: int = 64
    relative_attention_num_buckets: int = 32
    relative_attention_max_distance: int = 128
    layer_norm_epsilon: float = 1e-6
    feed_forward_proj: str = "gated-gelu"


@dataclass
class SiglipVisionConfig:
    """The fields of transformers.SiglipVisionConfig the FLUX.1 Redux image encoder reads (DESIGN.md §15)."""

    hidden_size: int = 1152
    num_attention_heads: int = 16
    intermediate_size: int = 4304
    num_hidden_layers: int = 27
    patch_size: int = 14
    image_size: int = 384
    layer_norm_eps: float = 1e-6
    hidden_act: str = "gelu_pytorch_tanh"

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_attention_heads

    @property
    def num_patches(self) -> int:
        """tokens per image: the stride-p convolution without padding drops image_size % patch_size pixels"""
        return (self.image_size // self.patch_size) ** 2


# google/siglip-so400m-patch14-384, the vision tower of BFL's FLUX.1 Redux [dev] (prepare_redux)
SIGLIP_SO400M_PATCH14_384 = SiglipVisionConfig()


def tiny_siglip_config(image_size: int = 98, layers: int = 2) -> SiglipVisionConfig:
    """Small SigLIP for tests: 2 heads of SigLIP's head dim 72, so the attention padding is exercised."""
    return SiglipVisionConfig(hidden_size=144, num_attention_heads=2, intermediate_size=304, num_hidden_layers=layers,
                              image_size=image_size)


@dataclass
class DepthAnythingConfig:
    """The fields of transformers.DepthAnythingConfig (with its Dinov2Config backbone) that FLUX.1 Depth's depth
    estimator reads (DESIGN.md §20)."""

    hidden_size: int = 1024
    num_attention_heads: int = 16
    intermediate_size: int = 4096
    num_hidden_layers: int = 24
    patch_size: int = 14
    image_size: int = 518                      # the position table covers (image_size / patch_size)^2 patches
    layer_norm_eps: float = 1e-6
    hidden_act: str = "gelu"
    out_indices: Tuple[int, ...] = (21, 22, 23, 24)
    neck_hidden_sizes: Tuple[int, ...] = (256, 512, 1024, 1024)
    reassemble_factors: Tuple[float, ...] = (4, 2, 1, 0.5)
    fusion_hidden_size: int = 256
    head_hidden_size: int = 32
    depth_estimation_type: str = "relative"

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_attention_heads

    @property
    def pos_grid(self) -> int:
        """side of the square position table without its CLS row: 518 / 14 = 37"""
        return self.image_size // self.patch_size


# LiheYoung/depth-anything-large-hf, the estimator of BFL's FLUX.1 Depth [dev] (DepthImageEncoder)
DEPTH_ANYTHING_LARGE = DepthAnythingConfig()


def tiny_depth_anything_config(layers: int = 4) -> DepthAnythingConfig:
    """Small Depth Anything for tests: 2 heads of 64, the last four layers as the stages, the smallest widths the
    kernels take (channel counts multiples of 64, fusion width 128 so the head's first convolution gives 64)."""
    return DepthAnythingConfig(hidden_size=128, num_attention_heads=2, intermediate_size=512, num_hidden_layers=layers,
                               out_indices=tuple(range(layers - 3, layers + 1)), neck_hidden_sizes=(64, 128, 128, 128),
                               fusion_hidden_size=128)


def tiny_clip_config(projection: bool = True, act: str = "quick_gelu") -> CLIPTextModelConfig:
    return CLIPTextModelConfig(num_layers=3, model_dims=128, num_heads=2, max_length=77, vocab_size=1000,
                               projection_dim=64 if projection else None, hidden_act=act)


def tiny_t5_config() -> T5EncoderConfig:
    return T5EncoderConfig(vocab_size=512, d_model=256, d_kv=64, d_ff=512, num_layers=3, num_heads=4)
