"""VAE decoder and encoder on H100 — host-side mirrors of the reference VAEDecoder / VAEEncoder
(python/src/diffusionkit/mlx/vae.py:336-401 and :404-467; ResnetBlock2D :60-101, Attention :28-57,
upsample_nearest :20-25, EncoderDecoderBlock2D :103-148).

Same parameter names as the reference module tree (SURVEY.md App. C).  Kernels (csrc/):
  conv 3x3        : wgmma implicit GEMM, the 9 taps are shifted 4-D TMA boxes (zero fill = padding), bias and the
                    ResNet skip fused in the epilogue
  GroupNorm(32)   : two-stage fp32 statistics + fused normalise/affine/SiLU
  conv 3x3 / 2    : same kernel, the TMA box walks the input with element stride 2 (zero fill = the reference's
                    bottom/right pad, vae.py:142-144)
  mid attention   : q/k/v/out projections and both S=HW x HW matmuls on the wgmma GEMM (scores materialised like the
                    reference, vae.py:49-52; V consumed as an MN-major operand), fp32 row softmax; 1/sqrt(C) is folded
                    into the query projection once at load (the reference scales q before q k^T, :49: the unscaled
                    product would reach the fp16 limit 22x earlier)
  fused convolution (decoder, wherever dk_conv_fused_supported accepts the shape — rows of >= 128 pixels, Cin <= 512):
                    csrc/conv_fused.cu, ONE kernel per convolution = GroupNorm-apply + SiLU on the staged halo tile ->
                    [nearest 2x by sub-pixel phases] -> conv 3x3 -> bias / skip -> output + the NEXT GroupNorm's partial
                    statistics.  No normalised tensor, no upsampled tensor and no separate statistics pass touch HBM.
                    Other shapes, and the whole encoder, run the three unfused kernels above.
  The whole decode is captured in a CUDA graph per input shape (graphs.py).
"""
from __future__ import annotations

import math
from typing import Dict

import torch

from . import ops
from ._lib import DkError
from .config import VAEDecoderConfig, VAEEncoderConfig
from .graphs import ShapeCache, default_settings


def _pad_dim(t: torch.Tensor, dim: int, to: int) -> torch.Tensor:
    if t.shape[dim] == to:
        return t.contiguous()
    shape = list(t.shape)
    shape[dim] = to - t.shape[dim]
    return torch.cat([t, torch.zeros(shape, dtype=t.dtype, device=t.device)], dim=dim).contiguous()


class _VAEBlocks:
    """Parameter handling and the building blocks the decoder and the encoder share."""

    fuse = True                                       # take the fused convolution wherever the shape allows

    def __init__(self, params: Dict[str, torch.Tensor], config, device=None):
        who = type(self).__name__
        any_p = next(iter(params.values()))
        self.device = torch.device(device) if device is not None else any_p.device
        if self.device.type != "cuda":
            raise DkError(f"{who}: parameters must live on a CUDA device (no CPU fallback)")
        self.dtype = any_p.dtype
        if self.dtype not in (torch.bfloat16, torch.float16):
            raise DkError(f"{who}: weights must be bf16 or fp16, got {self.dtype}")
        self.config = config
        self.groups = config.resnet_groups
        self.p = {k: v.to(device=self.device, dtype=self.dtype).contiguous() for k, v in params.items()}
        # attention scale 1/sqrt(C) folded into the query projection (fp32 product, rounded once): the reference computes
        # (q * scale) @ k^T (vae.py:49); scaling after the product would overflow fp16 22x earlier
        for k in [k for k in self.p if k.endswith("query_proj.weight")]:
            sc = 1.0 / math.sqrt(self.p[k].shape[0])
            self.p[k] = (self.p[k].float() * sc).to(self.dtype)
            kb = k[:-6] + "bias"
            self.p[kb] = (self.p[kb].float() * sc).to(self.dtype)

    # ------------------------------------------------------------------ building blocks
    def _conv(self, x, conv, norm=None, st=None, res=None, up=False):
        """[GroupNorm(norm) + SiLU] -> [nearest 2x] -> conv3x3 (+ bias, + res) -> (y, statistics of y).  One halo-tiled
        kernel where the module fuses and the shape allows, else GroupNorm-apply, upsample and implicit-GEMM conv."""
        w, b = self.p[conv + ".weight"], self.p[conv + ".bias"]
        B, H, W, C = x.shape
        Cout = w.shape[0]
        gn = None if norm is None else (st.get(), self.p[norm + ".weight"], self.p[norm + ".bias"], self.groups)
        if self.fuse and ops.conv_fused_supported(H, W, C, Cout):
            part = None
            if Cout % 128 == 0:                           # a narrow output tile (conv_out) writes no statistics
                part = torch.empty((B, (4 if up else 1) * H * W // 128, self.groups, 2), dtype=torch.float32,
                                   device=self.device)
            y = ops.conv3x3_fused(x, self.up_w[conv] if up else w, bias=b, res=res, up=up, gn=gn, silu=gn is not None,
                                  out_partial=part, out_G=self.groups)
            return y, _Stats(y, self.groups, part)
        if gn is not None:
            x = ops.groupnorm_apply(x, *gn, True)
        if up:
            x = ops.upsample_nearest2x(x)
        y = ops.conv3x3(x, w, b, res=res)
        return y, _Stats(y, self.groups)

    def _lin(self, x2d, name, res=None):
        return ops.gemm(x2d, self.p[name + ".weight"], bias=self.p[name + ".bias"], res=res)

    def _resnet(self, x, st, name):
        """ResnetBlock2D.__call__ (vae.py:86-101)"""
        y, st = self._conv(x, name + ".conv1", name + ".norm1", st)
        skip = x
        if (name + ".conv_shortcut.weight") in self.p:
            B, H, W, C = x.shape
            skip = self._lin(x.reshape(B * H * W, C), name + ".conv_shortcut").reshape(B, H, W, -1)
        return self._conv(y, name + ".conv2", name + ".norm2", st, res=skip)

    def _attention(self, x, st, name):
        """Attention.__call__ (vae.py:40-57): single head over the H*W positions."""
        B, H, W, C = x.shape
        S = H * W
        y = ops.groupnorm_apply(x, st.get(), self.p[name + ".group_norm.weight"], self.p[name + ".group_norm.bias"],
                                self.groups, False).reshape(B * S, C)
        q = self._lin(y, name + ".query_proj")
        k = self._lin(y, name + ".key_proj")
        v = self._lin(y, name + ".value_proj")
        o = torch.empty((B * S, C), dtype=self.dtype, device=self.device)
        scores = torch.empty((S, S), dtype=self.dtype, device=self.device)
        for b in range(B):
            sl = slice(b * S, (b + 1) * S)
            ops.gemm(q[sl], k[sl], out=scores)                       # (scale q) k^T: the scale lives in query_proj
            ops.softmax_rows(scores, 1.0)
            ops.gemm(scores, v[sl], out=o[sl], w_n_major=True)        # P v   (v is [S, C] = [K, N] row-major)
        out = self._lin(o, name + ".out_proj", res=x.reshape(B * S, C)).reshape(B, H, W, C)
        return out, _Stats(out, self.groups)

    def _pad_channels(self, x, to):
        B, H, W, C = x.shape
        xin = torch.zeros((B, H, W, to), dtype=self.dtype, device=self.device)
        ops.copy_rows(x, xin, B * H * W, 1, C, to // C, 0, 1, 0)
        return xin


class _Stats:
    """GroupNorm statistics of a tensor, produced on first use: folded from the partial sums the producing fused
    convolution wrote in its epilogue (dk_groupnorm_finalize), or, without them, by the standalone two-stage kernel."""

    def __init__(self, x, groups, partial=None):
        self.x, self.groups, self.partial, self._stats = x, groups, partial, None

    def get(self):
        if self._stats is None:
            B, H, W, C = self.x.shape
            G = self.groups
            if self.partial is not None:
                self._stats = ops.groupnorm_finalize(self.partial, B, G, H * W // 128, float(H * W * (C // G)), 1e-5)
            else:
                self._stats = ops.groupnorm_stats(self.x, G, 1e-5)
        return self._stats


class VAEDecoder(_VAEBlocks):
    def __init__(self, params: Dict[str, torch.Tensor], config: VAEDecoderConfig = VAEDecoderConfig(), device=None):
        super().__init__(params, config, device)
        # the tensor-core conv wants Cin % 64 == 0 and Cout % 8 == 0: zero-pad the two odd layers once
        self.cin_pad = 64
        self.p["conv_in.weight"] = _pad_dim(self.p["conv_in.weight"], 3, self.cin_pad)
        self.cout_pad = 8
        self.p["conv_out.weight"] = _pad_dim(self.p["conv_out.weight"], 0, self.cout_pad)
        self.p["conv_out.bias"] = _pad_dim(self.p["conv_out.bias"], 0, self.cout_pad)
        # sub-pixel phase weights of conv3x3(nearest2x(.)) for the upsample stages (dk_conv_up_weights)
        self.up_w = {k[:-len(".weight")]: ops.conv_up_weights(v) for k, v in self.p.items()
                     if k.endswith(".upsample.weight")}
        self._shapes = ShapeCache()
        self.use_cuda_graphs, self.max_cached_shapes = default_settings()

    def _decode(self, x: torch.Tensor) -> torch.Tensor:
        h, st = self._conv(self._pad_channels(x, self.cin_pad), "conv_in")
        h, st = self._resnet(h, st, "mid_blocks.0")
        h, st = self._attention(h, st, "mid_blocks.1")
        h, st = self._resnet(h, st, "mid_blocks.2")
        n = len(self.config.block_out_channels)
        for j in reversed(range(n)):                                  # reversed(self.up_blocks) (vae.py:393)
            for l in range(self.config.layers_per_block):
                h, st = self._resnet(h, st, f"up_blocks.{j}.resnets.{l}")
            if f"up_blocks.{j}.upsample.weight" in self.p:
                h, st = self._conv(h, f"up_blocks.{j}.upsample", up=True)             # vae.py:146-147
        # conv_norm_out + SiLU + conv_out, 3 real output channels padded to 8.  Fused, this is one narrow output tile:
        # the input crosses L2 -> SM once instead of nine times (the nine-box implicit GEMM ran it at 0.9 TB/s)
        return self._conv(h, "conv_out", "conv_norm_out", st)[0]

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        """x (B, H, W, 16) NHWC -> (B, 8H, 8W, 3) NHWC view (channel stride 1, pixel stride 8)."""
        if x.dim() != 4:
            raise ValueError(f"VAEDecoder expects NHWC rank-4 input, got rank {x.dim()}")
        x = x.to(device=self.device, dtype=self.dtype).contiguous()
        st = self._shapes.state(tuple(x.shape), self.max_cached_shapes)
        y = self._shapes.run(st, self.use_cuda_graphs, self._decode, x)
        return y[..., : self.config.out_channels]


class VAEEncoder(_VAEBlocks):
    """reference VAEEncoder (vae.py:404-467).  Input: the uint8 image itself — read_image's `/255*2-1`
    (__init__.py:548-549) is fused into the channel-padding kernel.  The reference keeps the encoder in fp32
    (load_vae_encoder(float16=False), __init__.py:116); here it runs in the pipeline's 16-bit activation type with fp32
    accumulation (DESIGN.md §7)."""

    fuse = False            # the fused convolution would change the encoder's outputs: it keeps the unfused kernels

    def __init__(self, params: Dict[str, torch.Tensor], config: VAEEncoderConfig = VAEEncoderConfig(), device=None):
        super().__init__(params, config, device)
        self.cin_pad = 64
        self.p["conv_in.weight"] = _pad_dim(self.p["conv_in.weight"], 3, self.cin_pad)

    def encode_hidden(self, x16: torch.Tensor) -> torch.Tensor:
        """x16 (B, H, W, cin_pad) 16-bit NHWC in [-1, 1] -> hidden (B, H/8, W/8, 32) = (mean | logvar)"""
        h, st = self._conv(x16, "conv_in")
        n = len(self.config.block_out_channels)
        for i in range(n):
            for l in range(self.config.layers_per_block):
                h, st = self._resnet(h, st, f"down_blocks.{i}.resnets.{l}")
            if f"down_blocks.{i}.downsample.weight" in self.p:        # pad (0,1),(0,1) + stride 2 (vae.py:142-144)
                h = ops.conv3x3_s2(h, self.p[f"down_blocks.{i}.downsample.weight"],
                                   self.p[f"down_blocks.{i}.downsample.bias"])
                st = _Stats(h, self.groups)
        h, st = self._resnet(h, st, "mid_blocks.0")
        h, st = self._attention(h, st, "mid_blocks.1")
        h, st = self._resnet(h, st, "mid_blocks.2")
        return self._conv(h, "conv_out", "conv_norm_out", st)[0]

    def __call__(self, image: torch.Tensor) -> torch.Tensor:
        """image: uint8 NHWC (B, H, W, >=3) on the device, or a 16/32-bit float NHWC (B, H, W, 3) already in [-1, 1]."""
        if image.dim() != 4:
            raise ValueError(f"VAEEncoder expects NHWC rank-4 input, got rank {image.dim()}")
        if image.shape[1] % 8 or image.shape[2] % 8:
            raise ValueError(f"VAEEncoder: image size {tuple(image.shape[1:3])} must be a multiple of 8")
        image = image.to(self.device)
        if image.dtype == torch.uint8:
            x16 = ops.image_pre(image.contiguous(), self.dtype, self.cin_pad)
        else:
            x16 = torch.zeros((*image.shape[:3], self.cin_pad), dtype=self.dtype, device=self.device)
            x16[..., :3] = image[..., :3].to(self.dtype)
        return self.encode_hidden(x16)
