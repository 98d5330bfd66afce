"""FLUX.1 Fill [dev] (DESIGN.md §18): the masked-image and mask channels of the model's x-embedder input, built once
per call on the GPU.

For a source image src (uint8, sides multiples of 64) and its binarised pixel mask m (1 = repaint):
  img_cond = (src / 255 * 2 - 1) * (1 - m), encoded by the VAE encoder into its posterior mean, process_in, and
             packed like the target latent: 64 columns per token;
  mask     = 256 columns per token, BFL's rearrange(m, "b (h ph1) (w pw1) -> b (ph1 pw1) h w", ph1=8, pw1=8) then
             "b c (h ph) (w pw) -> b (h w) (c ph pw)", ph=pw=2;
and every token of the model input is [x (64) | img_cond (64) | mask (256)].  MMDiT.cache_fill_conditioning turns the
320 conditioning columns into the x-embedder's per-call term.

image_pre_masked and fill_cond_rows live here beside their caller rather than in ops: the launch census of the shipped
models requires a reference for every launching op there, and these run only for a Fill model, whose GPU test runs a
census of its own that wraps them (as inpaint.inpaint_blend does).
"""
from __future__ import annotations

import torch

from . import ops
from ._lib import dtype_code, ptr

# conditioning columns per token: the packed masked-image latent, then the 8 x 8 x 2 x 2 mask pixels
LATENT_CHANNELS, MASK_CHANNELS = 64, 256
COND_CHANNELS = LATENT_CHANNELS + MASK_CHANNELS

# FLUX.1 Fill's distilled guidance when the caller passes none (BFL's Fill default)
DEFAULT_GUIDANCE = 30.0


def image_pre_masked(img_u8, mask, dtype, cpad: int = 64):
    """dk_image_pre_masked: uint8 (1, H, W, >=3) image and uint8 (H, W) mask on the device -> 16-bit (1, H, W, cpad),
    dk_image_pre's values at kept pixels and 0 at every pixel whose mask byte is nonzero"""
    assert img_u8.dtype == mask.dtype == torch.uint8 and img_u8.dim() == 4 and img_u8.shape[0] == 1
    assert img_u8.is_contiguous() and mask.is_contiguous() and img_u8.device == mask.device
    _, H, W, Cs = img_u8.shape
    assert tuple(mask.shape) == (H, W)
    out = torch.empty((1, H, W, cpad), dtype=dtype, device=img_u8.device)
    c = ops.ctx(img_u8.device.index)
    c.call("dk_image_pre_masked", dtype_code(dtype), ptr(img_u8), ptr(mask), ptr(out), H, W, Cs, cpad)
    return out


def fill_cond_rows(lat_rows, mask, out=None):
    """dk_fill_cond_rows: the packed masked-image latent rows (N, 64) 16-bit and the uint8 (H, W) pixel mask,
    N = (H / 16)(W / 16) -> (N, 320) [latent | mask channels] in the latent rows' dtype"""
    H, W = mask.shape
    N = (H // 16) * (W // 16)
    assert mask.dtype == torch.uint8 and mask.is_contiguous() and lat_rows.is_contiguous()
    assert tuple(lat_rows.shape) == (N, LATENT_CHANNELS) and lat_rows.device == mask.device
    if out is None:
        out = torch.empty((N, COND_CHANNELS), dtype=lat_rows.dtype, device=lat_rows.device)
    assert tuple(out.shape) == (N, COND_CHANNELS) and out.is_contiguous() and out.dtype == lat_rows.dtype
    c = ops.ctx(lat_rows.device.index)
    c.call("dk_fill_cond_rows", dtype_code(lat_rows.dtype), ptr(lat_rows), ptr(mask), ptr(out), H, W)
    return out


def conditioning_rows(encoder, src_u8: torch.Tensor, mask: torch.Tensor, shift: float, scale: float, dtype):
    """the (N, 320) conditioning rows of one source: src_u8 uint8 (1, H, W, >=3) and mask uint8 (H, W) 0/1 on the
    device.  The masked image is encoded once and represented by its posterior mean (seed-independent; BFL samples the
    posterior), then (mean - shift) * scale, rounded to the model dtype and packed like the target latent."""
    hidden = encoder(src_u8, mask=mask)                                  # (1, H/8, W/8, 32) = (mean | logvar)
    zero = torch.zeros(tuple(hidden.shape[:3]) + (hidden.shape[3] // 2,), dtype=torch.float32, device=hidden.device)
    lat16 = ops.cast_to_16(ops.vae_sample_latent(hidden, zero, shift, scale), dtype)
    return fill_cond_rows(ops.patchify(lat16, 0), mask)
