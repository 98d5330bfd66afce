"""Masked inpainting (DESIGN.md §17): the host-side mask preparation and the two launches it adds to a denoise.

A mask marks the pixels to regenerate (white, >= 128 after a grayscale conversion).  A latent position is repainted
when any pixel of its 8 x 8 block is marked.  After every solver step to sigma, the kept positions are reset to the
re-noised source sigma * eps + (1 - sigma) * x0 (inpaint_blend), so the last step, to sigma = 0, leaves them at x0
exactly; after the decode, every kept pixel is replaced by the source pixel (inpaint_paste).

inpaint_blend and inpaint_paste live here beside their callers rather than in ops: the launch census of the shipped
models requires a reference for every launching op there, and these run only with a mask, whose GPU test runs a census
of its own that wraps them (as pipeline.sampler_sde_step and image_encoders.image_patches do).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Tuple

import numpy as np
import torch

from . import ops
from ._lib import ptr

# a mask pixel at or above this gray level is repainted
THRESHOLD = 128


@dataclass(frozen=True)
class InpaintMask:
    """a prepared mask: `pixels` uint8 (Hp, Wp) and `latent` uint8 (Hp / 8, Wp / 8), 1 = repaint, 0 = keep"""
    pixels: np.ndarray
    latent: np.ndarray

    @property
    def masked_fraction(self) -> float:
        """the fraction of latent positions that are repainted"""
        return float(self.latent.mean())


def _mask_image(mask_image):
    """a path, a PIL image or a uint8 (H, W) / (H, W, 1|3|4) array -> a PIL image; ValueError for anything else"""
    from PIL import Image, UnidentifiedImageError

    if isinstance(mask_image, (str, bytes)) or hasattr(mask_image, "__fspath__"):
        try:
            im = Image.open(mask_image)
            im.load()
        except (OSError, UnidentifiedImageError) as e:
            raise ValueError(f"mask_image {mask_image!r} cannot be read: {e}") from None
        return im
    if isinstance(mask_image, np.ndarray):
        a = mask_image
        if a.dtype != np.uint8 or not (a.ndim == 2 or (a.ndim == 3 and a.shape[2] in (1, 3, 4))):
            raise ValueError(f"mask_image array must be uint8 (H, W) or (H, W, 1|3|4), got {a.dtype} {a.shape}")
        return Image.fromarray(np.ascontiguousarray(a[:, :, 0] if a.ndim == 3 and a.shape[2] == 1 else a))
    if isinstance(mask_image, Image.Image):
        return mask_image
    raise ValueError(f"mask_image must be a path, a PIL image or a uint8 array, got {type(mask_image).__name__}")


def prepare_mask(mask_image, source_size: Tuple[int, int]) -> InpaintMask:
    """The mask of one call.  source_size: (width, height) of the source image as given.  The mask must have that
    size; it is converted to grayscale (PIL "L"), resized like the source (LANCZOS down to multiples of 64, only when a
    side is not one already), binarised (>= THRESHOLD: repaint) and reduced to the latent grid: a latent position is
    repainted when any pixel of its 8 x 8 block is (diffusers samples one pixel per block, which can drop a stroke
    thinner than 8 pixels).  Raises ValueError, before any GPU work, for a mask the pipeline cannot take."""
    from PIL import Image

    im = _mask_image(mask_image).convert("L")
    if (im.width, im.height) != tuple(source_size):
        raise ValueError(f"mask_image is {im.width}x{im.height}, the source image {source_size[0]}x{source_size[1]}: "
                         "they must have the same size")
    W, H = (d - d % 64 for d in (im.width, im.height))
    if W == 0 or H == 0:
        raise ValueError(f"mask_image {im.width}x{im.height} is smaller than 64x64")
    if (W, H) != (im.width, im.height):
        im = im.resize((W, H), Image.LANCZOS)
    pixels = (np.asarray(im) >= THRESHOLD).astype(np.uint8)
    return InpaintMask(np.ascontiguousarray(pixels), latent_mask(pixels))


def latent_mask(pixels: np.ndarray) -> np.ndarray:
    """uint8 (Hp, Wp) 0/1, sides multiples of 8 -> uint8 (Hp / 8, Wp / 8): 1 where any pixel of the 8 x 8 block is 1"""
    Hp, Wp = pixels.shape
    return np.ascontiguousarray(pixels.reshape(Hp // 8, 8, Wp // 8, 8).any(axis=(1, 3)).astype(np.uint8))


def inpaint_blend(x, eps, x0, mask, a: float, b: float):
    """dk_inpaint_blend: x[:, p] = a * eps[:, p] + b * x0[:, p] (in place) at every position p with mask[p] == 0; the
    others keep their bits.  x, eps, x0 fp32 (B, H, W, C) contiguous, C % 4 == 0; mask uint8 (H, W) on the device."""
    assert x.dtype == eps.dtype == x0.dtype == torch.float32 and x.shape == eps.shape == x0.shape and x.dim() == 4
    assert x.is_contiguous() and eps.is_contiguous() and x0.is_contiguous() and mask.is_contiguous()
    B, H, W, C = x.shape
    assert mask.dtype == torch.uint8 and tuple(mask.shape) == (H, W) and mask.device == x.device
    c = ops.ctx(x.device.index)
    c.call("dk_inpaint_blend", ptr(x), ptr(eps), ptr(x0), ptr(mask), B, H * W, C, a, b)
    return x


def inpaint_paste(img, src, mask):
    """dk_inpaint_paste: img[:, p] = src[p] (in place) at every pixel p with mask[p] == 0.  img uint8 (B, Hp, Wp, 3),
    src uint8 (Hp, Wp, 3), mask uint8 (Hp, Wp), all contiguous on one device."""
    assert img.dtype == src.dtype == mask.dtype == torch.uint8 and img.dim() == 4 and img.shape[3] == 3
    B, Hp, Wp, _ = img.shape
    assert tuple(src.shape) == (Hp, Wp, 3) and tuple(mask.shape) == (Hp, Wp)
    assert img.is_contiguous() and src.is_contiguous() and mask.is_contiguous()
    assert src.device == img.device == mask.device
    c = ops.ctx(img.device.index)
    c.call("dk_inpaint_paste", ptr(img), ptr(src), ptr(mask), B, Hp * Wp)
    return img


class InpaintBlend:
    """the sampler-side state of one masked denoise: the seeded noise eps, the encoded source x0 (both (B, H, W, 16)
    fp32 in the process_in space) and the latent mask on the device.  CFGDenoiser calls blend after every solver step."""

    def __init__(self, eps: torch.Tensor, x0: torch.Tensor, mask: torch.Tensor):
        self.eps, self.x0, self.mask = eps, x0, mask

    def blend(self, x, sigma_next: float):
        """x <- mask ? x : sigma_next * eps + (1 - sigma_next) * x0, the coefficients as img2img's start forms them"""
        s = float(sigma_next)
        inpaint_blend(x, self.eps, self.x0, self.mask, s, 1.0 - s)
