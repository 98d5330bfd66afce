"""FLUX.1 Canny [dev] and FLUX.1 Depth [dev] (DESIGN.md §19): the control image's 64 columns of the model's x-embedder
input, built once per call on the GPU.

Every token of these models is [x (64) | control latent (64)].  The control latent is the VAE encoder's posterior
mean of the control image, process_in, rounded to the model dtype and packed like the target latent.  The control
image is, on a Canny model, cv2.Canny(img, 50, 200) of the RGB image after BFL's float round trip
((u8 / 127.5 - 1 + 1) * 127.5 truncated to uint8, ROUNDTRIP below), and on a Depth model the depth map the user gives.
MMDiT.cache_fill_conditioning turns the 64 columns into the x-embedder's per-call term, as for FLUX.1 Fill.

canny lives here beside its caller rather than in ops: the launch census of the shipped models requires a reference
for every launching op there, and it runs only for a Canny model, whose GPU test runs a census of its own that wraps it.
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np
import torch

from . import ops
from ._lib import ptr

KINDS = ("canny", "depth")
# BFL's cli_control guidance when the caller passes none
DEFAULT_GUIDANCE = {"canny": 30.0, "depth": 10.0}
# BFL's CannyImageEncoder: cv2.Canny(img, 50, 200)
DEFAULT_THRESHOLDS = (50, 200)
WS_BYTES_PER_PIXEL = 10                                   # DK_CANNY_WS_BYTES_PER_PIXEL
# latent columns per token of the control image (16 channels x 2 x 2)
LATENT_CHANNELS = 64


def _roundtrip() -> np.ndarray:
    """BFL's CannyImageEncoder input: the image arrives as u8 / 127.5 - 1 in fp32 and goes back to uint8 as
    ((x + 1) * 127.5).astype(uint8), which truncates; evaluated for every byte value in torch fp32"""
    x = torch.arange(256, dtype=torch.float32) / 127.5 - 1.0
    return ((x + 1.0) * 127.5).to(torch.uint8).numpy()


# value -> value after the round trip (1 .. 63 lose one, every other value is kept)
ROUNDTRIP = _roundtrip()
_luts = {}


def canny(img_u8: torch.Tensor, low: int = DEFAULT_THRESHOLDS[0], high: int = DEFAULT_THRESHOLDS[1],
          lut: Optional[torch.Tensor] = None) -> torch.Tensor:
    """dk_canny: uint8 (H, W, >=3) image on the device -> uint8 (H, W, 3) edges, 255 / 0 in every channel:
    cv2.Canny(lut[img], low, high).  lut: uint8 (256,) on the device, None for BFL's round trip ROUNDTRIP."""
    assert img_u8.dtype == torch.uint8 and img_u8.dim() == 3 and img_u8.is_contiguous()
    H, W, C = img_u8.shape
    dev = img_u8.device
    if lut is None:
        lut = _luts.get(dev)
        if lut is None:
            lut = _luts[dev] = torch.from_numpy(ROUNDTRIP).to(dev)
    assert lut.dtype == torch.uint8 and tuple(lut.shape) == (256,) and lut.device == dev
    out = torch.empty((H, W, 3), dtype=torch.uint8, device=dev)
    ws = torch.empty(WS_BYTES_PER_PIXEL * H * W, dtype=torch.uint8, device=dev)
    c = ops.ctx(dev.index)
    c.call("dk_canny", ptr(img_u8), ptr(lut), ptr(out), ptr(ws), H, W, C, int(low), int(high))
    return out


def check_thresholds(thresholds) -> Optional[Tuple[int, int]]:
    """canny_thresholds as the pipeline takes it -> None (the image is already an edge map) or (low, high) ints;
    ValueError for anything else"""
    if thresholds is None:
        return None
    try:
        low, high = thresholds
    except (TypeError, ValueError):
        raise ValueError(f"canny_thresholds must be (low, high) or None, got {thresholds!r}") from None
    if not all(isinstance(v, (int, np.integer)) and not isinstance(v, bool) for v in (low, high)):
        raise ValueError(f"canny_thresholds must be integers, got {thresholds!r}")
    if not 0 <= low <= high:
        raise ValueError(f"canny_thresholds must satisfy 0 <= low <= high, got {thresholds!r}")
    return int(low), int(high)


def load_control_image(image, size: Optional[Tuple[int, int]]) -> np.ndarray:
    """a path, a PIL image or a uint8 (H, W) / (H, W, 1|3|4) array -> uint8 (height, width, 3) RGB resized with PIL
    LANCZOS to exactly size = (width, height), aspect ratio not kept (BFL's prepare_control; None keeps the image's
    size); ValueError for an input that is none of these"""
    from PIL import Image

    if isinstance(image, (str, bytes)) or hasattr(image, "__fspath__"):
        try:
            image = Image.open(image)
            image.load()
        except OSError as e:
            raise ValueError(f"control_image could not be read: {e}") from None
    if isinstance(image, np.ndarray):
        if image.dtype != np.uint8 or not (image.ndim == 2 or (image.ndim == 3 and image.shape[2] in (1, 3, 4))):
            raise ValueError(f"control_image array must be uint8 (H, W) or (H, W, 1|3|4), got {image.dtype} "
                             f"{image.shape}")
        image = Image.fromarray(image[:, :, 0] if image.ndim == 3 and image.shape[2] == 1 else image)
    if not isinstance(image, Image.Image):
        raise ValueError(f"control_image must be a path, a PIL image or a uint8 array, got {type(image).__name__}")
    image = image.convert("RGB")
    if size is not None and image.size != tuple(size):
        image = image.resize(tuple(size), Image.LANCZOS)
    return np.array(image)


def control_rows(encoder, image_u8: torch.Tensor, kind: str, shift: float, scale: float, dtype,
                 thresholds: Optional[Tuple[int, int]] = DEFAULT_THRESHOLDS) -> torch.Tensor:
    """the (N, 64) control rows of one control image: image_u8 uint8 (H, W, 3) on the device, or the float (H, W, 3)
    image in [-1, 1] the VAE encoder also takes (FLUX.1 Depth's estimated depth, DESIGN.md §20), N = (H / 16)(W / 16).
    kind "canny" with thresholds runs canny first (thresholds None: the image is already an edge map); the image is
    encoded once into its posterior mean (seed-independent; BFL samples the posterior), then (mean - shift) * scale,
    rounded to dtype and packed like the target latent."""
    if kind not in KINDS:
        raise ValueError(f"control kind must be one of {KINDS}, got {kind!r}")
    if kind == "canny" and thresholds is not None:
        image_u8 = canny(image_u8, *thresholds)
    hidden = encoder(image_u8.unsqueeze(0))                               # (1, H/8, W/8, 32) = (mean | logvar)
    zero = torch.zeros(tuple(hidden.shape[:3]) + (hidden.shape[3] // 2,), dtype=torch.float32, device=hidden.device)
    lat16 = ops.cast_to_16(ops.vae_sample_latent(hidden, zero, shift, scale), dtype)
    return ops.patchify(lat16, 0)
