"""CPU statement of FLUX.1 Canny [dev] and FLUX.1 Depth [dev]'s input convention (DESIGN.md §19): BFL's
prepare_control, CannyImageEncoder and Flux.forward, on top of tests/fill_ref.py's forward with the concatenated
x-embedder, so no file under oracle/ changes.

- roundtrip_table: BFL's CannyImageEncoder receives the image as u8 / 127.5 - 1 in fp32 and converts it back with
  ((x + 1) * 127.5).astype(uint8), which truncates;
- canny: cv2.Canny(img, low, high) of OpenCV 4.x with the L1 gradient, stated in numpy (pinned against cv2 outputs in
  tests/golden/canny_cv2.npz and, where cv2 imports, against live cv2.Canny);
- the control rows: the control image encoded into its posterior mean, process_in, rounded to the model dtype and
  packed "b c (h ph) (w pw) -> b (h w) (c ph pw)";
- pipeline drivers and the launch-census reference of control.canny."""
from __future__ import annotations

import numpy as np
import torch
from scipy import ndimage

from oracle.mmdit_ref import _r
from tests.fill_ref import bfl_pack_latent


# ------------------------------------------------------------------------------------------------ Canny
def roundtrip_table() -> np.ndarray:
    """(256,) uint8: BFL's u8 -> fp32 [-1, 1] -> uint8 round trip of every byte value, in numpy fp32"""
    x = np.arange(256, dtype=np.uint8).astype(np.float32) / np.float32(127.5) - np.float32(1.0)
    return ((x + np.float32(1.0)) * np.float32(127.5)).astype(np.uint8)


def canny(img, low: int = 50, high: int = 200) -> np.ndarray:
    """cv2.Canny(img, low, high) of a uint8 (H, W) or (H, W, C) image (every channel takes part) -> uint8 (H, W) 0/255.
    1. 3 x 3 Sobel dx, dy per channel in integers, replicated borders; magnitude |dx| + |dy|;
    2. per pixel the channel of largest magnitude, the first on a tie;
    3. non-maximum suppression with magnitude 0 outside the image: x = |dx|, y = |dy| << 15, tg22x = 13573 x;
       y < tg22x: horizontal, keep if m > left and m >= right; y > tg22x + (x << 16): vertical, keep if m > up and
       m >= down; otherwise diagonal with s = -1 if dx ^ dy < 0 else 1: keep if m > mag[up][j - s] and
       m > mag[down][j + s];
    4. a kept pixel is a candidate when m > low, strong when m > high;
    5. output 255 for every candidate in an 8-connected component of candidates that holds a strong pixel."""
    img = np.asarray(img).astype(np.int32)
    if img.ndim == 2:
        img = img[..., None]
    p = np.pad(img, ((1, 1), (1, 1), (0, 0)), mode="edge")
    H, W = img.shape[:2]

    def s(dy, dx):
        return p[1 + dy:1 + dy + H, 1 + dx:1 + dx + W]

    dx = (s(-1, 1) + 2 * s(0, 1) + s(1, 1)) - (s(-1, -1) + 2 * s(0, -1) + s(1, -1))
    dy = (s(1, -1) + 2 * s(1, 0) + s(1, 1)) - (s(-1, -1) + 2 * s(-1, 0) + s(-1, 1))
    mag = np.abs(dx) + np.abs(dy)
    k = np.argmax(mag, axis=2)[..., None]                     # argmax returns the first maximum
    dx, dy, mag = (np.take_along_axis(a, k, 2)[..., 0] for a in (dx, dy, mag))
    M = np.pad(mag, 1)

    def m(oy, ox):
        return M[1 + oy:1 + oy + H, 1 + ox:1 + ox + W]

    x = np.abs(dx).astype(np.int64)
    y = np.abs(dy).astype(np.int64) << 15
    tg22x = x * 13573
    horiz = y < tg22x
    vert = ~horiz & (y > tg22x + (x << 16))
    diag = ~horiz & ~vert
    sgn = np.where((dx ^ dy) < 0, -1, 1)
    keep = horiz & (mag > m(0, -1)) & (mag >= m(0, 1))
    keep |= vert & (mag > m(-1, 0)) & (mag >= m(1, 0))
    keep |= diag & (sgn == 1) & (mag > m(-1, -1)) & (mag > m(1, 1))
    keep |= diag & (sgn == -1) & (mag > m(-1, 1)) & (mag > m(1, -1))
    cand = keep & (mag > low)
    strong = cand & (mag > high)
    lab, n = ndimage.label(cand, structure=np.ones((3, 3)))
    good = np.zeros(n + 1, bool)
    good[np.unique(lab[strong])] = True
    good[0] = False
    return (good[lab] * 255).astype(np.uint8)


def spiral(H: int, W: int, pitch: float = 7.0) -> np.ndarray:
    """uint8 (H, W) grey test image: a one-pixel Archimedean spiral on a flat background whose contrast falls from 60
    at the centre to 16 at the outside, so only its inner part is strong for (50, 200) and hysteresis alone carries
    the edge along the rest"""
    img = np.full((H, W), 100, dtype=np.int32)
    rmax = min(H, W) / 2 - 3
    n = int(8 * np.pi * (rmax / pitch) * rmax) + 16
    theta = np.linspace(0.0, 2 * np.pi * rmax / pitch, n)
    r = pitch * theta / (2 * np.pi)
    ys = np.round(H / 2 + r * np.sin(theta)).astype(int)
    xs = np.round(W / 2 + r * np.cos(theta)).astype(int)
    img[ys, xs] = 100 + np.round(60 - 44 * np.linspace(0.0, 1.0, n)).astype(int)
    return img.astype(np.uint8)


def canny_control(img_u8, thresholds=(50, 200)) -> np.ndarray:
    """BFL's Canny control image of a uint8 (H, W, >=3) RGB image: the round trip, cv2.Canny, 3 channels -> (H, W, 3)"""
    img = roundtrip_table()[np.asarray(img_u8)[..., :3]]
    return np.repeat(canny(img, *thresholds)[..., None], 3, axis=2)


# ------------------------------------------------------------------------------------------------ control rows
def loop_pack(lat: np.ndarray) -> np.ndarray:
    """(H, W, 16) -> ((H/2)(W/2), 64) one element at a time: token (h, w), column c * 4 + ph * 2 + pw holds
    lat[2h + ph, 2w + pw, c]"""
    H, W, C = lat.shape
    out = np.zeros(((H // 2) * (W // 2), 4 * C), dtype=lat.dtype)
    for h in range(H // 2):
        for w in range(W // 2):
            for c in range(C):
                for ph in range(2):
                    for pw in range(2):
                        out[h * (W // 2) + w, c * 4 + ph * 2 + pw] = lat[2 * h + ph, 2 * w + pw, c]
    return out


def oracle_control_rows(enc, control_u8, kind: str, shift: float, scale: float, dtype, thresholds=(50, 200)):
    """the whole conditioning in the oracle: the control image (Canny: canny_control unless thresholds is None) as
    u8 / 255 * 2 - 1 through an oracle.vae_ref.VAEEncoderRef, its posterior mean, (mean - shift) * scale rounded to
    dtype and packed -> (N, 64) fp32 holding dtype values"""
    img = np.asarray(control_u8)[..., :3]
    if kind == "canny" and thresholds is not None:
        img = canny_control(img, thresholds)
    x = torch.from_numpy(np.ascontiguousarray(img)).float()[None] / 255 * 2 - 1.0
    hidden = enc(x)
    mean = hidden[..., :hidden.shape[-1] // 2]
    return bfl_pack_latent(_r((mean - shift) * scale, dtype))[0]


# ------------------------------------------------------------------------------------------------ census check
def census_check_canny(L, a, s, r, census):
    """tests/launch_parity check of one control.canny launch (five kernels), bit for bit"""
    img = s["img_u8"].cpu().numpy()
    lut = roundtrip_table() if s.get("lut") is None else s["lut"].cpu().numpy()
    want = np.repeat(canny(lut[img[..., :3]], a["low"], a["high"])[..., None], 3, axis=2)
    L.exact("edges", r, torch.from_numpy(want).to(r.device))
    L.own(r)
    L.sig.update(H=r.shape[0], W=r.shape[1], low=a["low"], high=a["high"],
                 edges=round(float((r != 0).float().mean()), 3), dtype="uint8")
