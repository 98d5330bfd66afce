"""CPU restatement of masked inpainting (DESIGN.md §17): the mask preparation with plain loops, the per-step blend and
the paste-back, the five solvers with the blend after every full step, and the launch-census references of
inpaint.inpaint_blend and inpaint.inpaint_paste.  Independent of diffusionkit_b200.inpaint, which the tests check
against it.

Conventions are tests/solver_ref.py's and tests/sde_ref.py's: the model sees the state cast to act_dtype, the timesteps
are sigma * 1000 cast the same way, D is the CFG-mixed calculate_denoised, and the state stays in the dtype of x.  eps is
the seeded noise and x0 the encoded source (process_in space) of one image; mask is (H, W), nonzero = repaint."""
from __future__ import annotations

import math
from typing import Callable, Optional

import numpy as np
import torch


# ------------------------------------------------------------------------------------------------ the mask
def ref_binarise(gray: np.ndarray) -> np.ndarray:
    """uint8 (H, W) gray levels -> uint8 0/1, one pixel at a time: 1 where the level is 128 or more"""
    H, W = gray.shape
    out = np.zeros((H, W), dtype=np.uint8)
    for i in range(H):
        for j in range(W):
            out[i, j] = 1 if int(gray[i, j]) >= 128 else 0
    return out


def ref_latent_mask(pixels: np.ndarray) -> np.ndarray:
    """uint8 (Hp, Wp) 0/1 -> uint8 (Hp / 8, Wp / 8): a block is 1 when any of its 64 pixels is"""
    Hp, Wp = pixels.shape
    out = np.zeros((Hp // 8, Wp // 8), dtype=np.uint8)
    for i in range(Hp):
        for j in range(Wp):
            if pixels[i, j]:
                out[i // 8, j // 8] = 1
    return out


def ref_prepare(gray_image, size) -> tuple:
    """a PIL "L" image of the source's size (W, H) -> (pixel mask, latent mask): resized with the source's rule (LANCZOS
    down to multiples of 64 when a side is not one), then ref_binarise and ref_latent_mask"""
    from PIL import Image

    assert gray_image.mode == "L" and gray_image.size == tuple(size)
    W, H = (d - d % 64 for d in size)
    if (W, H) != tuple(size):
        gray_image = gray_image.resize((W, H), Image.LANCZOS)
    pixels = ref_binarise(np.asarray(gray_image))
    return pixels, ref_latent_mask(pixels)


# ------------------------------------------------------------------------------------------------ blend and paste
def ref_blend(x, eps, x0, mask, a: float, b: float):
    """fp64: x where mask != 0, else a eps + b x0; x, eps, x0 (B, H, W, C), mask (H, W)"""
    keep = (mask == 0).reshape(1, mask.shape[0], mask.shape[1], 1).to(x.device)
    return torch.where(keep, a * eps.double() + b * x0.double(), x.double())


def ref_paste(img, src, mask):
    """uint8: src where mask == 0, else img; img (B, Hp, Wp, 3), src (Hp, Wp, 3), mask (Hp, Wp)"""
    keep = (mask == 0).reshape(1, mask.shape[0], mask.shape[1], 1).to(img.device)
    return torch.where(keep, src.to(img.device).unsqueeze(0), img)


# ------------------------------------------------------------------------------------------------ samplers
SOLVERS = ("euler", "heun", "dpmpp_2m", "euler_ancestral", "dpmpp_2m_sde")


def sample(solver: str, den: Callable[[torch.Tensor, int, int], torch.Tensor], x: torch.Tensor, sigmas, eps, x0,
           mask, *, seed: int = 0, eta: float = 1.0) -> torch.Tensor:
    """one image (x (1, H, W, 16), the img2img start) through `solver`, the kept positions reset to
    sigma_{i+1} eps + (1 - sigma_{i+1}) x0 after every full step.  den(x, k, i): the denoised estimate at sigma_k of
    solver step i.  Heun's predictor and 2M's stored D are not blended."""
    from tests import sde_ref
    from tests.solver_ref import _lambda

    sig = [float(v) for v in sigmas]
    keep = (torch.as_tensor(mask) == 0).reshape(1, mask.shape[0], mask.shape[1], 1)

    def blend(x, s):
        return torch.where(keep, s * eps + (1.0 - s) * x0, x)

    n = len(sig) - 1
    coef = sde_ref.coefficients(solver, sigmas, eta) if solver in ("euler_ancestral", "dpmpp_2m_sde") else None
    den_prev = h_prev = None
    for i in range(n):
        s, nxt = sig[i], sig[i + 1]
        D = den(x, i, i)
        if solver == "euler" or (solver == "heun" and nxt == 0.0):
            x = x + (x - D) / s * (nxt - s)
        elif solver == "heun":
            d = (x - D) / s
            x2 = x + d * (nxt - s)
            d2 = (x2 - den(x2, i + 1, i)) / nxt
            x = x + (d + d2) / 2 * (nxt - s)
        elif solver == "dpmpp_2m":
            if nxt == 0.0:
                x = D
            else:
                h = _lambda(nxt) - _lambda(s)
                if i >= 1 and math.isfinite(h_prev) and i < n - 2:
                    r = h_prev / h
                    den_d = (1 + 1 / (2 * r)) * D - (1 / (2 * r)) * den_prev
                else:
                    den_d = D
                x = (nxt / s) * x - (1.0 - nxt) * math.expm1(-h) * den_d
                h_prev = h
        else:
            a, b, c, nz = coef[i]
            z = (torch.from_numpy(sde_ref.normals(seed, i, x.numel())).reshape(x.shape).to(x.dtype)
                 if nz != 0.0 else 0.0)
            x = a * x + b * D + (c * den_prev if c != 0.0 else 0.0) + nz * z
        den_prev = D
        x = blend(x, nxt)
    return x


def sample_model(solver: str, mmdit_call, cache_modulation, x, sigmas, conditioning, pooled, cfg_weight: float,
                 act_dtype: Optional[torch.dtype], *, eps, x0, mask, seed: int = 0, eta: float = 1.0):
    """an oracle MMDiT (tests/solver_ref.sample_heun's arguments) through sample()"""
    from tests.solver_ref import _denoiser, _setup

    cast, timesteps = _setup(cache_modulation, sigmas, pooled, act_dtype)
    sig = [float(v) for v in sigmas]
    return sample(solver, lambda xx, k, i: _denoiser(mmdit_call, xx, conditioning, timesteps[k], sig[k], cfg_weight,
                                                      cast), x, sigmas, eps, x0, mask, seed=seed, eta=eta)


def sample_slg(solver: str, model, x, sigmas, conditioning, pooled, cfg_weight: float,
               act_dtype: Optional[torch.dtype], *, eps, x0, mask, seed: int = 0, eta: float = 1.0, scale: float = 0.0,
               layers=(), start: float = 0.0, end: float = 0.0):
    """an SD3.5-medium oracle model (tests/sd35_medium_ref.MMDiTXRef) under CFG with skip-layer guidance; both Heun
    evaluations of a step take its decision"""
    from tests.sd35_medium_ref import slg_denoiser, slg_window

    def cast(t):
        return t if act_dtype is None else t.to(act_dtype).to(torch.float32)

    timesteps = cast(sigmas * 1000.0)
    model.cache_modulation_params(pooled, timesteps)
    window = set(slg_window(len(sigmas) - 1, start, end))
    sig = [float(v) for v in sigmas]
    return sample(solver, lambda xx, k, i: slg_denoiser(model, xx, conditioning, timesteps[k], sig[k], cfg_weight, cast,
                                                         scale, layers, i in window),
                  x, sigmas, eps, x0, mask, seed=seed, eta=eta)


# ------------------------------------------------------------------------------------------------ census checks
def census_check_blend(L, a, s, r, census):
    """tests/launch_parity check of one inpaint.inpaint_blend launch: the kept positions within fp32 rounding of the
    fp64 reference, the repainted ones bit for bit unchanged"""
    from tests import launch_parity as lp

    mask = s["mask"]
    L.close("x", r, ref_blend(s["x"], s["eps"], s["x0"], mask, a["a"], a["b"]), lp.TOL_F32)
    rep = (mask != 0).reshape(1, mask.shape[0], mask.shape[1], 1).expand_as(r)
    L.exact("repainted", r[rep], s["x"][rep])
    L.own(r)
    L.sig.update(B=r.shape[0], HW=mask.numel(), C=r.shape[3], repainted=round(float((mask != 0).float().mean()), 3),
                 dtype="float32")


def census_check_paste(L, a, s, r, census):
    """tests/launch_parity check of one inpaint.inpaint_paste launch, bit for bit"""
    L.exact("img", r, ref_paste(s["img"], s["src"], s["mask"]))
    L.own(r)
    L.sig.update(B=r.shape[0], pixels=s["mask"].numel(), dtype="uint8")
