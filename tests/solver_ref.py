"""CPU restatement of the Heun and DPM-Solver++(2M) samplers (DESIGN.md §11) with oracle.sampler_ref.sample_euler's
signature and 16-bit conventions: the model sees the state cast to act_dtype, the timesteps are sigma * 1000 cast the
same way, D is the CFG-mixed calculate_denoised, and the state stays in the dtype of x (fp32, or fp64 for the exact-ODE
tests).  Kept beside the tests, like tests/step_cache_ref.py, so no file under oracle/ changes.

Written in textbook form (d, d2, D', expm1) and independent of diffusionkit_b200.sampler.dpmpp_2m_coefficients, which
the tests check against it."""
from __future__ import annotations

import math
from typing import Callable, Optional

import torch


def _denoiser(mmdit_call, x, conditioning, timestep, sigma, cfg_weight, cast):
    """CFGDenoiser.__call__ + calculate_denoised + the CFG mix, as oracle.sampler_ref.sample_euler inlines them"""
    xin = cast(x) if cfg_weight <= 0 else cast(torch.cat([x, x], dim=0))
    out = mmdit_call(xin, conditioning, timestep.reshape(1).repeat(xin.shape[0]))
    den = xin - out * sigma
    if cfg_weight > 0:
        den_text, den_neg = den.chunk(2, dim=0)
        den = den_neg + cfg_weight * (den_text - den_neg)
    return den


def _setup(cache_modulation, sigmas, pooled, act_dtype):
    def cast(t):
        return t if act_dtype is None else t.to(act_dtype).to(torch.float32)

    timesteps = cast(sigmas * 1000.0)
    cache_modulation(pooled, timesteps)
    return cast, timesteps


def sample_heun(
    mmdit_call: Callable[[torch.Tensor, torch.Tensor, torch.Tensor], torch.Tensor],
    cache_modulation: Callable[[torch.Tensor, torch.Tensor], None],
    x: torch.Tensor,
    sigmas: torch.Tensor,
    conditioning: torch.Tensor,
    pooled: torch.Tensor,
    cfg_weight: float,
    act_dtype: Optional[torch.dtype],
) -> torch.Tensor:
    """Karras et al. (2022), Algorithm 2 without churn: Euler predictor, trapezoidal corrector; Euler into sigma = 0"""
    cast, timesteps = _setup(cache_modulation, sigmas, pooled, act_dtype)
    for i in range(len(sigmas) - 1):
        sigma, sigma_next = float(sigmas[i]), float(sigmas[i + 1])
        den = _denoiser(mmdit_call, x, conditioning, timesteps[i], sigma, cfg_weight, cast)
        d = (x - den) / sigma
        x2 = x + d * (sigma_next - sigma)
        if sigma_next == 0:
            x = x2
            continue
        den2 = _denoiser(mmdit_call, x2, conditioning, timesteps[i + 1], sigma_next, cfg_weight, cast)
        d2 = (x2 - den2) / sigma_next
        x = x + (d + d2) / 2 * (sigma_next - sigma)
    return x


def _lambda(sigma: float) -> float:
    """log(alpha / sigma) with alpha = 1 - sigma: -inf at sigma = 1"""
    return -math.inf if sigma == 1.0 else math.log((1.0 - sigma) / sigma)


def sample_dpmpp_2m(
    mmdit_call: Callable[[torch.Tensor, torch.Tensor, torch.Tensor], torch.Tensor],
    cache_modulation: Callable[[torch.Tensor, torch.Tensor], None],
    x: torch.Tensor,
    sigmas: torch.Tensor,
    conditioning: torch.Tensor,
    pooled: torch.Tensor,
    cfg_weight: float,
    act_dtype: Optional[torch.dtype],
) -> torch.Tensor:
    """DPM-Solver++(2M), data prediction, alpha = 1 - sigma:
        x_{i+1} = (sigma_{i+1} / sigma_i) x_i - alpha_{i+1} expm1(-h_i) D',  h_i = lambda_{i+1} - lambda_i,
        D' = (1 + 1/(2r)) D_i - 1/(2r) D_{i-1}, r = h_{i-1} / h_i, or D' = D_i (first order) on the first step, after an
        interval with h = inf and on the last two steps; x_{i+1} = D_i when sigma_{i+1} = 0."""
    cast, timesteps = _setup(cache_modulation, sigmas, pooled, act_dtype)
    n = len(sigmas) - 1
    den_prev, h_prev = None, None
    for i in range(n):
        sigma, sigma_next = float(sigmas[i]), float(sigmas[i + 1])
        den = _denoiser(mmdit_call, x, conditioning, timesteps[i], sigma, cfg_weight, cast)
        if sigma_next == 0:
            x = den
            continue
        h = _lambda(sigma_next) - _lambda(sigma)
        if i >= 1 and math.isfinite(h_prev) and i < n - 2:
            r = h_prev / h
            den_d = (1 + 1 / (2 * r)) * den - (1 / (2 * r)) * den_prev
        else:
            den_d = den
        x = (sigma_next / sigma) * x - (1.0 - sigma_next) * math.expm1(-h) * den_d
        den_prev, h_prev = den, h
    return x
