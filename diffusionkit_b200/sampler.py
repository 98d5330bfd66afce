"""Sampler schedules — same classes and methods as the reference (python/src/diffusionkit/mlx/sampler.py:10-77).

Host-side scalar arithmetic (numpy fp32, like the reference's fp32 mx arrays); the per-step tensor math runs in the
fused CUDA sampler kernels (csrc/elementwise.cu: dk_sampler_prepare / dk_sampler_step, and the Heun and
DPM-Solver++(2M) updates, whose fp64 coefficients dpmpp_2m_coefficients computes, and the stochastic samplers' update
dk_sampler_sde_step, whose coefficients euler_ancestral_coefficients / dpmpp_2m_sde_coefficients compute).
"""
import math
from dataclasses import dataclass
from typing import List, Tuple

import numpy as np


class ModelSamplingDiscreteFlow:
    """Helper for sampler scheduling (timestep/sigma calculations) for Discrete Flow models (sampler.py:10-42)."""

    _t_first = 1

    def __init__(self, shift=1.0):
        self.shift = shift
        timesteps = 1000
        self.sigmas = self.sigma(np.arange(self._t_first, timesteps + 1, 1, dtype=np.float32))

    @property
    def sigma_min(self):
        return self.sigmas[0]

    @property
    def sigma_max(self):
        return self.sigmas[-1]

    def timestep(self, sigma):
        return sigma * np.float32(1000)

    def sigma(self, timestep):
        timestep = np.asarray(timestep, dtype=np.float32) / np.float32(1000.0)
        if self.shift == 1.0:
            return timestep
        s = np.float32(self.shift)
        return s * timestep / (np.float32(1) + (s - np.float32(1)) * timestep)

    def calculate_denoised(self, sigma, model_output, model_input):
        # tensor form lives in dk_sampler_step; this scalar/array form is kept for API parity (sampler.py:37-39)
        return model_input - model_output * sigma

    def noise_scaling(self, sigma, noise, latent_image, max_denoise=False):
        return sigma * noise + (1.0 - sigma) * latent_image


class FluxSampler(ModelSamplingDiscreteFlow):
    """Helper for sampler scheduling for Flux models (sampler.py:45-77): table over t = 0..1000."""

    _t_first = 0


def flux_resolution_shift(latent_size, base_shift: float = 0.5, max_shift: float = 1.15) -> float:
    """exp(mu) of BFL's resolution-dependent FLUX.1-dev schedule, for FluxSampler(shift=...) / FluxPipeline(shift=...).
    mu is linear in the image token count n = (H/2)·(W/2) of the latent (H, W): base_shift at 256 tokens, max_shift at
    4096.  BFL applies time_shift(mu, 1, t) = e^mu / (e^mu + 1/t - 1) to t on linspace(1, 0, steps + 1); FluxSampler
    with shift = e^mu gives the same sigmas.  1024^2 (latent 128^2): 3.1582."""
    H, W = (int(s) for s in latent_size)
    if H < 2 or W < 2:
        raise ValueError(f"latent_size must be at least (2, 2), got {tuple(latent_size)}")
    n = (H // 2) * (W // 2)
    mu = base_shift + (max_shift - base_shift) * (n - 256) / (4096 - 256)
    return math.exp(mu)


def dpmpp_2m_coefficients(sigmas) -> np.ndarray:
    """DPM-Solver++(2M) (Lu et al. 2022) for x = (1 - sigma) x0 + sigma eps, as per-step coefficients of
    x_{i+1} = a x_i + b D_i + c D_{i-1} (dk_sampler_dpmpp_2m), in fp64 -> (n, 3) for n + 1 sigmas.

    alpha = 1 - sigma, lambda = log(alpha / sigma), h_i = lambda_{i+1} - lambda_i.  First order, a = sigma_{i+1} /
    sigma_i and b = -alpha_{i+1} expm1(-h_i), is the Euler step; sigma_i = 1 gives h_i = inf and b = alpha_{i+1}.
    Second order extrapolates D' = (1 + 1/(2r)) D_i - 1/(2r) D_{i-1}, r = h_{i-1} / h_i.  It is used except on the
    first step, after an interval with h = inf, and on the last two steps: on the SD3 schedules the step from about
    1/n down to sigma_min has r << 1, and extrapolating across it is less accurate than Euler.  A step to sigma = 0
    returns D_i: (0, 1, 0)."""
    s = np.asarray(sigmas, dtype=np.float64)
    n = len(s) - 1
    with np.errstate(divide="ignore"):
        lam = np.log1p(-s) - np.log(s)                  # -inf at sigma = 1, +inf at sigma = 0
    h = lam[1:] - lam[:-1]
    coef = np.zeros((n, 3), dtype=np.float64)
    for i in range(n):
        if s[i + 1] == 0.0:
            coef[i] = (0.0, 1.0, 0.0)
            continue
        b1 = -(1.0 - s[i + 1]) * np.expm1(-h[i])
        if 1 <= i < n - 2 and np.isfinite(h[i - 1]):
            half_r = 0.5 * h[i] / h[i - 1]              # 1 / (2r)
            coef[i] = (s[i + 1] / s[i], b1 * (1.0 + half_r), -b1 * half_r)
        else:
            coef[i] = (s[i + 1] / s[i], b1, 0.0)
    return coef


def check_eta(eta) -> float:
    """the noise scale of a stochastic sampler: finite and >= 0 (ValueError otherwise)"""
    e = float(eta)
    if not (math.isfinite(e) and e >= 0.0):
        raise ValueError(f"eta must be finite and >= 0, got {eta}")
    return e


def euler_ancestral_coefficients(sigmas, eta: float = 1.0) -> np.ndarray:
    """The rectified-flow ancestral Euler step as per-step coefficients of x_{i+1} = a x_i + b D_i + c D_{i-1} + n z_i
    (dk_sampler_sde_step), in fp64 -> (steps, 4) for steps + 1 sigmas; c is always 0.

    sigma_down = sigma_{i+1} (1 + (sigma_{i+1} / sigma_i - 1) eta), alpha = 1 - sigma.  A deterministic Euler step to
    sigma_down, rescaled by alpha_{i+1} / alpha_down, plus noise of standard deviation
    sqrt(sigma_{i+1}^2 - (sigma_down alpha_{i+1} / alpha_down)^2):
        a = (alpha_{i+1} / alpha_down) sigma_down / sigma_i,  b = (alpha_{i+1} / alpha_down) (1 - sigma_down / sigma_i).
    eta = 0 gives Euler, (sigma_{i+1} / sigma_i, 1 - sigma_{i+1} / sigma_i, 0, 0).  An eta large enough to push
    sigma_down below 0 is held at sigma_down = 0 (D re-noised to sigma_{i+1}).  A step to sigma = 0 returns D: (0, 1, 0, 0).

    Check (fp64): with the exact denoiser D = x0 and x_i = alpha_i x0 + sigma_i eps, the coefficients of x0,
    a alpha_i + b + c, sum to alpha_{i+1}, and the independent noise a sigma_i eps + n z has standard deviation
    sqrt(a^2 sigma_i^2 + n^2) = sigma_{i+1}: each step lands on the marginal of x_{i+1}."""
    s = np.asarray(sigmas, dtype=np.float64)
    eta = check_eta(eta)
    coef = np.zeros((len(s) - 1, 4), dtype=np.float64)
    for i in range(len(s) - 1):
        sn = s[i + 1]
        if sn == 0.0:
            coef[i] = (0.0, 1.0, 0.0, 0.0)
            continue
        ratio = sn / s[i]
        sd = max(sn * (1.0 + (ratio - 1.0) * eta), 0.0)
        scale = (1.0 - sn) / (1.0 - sd)
        dn = sd * scale                                 # sigma_down alpha_{i+1} / alpha_down
        coef[i] = (scale * (sd / s[i]), scale * (1.0 - sd / s[i]), 0.0, math.sqrt(max(sn * sn - dn * dn, 0.0)))
    return coef


def dpmpp_2m_sde_coefficients(sigmas, eta: float = 1.0) -> np.ndarray:
    """DPM-Solver++(2M) SDE (Lu et al. 2022, data prediction, midpoint form) for x = (1 - sigma) x0 + sigma eps, as
    per-step coefficients of x_{i+1} = a x_i + b D_i + c D_{i-1} + n z_i (dk_sampler_sde_step), in fp64 -> (steps, 4).

    With h_i = lambda_{i+1} - lambda_i (lambda = log(alpha / sigma)):
        a = (sigma_{i+1} / sigma_i) e^{-eta h},  b1 = alpha_{i+1} (1 - e^{-(1 + eta) h}),
        n = sigma_{i+1} sqrt(1 - e^{-2 eta h}),
    and b1 is split into b and c by dpmpp_2m_coefficients' second-order rule D' = (1 + 1/(2r)) D_i - 1/(2r) D_{i-1}, on
    the same steps (not the first, not after an interval with h = inf, not the last two).  eta = 0 gives
    dpmpp_2m_coefficients exactly (n = 0).  A step from sigma = 1 (h = inf) has a = 0 for eta > 0; a step to sigma = 0
    returns D: (0, 1, 0, 0).

    Check (fp64): with D = x0, a alpha_i + b + c = alpha_{i+1} (since (sigma_{i+1} / sigma_i) alpha_i = alpha_{i+1} e^{-h})
    and sqrt(a^2 sigma_i^2 + n^2) = sigma_{i+1}, as for euler_ancestral_coefficients."""
    s = np.asarray(sigmas, dtype=np.float64)
    eta = check_eta(eta)
    n = len(s) - 1
    with np.errstate(divide="ignore"):
        lam = np.log1p(-s) - np.log(s)
    h = lam[1:] - lam[:-1]
    coef = np.zeros((n, 4), dtype=np.float64)
    for i in range(n):
        if s[i + 1] == 0.0:
            coef[i] = (0.0, 1.0, 0.0, 0.0)
            continue
        eh = eta * h[i] if eta > 0.0 else 0.0          # eta = 0 at h = inf is 0, not 0 * inf
        a = s[i + 1] / s[i] * math.exp(-eh)
        b1 = -(1.0 - s[i + 1]) * np.expm1(-(1.0 + eta) * h[i])
        noise = s[i + 1] * math.sqrt(-math.expm1(-2.0 * eh))
        if 1 <= i < n - 2 and np.isfinite(h[i - 1]):
            half_r = 0.5 * h[i] / h[i - 1]              # 1 / (2r)
            coef[i] = (a, b1 * (1.0 + half_r), -b1 * half_r, noise)
        else:
            coef[i] = (a, b1, 0.0, noise)
    return coef


@dataclass(frozen=True)
class SkipLayerGuidance:
    """Skip-layer guidance (SLG) for SD3-family models under CFG, as Stability's SkipLayerCFGDenoiser applies it: on the
    steps i of the n run with start·n < i < end·n, D = D_neg + w (D_pos - D_neg) + scale (D_pos - D_skip), where D_skip
    is the positive prompt's estimate from a forward that skips the joint blocks `layers`.  The defaults are
    Stability's published setting for SD3.5 Medium."""

    scale: float = 2.5
    layers: Tuple[int, ...] = (7, 8, 9)
    start: float = 0.01
    end: float = 0.20


def check_skip_layer_guidance(slg: SkipLayerGuidance, cfg_weight: float, depth: int) -> None:
    """Raise ValueError for a setting a model of `depth` joint blocks cannot run (before any GPU work)."""
    if not isinstance(slg, SkipLayerGuidance):
        raise ValueError(f"slg must be a SkipLayerGuidance or None, got {type(slg).__name__}")
    if not cfg_weight > 0:
        raise ValueError(f"skip-layer guidance needs CFG (cfg_weight > 0), got cfg_weight={cfg_weight}")
    layers = tuple(slg.layers)
    if not layers or len(set(layers)) != len(layers) or not all(
            isinstance(i, (int, np.integer)) and 0 <= i < depth for i in layers):
        raise ValueError(f"skip-layer guidance layers {layers} must be distinct joint block indices in [0, {depth})")
    if not 0.0 <= slg.start < slg.end <= 1.0:
        raise ValueError(f"skip-layer guidance window needs 0 <= start < end <= 1, got start={slg.start}, "
                         f"end={slg.end}")
    if not math.isfinite(slg.scale):
        raise ValueError(f"skip-layer guidance scale must be finite, got {slg.scale}")


def skip_layer_guidance_steps(slg: SkipLayerGuidance, n: int) -> List[int]:
    """the steps i of n where SLG applies: start·n < i < end·n (Stability's window, in the steps actually run)"""
    return [i for i in range(n) if slg.start * n < i < slg.end * n]
