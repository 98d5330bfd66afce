"""CPU restatement of the stochastic samplers (DESIGN.md §16): the noise contract (numpy Philox4x32-10, the 23-bit
uniforms, Box-Muller in fp64 from the fp32 uniforms), the per-step coefficients in textbook form, Euler ancestral and
DPM-Solver++(2M) SDE over the oracle's model calls, and the launch-census reference of
pipeline.sampler_sde_step.  Independent of diffusionkit_b200.sampler, which the tests check against it.

Conventions are tests/solver_ref.py's: the model sees the state cast to act_dtype, the timesteps are sigma * 1000 cast
the same way, D is the CFG-mixed calculate_denoised, and the state stays in the dtype of x."""
from __future__ import annotations

import math
from typing import Callable, Optional

import numpy as np
import torch

_M32 = np.uint64(0xFFFFFFFF)
_PHILOX_M = (np.uint64(0xD2511F53), np.uint64(0xCD9E8D57))
_PHILOX_W = (np.uint64(0x9E3779B9), np.uint64(0xBB67AE85))


# ------------------------------------------------------------------------------------------------ noise
def philox4x32_10(ctr, key) -> np.ndarray:
    """Philox4x32-10 (Salmon et al. 2011): ctr (N, 4) or (4,) 32-bit words, key (2,) -> (N, 4) uint32"""
    c = np.atleast_2d(np.asarray(ctr, dtype=np.uint64))
    x0, x1, x2, x3 = (c[:, j].copy() for j in range(4))
    k0, k1 = np.uint64(int(key[0]) & 0xFFFFFFFF), np.uint64(int(key[1]) & 0xFFFFFFFF)
    for r in range(10):
        if r:
            k0, k1 = (k0 + _PHILOX_W[0]) & _M32, (k1 + _PHILOX_W[1]) & _M32
        p0, p1 = _PHILOX_M[0] * x0, _PHILOX_M[1] * x2        # 32 x 32 -> 64 bits: no wrap in uint64
        x0, x1, x2, x3 = (p1 >> np.uint64(32)) ^ x1 ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ x3 ^ k1, p0 & _M32
    return np.stack([x0, x1, x2, x3], axis=1).astype(np.uint32)


def uniforms(v: np.ndarray) -> np.ndarray:
    """((v >> 9) + 0.5) 2^-23 as fp32 (exact; strictly inside (0, 1))"""
    return (((v.astype(np.uint32) >> np.uint32(9)).astype(np.float64) + 0.5) * 2.0 ** -23).astype(np.float32)


def normals(seed: int, step: int, n: int) -> np.ndarray:
    """the fp64 normals z[0..n) of one image (seed) at one solver step, element e from Philox counter
    (e // 4, step, 0, 0) and key (lo32(seed), hi32(seed)): Box-Muller on (u0, u1) for e % 4 in {0, 1}, on (u2, u3) for
    {2, 3}, computed in fp64 from the fp32 uniforms"""
    assert n % 4 == 0 and 0 <= seed < 2 ** 64
    q = np.arange(n // 4, dtype=np.uint64)
    ctr = np.stack([q, np.full_like(q, step), np.zeros_like(q), np.zeros_like(q)], axis=1)
    u = uniforms(philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))).astype(np.float64)
    z = np.empty((n // 4, 4), dtype=np.float64)
    for j in (0, 2):
        r = np.sqrt(-2.0 * np.log(u[:, j]))
        z[:, j] = r * np.cos(2.0 * np.pi * u[:, j + 1])
        z[:, j + 1] = r * np.sin(2.0 * np.pi * u[:, j + 1])
    return z.reshape(-1)


# ------------------------------------------------------------------------------------------------ coefficients
def _lam(sigma: float) -> float:
    """log(alpha / sigma), alpha = 1 - sigma: -inf at sigma = 1, +inf at sigma = 0"""
    if sigma == 1.0:
        return -math.inf
    if sigma == 0.0:
        return math.inf
    return math.log((1.0 - sigma) / sigma)


def coefficients(solver: str, sigmas, eta: float) -> np.ndarray:
    """(steps, 4) fp64 (a, b, c, n) of x_{i+1} = a x_i + b D_i + c D_{i-1} + n z_i, step by step from the textbook
    forms: the rectified-flow ancestral step (an Euler step to sigma_down, rescaled by alpha_{i+1} / alpha_down, noise
    to reach sigma_{i+1}), and DPM-Solver++(2M) SDE with D' = (1 + 1/(2r)) D_i - 1/(2r) D_{i-1} on the steps
    DPM-Solver++(2M) takes it"""
    s = [float(v) for v in np.asarray(sigmas, dtype=np.float64)]
    n = len(s) - 1
    out = np.zeros((n, 4))
    h_prev = None
    for i in range(n):
        sig, nxt = s[i], s[i + 1]
        h = _lam(nxt) - _lam(sig)
        if nxt == 0.0:
            out[i] = (0.0, 1.0, 0.0, 0.0)
        elif solver == "euler_ancestral":
            down = max(nxt * (1.0 + (nxt / sig - 1.0) * eta), 0.0)
            k = (1.0 - nxt) / (1.0 - down)
            std = math.sqrt(max(nxt ** 2 - (down * k) ** 2, 0.0))
            out[i] = (k * down / sig, k * (1.0 - down / sig), 0.0, std)
        else:
            decay = 0.0 if (eta > 0 and math.isinf(h)) else math.exp(-eta * h) if eta > 0 else 1.0
            a = nxt / sig * decay
            b1 = (1.0 - nxt) * (1.0 - math.exp(-(1.0 + eta) * h))
            std = nxt * math.sqrt(max(1.0 - decay * decay, 0.0))
            if 1 <= i < n - 2 and math.isfinite(h_prev):
                r = h_prev / h
                out[i] = (a, b1 * (1.0 + 1.0 / (2.0 * r)), -b1 / (2.0 * r), std)
            else:
                out[i] = (a, b1, 0.0, std)
        h_prev = h
    return out


# ------------------------------------------------------------------------------------------------ samplers
def sample(solver: str, denoise: Callable[[torch.Tensor, int], torch.Tensor], x: torch.Tensor, sigmas, seed: int,
           eta: float = 1.0) -> torch.Tensor:
    """one image (x (1, H, W, 16)) through `solver`; denoise(x, i) is the step-i denoised estimate; z_i from
    normals(seed, i, .) in x's dtype"""
    coef = coefficients(solver, sigmas, eta)
    den_prev = None
    for i, (a, b, c, n) in enumerate(coef):
        den = denoise(x, i)
        z = torch.from_numpy(normals(seed, i, x.numel())).reshape(x.shape).to(x.dtype) if n != 0.0 else 0.0
        x = a * x + b * den + (c * den_prev if c != 0.0 else 0.0) + n * z
        den_prev = den
    return x


def _solver_call(solver, mmdit_call, cache_modulation, x, sigmas, conditioning, pooled, cfg_weight, act_dtype, seed,
                 eta):
    from tests.solver_ref import _denoiser, _setup

    cast, timesteps = _setup(cache_modulation, sigmas, pooled, act_dtype)
    sig = [float(v) for v in sigmas]
    return sample(solver, lambda xx, i: _denoiser(mmdit_call, xx, conditioning, timesteps[i], sig[i], cfg_weight, cast),
                  x, sigmas, seed, eta)


def sample_euler_ancestral(mmdit_call, cache_modulation, x, sigmas, conditioning, pooled, cfg_weight: float,
                           act_dtype: Optional[torch.dtype], *, seed: int, eta: float = 1.0) -> torch.Tensor:
    """tests/solver_ref.sample_heun's signature plus the image's noise seed and eta"""
    return _solver_call("euler_ancestral", mmdit_call, cache_modulation, x, sigmas, conditioning, pooled, cfg_weight,
                        act_dtype, seed, eta)


def sample_dpmpp_2m_sde(mmdit_call, cache_modulation, x, sigmas, conditioning, pooled, cfg_weight: float,
                        act_dtype: Optional[torch.dtype], *, seed: int, eta: float = 1.0) -> torch.Tensor:
    return _solver_call("dpmpp_2m_sde", mmdit_call, cache_modulation, x, sigmas, conditioning, pooled, cfg_weight,
                        act_dtype, seed, eta)


def sample_slg(solver: str, model, x, sigmas, conditioning, pooled, cfg_weight: float,
               act_dtype: Optional[torch.dtype], *, seed: int, eta: float = 1.0, scale: float = 0.0, layers=(),
               start: float = 0.0, end: float = 0.0) -> torch.Tensor:
    """an SD3.5-medium oracle model (tests/sd35_medium_ref.MMDiTXRef) under CFG with skip-layer guidance"""
    from tests.sd35_medium_ref import slg_denoiser, slg_window

    def cast(t):
        return t if act_dtype is None else t.to(act_dtype).to(torch.float32)

    timesteps = cast(sigmas * 1000.0)
    model.cache_modulation_params(pooled, timesteps)
    window = set(slg_window(len(sigmas) - 1, start, end))
    sig = [float(v) for v in sigmas]
    return sample(solver, lambda xx, i: slg_denoiser(model, xx, conditioning, timesteps[i], sig[i], cfg_weight, cast,
                                                     scale, layers, i in window), x, sigmas, seed, eta)


# ------------------------------------------------------------------------------------------------ kernel reference
def ref_sde_step(x, d_prev, xin, out, sigma, a, b, c, noise, cfg_weight, slg, seeds, step):
    """-> (a x + b D + c d_prev + noise z, D) in fp64 on x's device, z image by image from normals(seeds[b], step)"""
    from tests.kernel_checks import ref_denoised

    B = x.shape[0]
    n = x.numel()
    den = ref_denoised(xin, out, sigma, cfg_weight, n, slg).double().reshape(x.shape)
    y = a * x.double() + b * den
    if c != 0.0:
        y = y + c * d_prev.double()
    if noise != 0.0:
        sv = [int(v) for v in seeds.cpu().numpy()]
        z = np.stack([normals(sv[i], step, n // B) for i in range(B)]).reshape(tuple(x.shape))
        y = y + noise * torch.from_numpy(z).to(x.device)
    return y, den


def census_check(L, a, s, r, census):
    """tests/launch_parity check of one pipeline.sampler_sde_step launch"""
    from tests import launch_parity as lp

    x_ref, d_ref = ref_sde_step(s["x"], s["d_prev"], s["xin"], s["out"], a["sigma"], a["a"], a["b"], a["c"],
                                a["noise"], a["cfg_weight"], a["slg"], s["seeds"], a["step"])
    L.close("x", r, x_ref, lp.TOL_F32)
    L.own(r)
    if a["d_prev"] is not None:
        L.close("d_prev", a["d_prev"], d_ref, lp.TOL_F32)
        L.own(a["d_prev"])
    L.sig.update(B=r.shape[0], reps=s["xin"].numel() // r.numel(), cfg=a["cfg_weight"] > 0, slg=a["slg"] != 0.0,
                 d_prev=a["d_prev"] is not None, second_order=a["c"] != 0.0, noise=a["noise"] != 0.0,
                 dtype=str(s["xin"].dtype)[6:])
