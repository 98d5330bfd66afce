"""The stochastic samplers without a GPU (DESIGN.md §16): the oracle's Philox against the published known-answer
vectors, the uniforms, the coefficients at eta = 0, the marginal identity every step must satisfy, the closed-form
moments of Gaussian data under the exact denoiser, and the argument checks of both pipelines."""
import math

import numpy as np
import pytest

from diffusionkit_b200.pipeline import SDE_SOLVERS, SOLVERS, DiffusionPipeline, FluxPipeline
from diffusionkit_b200.sampler import (dpmpp_2m_coefficients, dpmpp_2m_sde_coefficients,
                                       euler_ancestral_coefficients)
from tests import sde_ref
from tests.test_solvers_cpu import product_sigmas

PRODUCT = {"euler_ancestral": euler_ancestral_coefficients, "dpmpp_2m_sde": dpmpp_2m_sde_coefficients}
# FLUX (shift 1) and SD3 (shift 3) schedules
SCHEDULES = [("flux", 1.0), ("sd3", 3.0)]


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    assert tuple(int(v) for v in sde_ref.philox4x32_10(ctr, key)[0]) == want


def test_uniforms_are_exact_and_strictly_inside_the_unit_interval():
    v = np.array([0, 1, 511, 512, 2 ** 31, 2 ** 32 - 513, 2 ** 32 - 512, 2 ** 32 - 1], dtype=np.uint32)
    u = sde_ref.uniforms(v)
    exact = ((v >> 9).astype(np.float64) + 0.5) * 2.0 ** -23
    assert u.dtype == np.float32 and np.array_equal(u.astype(np.float64), exact)
    assert float(u.min()) == 2.0 ** -24 and float(u.max()) == 1.0 - 2.0 ** -24
    v = sde_ref.philox4x32_10(np.stack([np.arange(1 << 16), np.zeros(1 << 16), np.zeros(1 << 16),
                                        np.zeros(1 << 16)], 1), (5, 0)).reshape(-1)
    u = sde_ref.uniforms(v)
    assert 0.0 < float(u.min()) and float(u.max()) < 1.0
    # the 24-bit form (k + 0.5) 2^-24 is not representable for k >= 2^23: fp32 rounds it, up to 1.0 at the top
    assert float(np.float32(2 ** 24 - 1) + np.float32(0.5)) * 2.0 ** -24 == 1.0


@pytest.mark.parametrize("kind,shift", SCHEDULES)
def test_eta_zero_is_the_deterministic_step(kind, shift):
    for n in (1, 2, 4, 8, 28):
        sig = product_sigmas(kind, shift, n)
        sde = dpmpp_2m_sde_coefficients(sig, 0.0)
        assert np.array_equal(sde[:, :3], dpmpp_2m_coefficients(sig)) and np.array_equal(sde[:, 3], np.zeros(n))
        anc = euler_ancestral_coefficients(sig, 0.0)
        for i in range(n - 1):
            r = sig[i + 1] / sig[i]
            assert tuple(anc[i]) == (r, 1.0 - r, 0.0, 0.0), (n, i)
        assert tuple(anc[-1]) == (0.0, 1.0, 0.0, 0.0)


@pytest.mark.parametrize("kind,shift", SCHEDULES)
@pytest.mark.parametrize("eta", [0.5, 1.0])
def test_every_step_lands_on_the_marginal(kind, shift, eta):
    """with the exact denoiser D = x0: a alpha_i + b + c = alpha_{i+1} and a^2 sigma_i^2 + n^2 = sigma_{i+1}^2"""
    for n in (4, 8, 28):
        sig = product_sigmas(kind, shift, n)
        for solver, fn in PRODUCT.items():
            coef = fn(sig, eta)
            assert coef.shape == (n, 4) and coef.dtype == np.float64
            assert np.allclose(coef, sde_ref.coefficients(solver, sig, eta), rtol=1e-12, atol=1e-14), (solver, n)
            assert tuple(coef[-1]) == (0.0, 1.0, 0.0, 0.0)
            for i, (a, b, c, nz) in enumerate(coef):
                assert abs(a * (1.0 - sig[i]) + b + c - (1.0 - sig[i + 1])) <= 1e-12, (solver, n, i)
                assert abs(math.sqrt(a * a * sig[i] ** 2 + nz * nz) - sig[i + 1]) <= 1e-12, (solver, n, i)
            if solver == "dpmpp_2m_sde":
                assert sig[0] == 1.0 and coef[0][0] == 0.0              # from sigma = 1 (h = inf) a = 0
                assert [c != 0 for c in coef[:, 2]] == [c != 0 for c in dpmpp_2m_coefficients(sig)[:, 2]]
            assert all(v > 0 for v in coef[:-1, 3])


def test_a_large_eta_holds_sigma_down_at_zero():
    sig = product_sigmas("sd3", 3.0, 8)
    coef = euler_ancestral_coefficients(sig, 50.0)
    for i, (a, b, c, nz) in enumerate(coef[:-1]):
        assert a == 0.0 and b == 1.0 - sig[i + 1] and nz == sig[i + 1]


# ------------------------------------------------------------------------------------------------ Gaussian moments
MU, S = 0.3, 0.7


def _propagate(coef, sig):
    """mean and covariance of (x_i, D_{i-1}) for x0 ~ N(MU, S^2), x_0 = alpha_0 x0 + sigma_0 eps, under
    x <- a x + b D(x) + c D_prev + n z with the exact denoiser D(x, sigma) = p + q x -> terminal (mean, std)"""
    m = np.array([(1.0 - sig[0]) * MU, 0.0])
    cov = np.array([[(1.0 - sig[0]) ** 2 * S * S + sig[0] ** 2, 0.0], [0.0, 0.0]])
    for i, (a, b, c, nz) in enumerate(coef):
        al, s = 1.0 - sig[i], sig[i]
        q = al * S * S / (al * al * S * S + s * s)
        p = MU - q * al * MU
        M = np.array([[a + b * q, c], [q, 0.0]])
        m = M @ m + np.array([b * p, p])
        cov = M @ cov @ M.T + np.diag([nz * nz, 0.0])
    return m[0], math.sqrt(cov[0, 0])


@pytest.mark.parametrize("kind,shift", SCHEDULES)
def test_terminal_error_falls_with_the_step_count(kind, shift):
    """the W2 distance of the terminal Gaussian from N(MU, S^2), in closed form (2 x 2 covariance for the 2M SDE)"""
    err = {}
    for solver, fn in PRODUCT.items():
        for n in (8, 16, 32, 64):
            sig = product_sigmas(kind, shift, n)
            mean, std = _propagate(fn(sig, 1.0), sig)
            err[solver, n] = math.hypot(mean - MU, std - S)
    print(kind, shift, {k: f"{v:.3e}" for k, v in err.items()})
    for solver in PRODUCT:
        assert err[solver, 64] < err[solver, 8], (solver, err[solver, 8], err[solver, 64])


# ------------------------------------------------------------------------------------------------ arguments
@pytest.mark.parametrize("cls", [FluxPipeline, DiffusionPipeline])
def test_eta_is_refused_before_any_work(cls):
    p = object.__new__(cls)                     # no device, no model: the checks run first
    assert sorted(SDE_SOLVERS) == ["dpmpp_2m_sde", "euler_ancestral"] and not set(SOLVERS) & set(SDE_SOLVERS)
    bad = [("euler", 1.0), ("dpmpp_2m", 0.0), ("heun", 0.5), ("euler_ancestral", -0.1), ("dpmpp_2m_sde", float("nan")),
           ("euler_ancestral", float("inf"))]
    for solver, eta in bad:
        for call in (lambda: p.denoise_latents(None, None, solver=solver, eta=eta),
                     lambda: p.generate_image("", solver=solver, eta=eta)):
            with pytest.raises(ValueError, match="eta"):
                call()
    with pytest.raises(ValueError) as e:
        p.denoise_latents(None, None, solver="euler_a")
    assert all(repr(k) in str(e.value) for k in (*SOLVERS, *SDE_SOLVERS))
