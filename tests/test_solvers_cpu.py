"""The Heun and DPM-Solver++(2M) rules without a GPU, on an ODE whose solution is known exactly.

For Gaussian data x0 ~ N(mu, s^2) per element and x = (1 - sigma) x0 + sigma eps, the ideal denoiser is
D(x, sigma) = mu + (1 - sigma) s^2 / ((1 - sigma)^2 s^2 + sigma^2) (x - (1 - sigma) mu), and the probability-flow ODE
dx/dsigma = (x - D) / sigma carries x(1) = eps to x(0) = mu + s eps.  On the product's schedules (FLUX and SD3, shift 1
and 3) every solver's error against that endpoint is compared with Euler's at the same number of steps."""
import numpy as np
import pytest
import torch

from diffusionkit_b200.pipeline import SOLVERS, DiffusionPipeline, FluxPipeline
from diffusionkit_b200.sampler import FluxSampler, ModelSamplingDiscreteFlow, dpmpp_2m_coefficients
from oracle import sampler_ref as sr
from tests import solver_ref

MU, S = 0.3, 0.7
EPS = torch.from_numpy(np.random.RandomState(0).randn(1, 10000))        # float64
EXACT = MU + S * EPS
SCHEDULES = [("flux", 1.0), ("flux", 3.0), ("sd3", 1.0), ("sd3", 3.0)]


def exact_denoiser(x, sigma):
    a = 1.0 - sigma
    return MU + a * S * S / (a * a * S * S + sigma * sigma) * (x - a * MU)


def product_sigmas(kind, shift, n):
    """the product's get_sigmas (fp32), in fp64"""
    cls, sampler = (FluxPipeline, FluxSampler) if kind == "flux" else (DiffusionPipeline, ModelSamplingDiscreteFlow)
    p = object.__new__(cls)
    p.sampler = sampler(shift)
    return p.get_sigmas(p.sampler, n).astype(np.float64)


def run_oracle(sample, sig):
    """an oracle sampler (sample_euler's signature) with the exact denoiser as the model, in fp64"""
    sigmas = torch.from_numpy(sig)
    sigma_of = {float(t): float(s) for t, s in zip(sigmas * 1000.0, sigmas)}

    def model(xin, cond, t):                    # the velocity whose calculate_denoised is D
        sigma = sigma_of[float(t[0])]
        return (xin - exact_denoiser(xin, sigma)) / sigma

    return sample(model, lambda pooled, ts: None, EPS.clone(), sigmas, None, None, 0.0, None)


def run_product_2m(sig):
    """x <- a x + b D + c D_prev with the product's coefficients, as dk_sampler_dpmpp_2m applies them"""
    x, d_prev = EPS.clone(), None
    for i, (a, b, c) in enumerate(dpmpp_2m_coefficients(sig)):
        den = exact_denoiser(x, float(sig[i]))
        x = a * x + b * den + (c * d_prev if c != 0.0 else 0.0)
        d_prev = den
    return x


def rms(x):
    return float(((x - EXACT) ** 2).mean().sqrt())


@pytest.mark.parametrize("kind,shift", SCHEDULES)
def test_solvers_beat_euler_on_the_exact_ode(kind, shift):
    err = {}
    for n in (8, 16, 32):
        sig = product_sigmas(kind, shift, n)
        assert sig[0] == 1.0 and sig[-1] == 0.0 and np.all(sig[:-1] > 0)
        two_m = run_product_2m(sig)
        oracle_2m = run_oracle(solver_ref.sample_dpmpp_2m, sig)
        assert float((two_m - oracle_2m).abs().max()) <= 1e-12, n
        err[n] = {"euler": rms(run_oracle(sr.sample_euler, sig)), "heun": rms(run_oracle(solver_ref.sample_heun, sig)),
                  "dpmpp_2m": rms(two_m)}
    ratio = {n: {k: e[k] / e["euler"] for k in ("heun", "dpmpp_2m")} for n, e in err.items()}
    print(kind, shift, {n: {k: round(v, 3) for k, v in r.items()} for n, r in ratio.items()})
    for n in (16, 32):
        assert ratio[n]["heun"] <= 0.35, (n, ratio[n])
    assert ratio[16]["dpmpp_2m"] <= 0.65 and ratio[32]["dpmpp_2m"] <= 0.25, ratio
    assert ratio[8]["heun"] < 1 and ratio[8]["dpmpp_2m"] < 1, ratio[8]
    for k in ("euler", "heun", "dpmpp_2m"):
        assert err[32][k] < err[16][k], (k, err[16][k], err[32][k])


def test_dpmpp_2m_coefficients_at_the_ends():
    for kind, shift in SCHEDULES:
        for n in (1, 2, 4, 16):
            sig = product_sigmas(kind, shift, n)
            coef = dpmpp_2m_coefficients(sig)
            assert coef.shape == (n, 3) and coef.dtype == np.float64
            assert tuple(coef[-1]) == (0.0, 1.0, 0.0)
            if n > 1:
                assert tuple(coef[0]) == (sig[1], 1.0 - sig[1], 0.0)
            # a first-order step is the Euler step: a = sigma'/sigma, b = 1 - sigma'/sigma
            for i, (a, b, c) in enumerate(coef[:-1]):
                assert a == sig[i + 1] / sig[i]
                if c == 0.0:
                    assert abs(a + b - 1.0) <= 1e-14
                else:
                    assert abs(a + b + c - 1.0) <= 1e-14      # D' is an affine combination of D_i and D_{i-1}


def test_dpmpp_2m_second_order_steps():
    """second order everywhere except the first step, after an infinite interval and on the last two steps"""
    sig = product_sigmas("sd3", 3.0, 8)
    assert sig[0] == 1.0                        # h_0 = inf, so step 1 is first order too
    assert [c != 0.0 for _, _, c in dpmpp_2m_coefficients(sig)] == [False, False] + [True] * 4 + [False, False]
    # img2img: a trimmed schedule starts below sigma = 1, so its first interval is finite
    assert [c != 0.0 for _, _, c in dpmpp_2m_coefficients(sig[3:])] == [False, True, True, False, False]
    assert [c != 0.0 for _, _, c in dpmpp_2m_coefficients(sig[-3:])] == [False, False]


@pytest.mark.parametrize("cls", [FluxPipeline, DiffusionPipeline])
def test_unknown_solver_is_refused_before_any_work(cls):
    p = object.__new__(cls)                     # no device, no model: the check runs first
    assert sorted(SOLVERS) == ["dpmpp_2m", "euler", "heun"]
    for call in (lambda: p.denoise_latents(None, None, solver="dpm++"),
                 lambda: p.generate_image("", solver="Euler")):
        with pytest.raises(ValueError) as e:
            call()
        assert all(repr(name) in str(e.value) for name in SOLVERS), str(e.value)
