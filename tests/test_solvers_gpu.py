"""GPU checks of the Heun and DPM-Solver++(2M) samplers: the three step kernels against fp32 torch evaluations of their
formulas, the tiny FLUX and SD3-CFG pipelines against the oracle's solvers (tests/solver_ref.py), Euler unchanged,
determinism with and without CUDA graphs, the step cache at threshold 0, img2img and FP8."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
bf16, fp16 = torch.bfloat16, torch.float16
NEW_SOLVERS = ["heun", "dpmpp_2m"]


@pytest.fixture(scope="module")
def kc():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    from tests import kernel_checks

    kernel_checks._setup()
    return kernel_checks


# ------------------------------------------------------------------------------------------------ kernels
def _inputs(dtype, cfg, n, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    reps = 2 if cfg > 0 else 1
    x = torch.randn((n,), generator=g, device=DEV)
    xin = torch.randn((reps * n,), generator=g, device=DEV).to(dtype)
    out = torch.randn((reps * n,), generator=g, device=DEV).to(dtype)
    return x, xin, out


N_ODD = 3 * 4099          # not a multiple of the block or of any vector width


@pytest.mark.parametrize("dtype", [bf16, fp16])
@pytest.mark.parametrize("cfg", [0.0, 5.0])
def test_heun_kernels(kc, dtype, cfg):
    from diffusionkit_b200 import ops

    n, sigma, sigma_next = N_ODD, 0.6875, 0.5
    x, xin, out = _inputs(dtype, cfg, n, 1)
    x0 = x.clone()
    d, x2 = ops.sampler_heun_predict(x, xin, out, sigma, sigma_next, cfg)
    assert torch.equal(x, x0), "the predictor modified x"
    d_ref = (x - kc.ref_denoised(xin, out, sigma, cfg, n)) / sigma
    x2_ref = x + d_ref * (sigma_next - sigma)
    kc._assert_close("heun_predict_d", d, d_ref, 1e-6)
    kc._assert_close("heun_predict_x2", x2, x2_ref, 1e-6)
    _, xin2, out2 = _inputs(dtype, cfg, n, 2)                   # the forward at (x2, sigma_next)
    d2_ref = (x2 - kc.ref_denoised(xin2, out2, sigma_next, cfg, n)) / sigma_next
    want = x + (d + d2_ref) / 2 * (sigma_next - sigma)
    got = ops.sampler_heun_correct(x.clone(), d, x2, xin2, out2, sigma, sigma_next, cfg)
    kc._assert_close("heun_correct", got, want, 1e-6)


@pytest.mark.parametrize("dtype", [bf16, fp16])
@pytest.mark.parametrize("cfg", [0.0, 5.0])
def test_dpmpp_2m_kernel(kc, dtype, cfg):
    from diffusionkit_b200 import ops
    from diffusionkit_b200.pipeline import FluxPipeline
    from diffusionkit_b200.sampler import FluxSampler, dpmpp_2m_coefficients

    p = object.__new__(FluxPipeline)
    sig = p.get_sigmas(FluxSampler(3.0), 16)
    coef = dpmpp_2m_coefficients(sig)
    n = N_ODD
    x, xin, out = _inputs(dtype, cfg, n, 3)
    for i in (0, 5, 15):                                        # sigma = 1, a second-order step, the step to 0
        a, b, c = (float(v) for v in coef[i])
        sigma = float(sig[i])
        d_prev = torch.randn((n,), device=DEV)
        den = kc.ref_denoised(xin, out, sigma, cfg, n)
        want = a * x + b * den + c * d_prev
        got_prev = d_prev.clone()
        got = ops.sampler_dpmpp_2m(x.clone(), got_prev, xin, out, sigma, a, b, c, cfg)
        kc._assert_close(f"dpmpp_2m_{i}", got, want, 1e-6)
        kc._assert_close(f"dpmpp_2m_{i}_d_prev", got_prev, den, 1e-6)
    assert coef[5][2] != 0.0


def test_dpmpp_2m_does_not_read_d_prev_when_c_is_zero(kc):
    from diffusionkit_b200 import ops

    n = N_ODD
    x, xin, out = _inputs(bf16, 0.0, n, 4)
    d_prev = torch.full((n,), float("nan"), device=DEV)
    got = ops.sampler_dpmpp_2m(x.clone(), d_prev, xin, out, 1.0, 0.75, 0.25, 0.0, 0.0)
    assert bool(torch.isfinite(got).all()) and bool(torch.isfinite(d_prev).all())
    kc._assert_close("dpmpp_2m_first", got, 0.75 * x + 0.25 * kc.ref_denoised(xin, out, 1.0, 0.0, n), 1e-6)


def test_heun_correct_refuses_sigma_next_zero(kc):
    from diffusionkit_b200 import DkError, ops

    c = ops.ctx(0)
    n0 = c.launches
    x, xin, out = _inputs(bf16, 0.0, 64, 5)
    with pytest.raises(DkError, match="sigma_next must be non-zero"):
        ops.sampler_heun_correct(x, x.clone(), x.clone(), xin, out, 0.25, 0.0, 0.0)
    assert c.launches == n0


# ------------------------------------------------------------------------------------------------ pipelines
CASES = {  # kind: (config factory, dtype, steps, cfg weight, shift, text length, pipeline, model version, format)
    "flux": ("tiny_flux_config", bf16, 4, 0.0, 1.0, 16, "FluxPipeline", "argmaxinc/mlx-FLUX.1-schnell", "flux"),
    "sd3": ("tiny_sd3_config", fp16, 6, 5.0, 3.0, 24, "DiffusionPipeline", "argmaxinc/mlx-stable-diffusion-3-medium",
            "sd3"),
}
LAT = (8, 12)
SEEDS = [11, 12]


def _weights(kind):
    from diffusionkit_b200 import config
    from diffusionkit_b200.config import VAEDecoderConfig
    from diffusionkit_b200.weights import init_params, mmdit_param_specs, vae_decoder_param_specs

    cfg = getattr(config, CASES[kind][0])()
    dtype = CASES[kind][1]
    # generated in fp32 on the host and rounded, so the oracle sees exactly the device's weights
    p16 = {k: v.to(dtype) for k, v in init_params(mmdit_param_specs(cfg), seed=7, dtype=torch.float32).items()}
    vp16 = {k: v.to(dtype) for k, v in init_params(vae_decoder_param_specs(VAEDecoderConfig()), seed=8,
                                                    dtype=torch.float32).items()}
    return cfg, p16, vp16


def _pipe(kind, p16, vp16=None, **kw):
    import diffusionkit_b200 as dk

    make, _, _, _, shift, _, cls, mv, _ = CASES[kind]
    from diffusionkit_b200 import config

    return getattr(dk, cls)(w16=True, a16=True, shift=shift, model_version=mv, mmdit_config=getattr(config, make)(),
                            params={k: v.to(DEV) for k, v in p16.items()},
                            vae_params=None if vp16 is None else {k: v.to(DEV) for k, v in vp16.items()},
                            load_decoder=vp16 is not None, **kw)


def _denoise(pipe, kind, cond, pooled, **kw):
    steps, cfgw = CASES[kind][2], CASES[kind][3]
    lat, it = pipe.denoise_latents(cond, pooled, num_steps=steps, cfg_weight=cfgw, latent_size=LAT, seed=SEEDS, **kw)
    torch.cuda.synchronize()
    return lat.clone(), it


def _oracle_latents(kind, solver, cfg, p16, cond, pooled, sig=None, x0s=None):
    """the oracle's solver of that name, one image at a time (CFG doubles it), -> process_out latents"""
    from oracle import sampler_ref as sr
    from oracle.mmdit_ref import MMDiTRef
    from tests import solver_ref
    from tests.oracle_bridge import ref_config

    _, dtype, steps, cfgw, shift, _, _, _, fmt = CASES[kind]
    sample = {"euler": sr.sample_euler, "heun": solver_ref.sample_heun,
              "dpmpp_2m": solver_ref.sample_dpmpp_2m}[solver]
    sampler = sr.FluxSamplerRef(shift) if kind == "flux" else sr.ModelSamplingDiscreteFlowRef(shift)
    if sig is None:
        sig = sr.get_sigmas(sampler, steps)
    H, W = LAT
    n = len(SEEDS)
    reps = 2 if cfgw > 0 else 1
    outs = []
    for i, s in enumerate(SEEDS):
        ref = MMDiTRef(ref_config(cfg), {k: v.float() for k, v in p16.items()})
        idx = [i + k * n for k in range(reps)]
        x0 = (sampler.noise_scaling(float(sig[0]), sr.get_noise(s, H, W), sr.get_empty_latent(H, W))
              if x0s is None else x0s[i])
        x = sample(lambda xin, c, t: ref(xin, c, t), ref.cache_modulation_params, x0, sig, cond[idx].float(),
                   pooled[idx].float(), cfgw, dtype)
        outs.append(sr.process_out(x, fmt))
    return torch.cat(outs)


@pytest.mark.parametrize("solver", NEW_SOLVERS)
@pytest.mark.parametrize("kind", ["flux", "sd3"])
def test_pipeline_against_the_oracle(kc, kind, solver):
    from oracle.vae_ref import VAEDecoderRef, decode_latents_to_image
    from tests.model_checks import psnr, rel_l2

    cfg, p16, vp16 = _weights(kind)
    pipe = _pipe(kind, p16, vp16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=CASES[kind][5])
    steps, cfgw = CASES[kind][2], CASES[kind][3]
    latent, iter_time = _denoise(pipe, kind, cond, pooled, solver=solver)
    assert latent.shape == (len(SEEDS), *LAT, 16) and len(iter_time) == steps
    want = _oracle_latents(kind, solver, cfg, p16, cond, pooled)
    r = rel_l2(latent, want)
    dtype = CASES[kind][1]
    img_want = decode_latents_to_image(VAEDecoderRef({k: v.float() for k, v in vp16.items()}), want.to(dtype).float())
    ps = psnr(img_want, pipe.decode_latents_to_image(latent))
    euler = _oracle_latents(kind, "euler", cfg, p16, cond, pooled)
    print(f"{kind} {solver}: final latent rel_l2 {r:.3e}, decoded psnr {ps:.1f} dB; "
          f"oracle {solver} vs oracle euler rel_l2 {rel_l2(want, euler):.3e}")
    assert r <= 5e-2, f"{kind} {solver} final latent rel_l2 {r:.3e}"
    assert ps >= (30.0 if kind == "flux" else 20.0), f"{kind} {solver} decoded RGB psnr {ps:.1f}"
    # generate_image logs the solver and its model evaluations
    reps = 2 if cfgw > 0 else 1
    idx = [0] + ([len(SEEDS)] if reps == 2 else [])
    image, log = pipe.generate_image("", num_steps=steps, cfg_weight=cfgw, latent_size=LAT, seed=SEEDS[0],
                                     verbose=False, conditioning=cond[idx], pooled_conditioning=pooled[idx],
                                     solver=solver)
    assert image.size == (LAT[1] * 8, LAT[0] * 8) and len(log["denoising"]["iter_time"]) == steps
    assert log["denoising"]["solver"] == solver
    assert log["denoising"]["nfe"] == (2 * steps - 1 if solver == "heun" else steps)
    _, log = pipe.generate_image("", num_steps=steps, cfg_weight=cfgw, latent_size=LAT, seed=SEEDS[0], verbose=False,
                                 conditioning=cond[idx], pooled_conditioning=pooled[idx])
    assert "solver" not in log["denoising"] and "nfe" not in log["denoising"]


@pytest.mark.parametrize("kind", ["flux", "sd3"])
def test_euler_argument_changes_nothing(kc, kind):
    from diffusionkit_b200 import ops

    _, p16, _ = _weights(kind)
    pipe = _pipe(kind, p16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=CASES[kind][5])
    _denoise(pipe, kind, cond, pooled)                          # captures the forward's graph
    n0 = ops.launch_count()
    plain, _ = _denoise(pipe, kind, cond, pooled)
    n1 = ops.launch_count()
    named, _ = _denoise(pipe, kind, cond, pooled, solver="euler")
    n2 = ops.launch_count()
    assert torch.equal(plain, named)
    assert n2 - n1 == n1 - n0


@pytest.mark.parametrize("kind", ["flux", "sd3"])
def test_new_solvers_are_deterministic_with_and_without_graphs(kc, monkeypatch, kind):
    _, p16, _ = _weights(kind)
    runs = {}
    for graphs in ("1", "0"):
        monkeypatch.setenv("DK_CUDA_GRAPHS", graphs)
        pipe = _pipe(kind, p16)
        assert pipe.mmdit.use_cuda_graphs == (graphs == "1")
        cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=CASES[kind][5])
        for solver in NEW_SOLVERS:
            a, _ = _denoise(pipe, kind, cond, pooled, solver=solver)
            b, _ = _denoise(pipe, kind, cond, pooled, solver=solver)
            assert torch.equal(a, b), (graphs, solver)
            assert bool(torch.isfinite(a).all())
            runs[graphs, solver] = a
        del pipe
    for solver in NEW_SOLVERS:
        assert torch.equal(runs["1", solver], runs["0", solver]), solver
    assert not torch.equal(runs["1", "heun"], runs["1", "dpmpp_2m"])


@pytest.mark.parametrize("solver", NEW_SOLVERS)
@pytest.mark.parametrize("kind", ["flux", "sd3"])
def test_step_cache_threshold_zero_under_the_new_solvers(kc, kind, solver):
    _, p16, _ = _weights(kind)
    pipe = _pipe(kind, p16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=CASES[kind][5])
    off, _ = _denoise(pipe, kind, cond, pooled, solver=solver)
    pipe.set_step_cache(0.0)
    on, it = _denoise(pipe, kind, cond, pooled, solver=solver)
    steps = CASES[kind][2]
    log = pipe.mmdit.step_cache_log
    assert torch.equal(on, off) and len(it) == steps
    assert len(log) == (2 * steps - 1 if solver == "heun" else steps) and not any(s for _, s in log)


@pytest.mark.parametrize("solver", NEW_SOLVERS)
def test_img2img_against_the_oracle(kc, solver):
    """denoise 0.6 on 6 FLUX steps: the trimmed schedule [sigma_2 .. 0] (2M has one second-order step on it)"""
    from diffusionkit_b200.config import VAEEncoderConfig
    from diffusionkit_b200.weights import init_params, vae_encoder_param_specs
    from oracle import sampler_ref as sr
    from oracle.vae_ref import VAEEncoderRef, encode_image_to_latents, read_image_array
    from tests.model_checks import _test_image, rel_l2

    kind, steps, denoise = "flux", 6, 0.6
    cfg, p16, _ = _weights(kind)
    ep16 = {k: v.to(bf16) for k, v in init_params(vae_encoder_param_specs(VAEEncoderConfig()), seed=9,
                                                   dtype=torch.float32).items()}
    pipe = _pipe(kind, p16, vae_encoder_params={k: v.to(DEV) for k, v in ep16.items()})
    img = _test_image(64, 128)                                  # both sides multiples of 64: no resize
    lat = (8, 16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=CASES[kind][5])
    latent, iter_time = pipe.denoise_latents(cond, pooled, num_steps=steps, seed=SEEDS, image_path=img,
                                             denoise=denoise, solver=solver)
    trim = int(steps * (1 - denoise))
    assert latent.shape == (len(SEEDS), *lat, 16) and len(iter_time) == steps - trim
    sampler = sr.FluxSamplerRef(1.0)
    sig = sr.get_sigmas(sampler, steps)[trim:]
    enc_ref = VAEEncoderRef({k: v.float() for k, v in ep16.items()})
    image = read_image_array(torch.from_numpy(img))
    x0s = []
    for s in SEEDS:
        noise = sr.get_noise(s, *lat)
        x_T = (encode_image_to_latents(enc_ref, image, noise) - 0.1159) * 0.3611       # FluxLatentFormat.process_in
        x0s.append(sampler.noise_scaling(float(sig[0]), noise, x_T))
    want = _oracle_latents(kind, solver, cfg, p16, cond, pooled, sig=sig, x0s=x0s)
    r = rel_l2(latent, want)
    print(f"img2img {solver}: final latent rel_l2 {r:.3e}")
    assert r <= 5e-2, f"img2img {solver} final latent rel_l2 {r:.3e}"


def test_fp8_with_the_new_solvers(kc):
    """FP8 composes: each solver's FP8 run stays within the FP8 pipeline bound of DESIGN.md §9 of its 16-bit run"""
    from tests.model_checks import psnr, rel_l2

    kind = "flux"
    _, p16, vp16 = _weights(kind)
    pipe = _pipe(kind, p16, vp16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=CASES[kind][5])
    for solver in NEW_SOLVERS:
        pipe.set_fp8(False)
        ref, _ = _denoise(pipe, kind, cond, pooled, solver=solver)
        pipe.set_fp8(True)
        got, _ = _denoise(pipe, kind, cond, pooled, solver=solver)
        ps = psnr(pipe.decode_latents_to_image(ref), pipe.decode_latents_to_image(got))
        print(f"fp8 {solver} vs 16-bit {solver}: latent rel_l2 {rel_l2(got, ref):.3e}, decoded psnr {ps:.1f} dB")
        assert bool(torch.isfinite(got).all()) and ps >= 20.0
        assert not np.array_equal(got.cpu().numpy(), ref.cpu().numpy())
    pipe.set_fp8(False)
