"""GPU checks of the stochastic samplers (DESIGN.md §16): dk_sampler_sde_step's noise against the contract's oracle
(tests/sde_ref.py) and its statistics, batch invariance, the update against its fp32 reference, argument errors, the
tiny FLUX and SD3.5-medium (CFG + skip-layer guidance) pipelines against the oracle under a launch census of their own,
reproducibility, eta = 0, the unchanged deterministic solvers and the rest of the stack."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
bf16, fp16 = torch.bfloat16, torch.float16
SDE = ["euler_ancestral", "dpmpp_2m_sde"]
LAT = (8, 12)
SEEDS = [11, 12]
STEPS = 4


@pytest.fixture(scope="module")
def kc():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    from tests import kernel_checks

    kernel_checks._setup()
    return kernel_checks


def _seeds(vals):
    from diffusionkit_b200.pipeline import seeds_tensor

    return seeds_tensor(vals, DEV)


def _step(x, d_prev, xin, out, coef, seeds, step, sigma=0.6875, cfg=0.0, slg=0.0):
    from diffusionkit_b200.pipeline import sampler_sde_step

    a, b, c, n = coef
    return sampler_sde_step(x, d_prev, xin, out, sigma, a, b, c, n, cfg, slg, seeds, step)


def _inputs(dtype, B, n_img, reps, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn((B, n_img), generator=g, device=DEV)
    xin = torch.randn((reps * B, n_img), generator=g, device=DEV).to(dtype)
    out = torch.randn((reps * B, n_img), generator=g, device=DEV).to(dtype)
    return x, xin, out


def _cfg_slg(reps):
    return {1: (0.0, 0.0), 2: (5.0, 0.0), 3: (4.5, 2.5)}[reps]


def _noise(B, n_img, seeds, step, reps=1, dtype=bf16):
    """z alone: (a, b, c, n) = (0, 0, 0, 1)"""
    x, xin, out = _inputs(dtype, B, n_img, reps, 1)
    cfg, slg = _cfg_slg(reps)
    _step(x, None, xin, out, (0.0, 0.0, 0.0, 1.0), _seeds(seeds), step, cfg=cfg, slg=slg)
    torch.cuda.synchronize()
    return x


# ------------------------------------------------------------------------------------------------ the noise
def test_noise_matches_the_contract(kc):
    from tests.sde_ref import normals

    n_img = 16 * 8 * 12
    for seeds in ([5], [0, 2 ** 32 + 7, 2 ** 64 - 1]):
        for step in (0, 1, 27):
            z = _noise(len(seeds), n_img, seeds, step).double().cpu()
            for b, s in enumerate(seeds):
                want = torch.from_numpy(normals(s, step, n_img))
                err = (z[b] - want).abs() - (1e-6 * want.abs().clamp(min=1.0) + 1e-6)
                assert float(err.max()) <= 0.0, (s, step, float((z[b] - want).abs().max()))


def test_noise_statistics(kc):
    """16.8 M draws: moments within 5 standard errors of N(0, 1), and no lag-1 correlation between neighbouring
    elements, steps or seeds"""
    n_img = 128 * 128 * 16 * 16
    seeds = [1, 2, 3, 4]
    z = _noise(4, n_img, seeds, 0).double()
    N = z.numel()
    m = float(z.mean())
    c = z - m
    var = float((c * c).mean())
    skew = float((c ** 3).mean()) / var ** 1.5
    kurt = float((c ** 4).mean()) / var ** 2 - 3.0
    print(f"N={N}: mean {m:.2e}, var {var:.6f}, skew {skew:.2e}, excess kurtosis {kurt:.2e}")
    assert abs(m) <= 5 / math.sqrt(N) and abs(var - 1) <= 5 * math.sqrt(2 / N)
    assert abs(skew) <= 5 * math.sqrt(6 / N) and abs(kurt) <= 5 * math.sqrt(24 / N)

    def corr(u, v):
        u, v = u - u.mean(), v - v.mean()
        return float((u * v).mean() / (u.std() * v.std()))

    flat = z.reshape(-1)
    pairs = {"elements": corr(flat[:-1], flat[1:]), "seeds": corr(z[0], z[1]),
             "steps": corr(z[0], _noise(1, n_img, seeds[:1], 1).double()[0])}
    print("lag-1 correlations:", {k: f"{v:.2e}" for k, v in pairs.items()})
    for k, v in pairs.items():
        n = flat.numel() - 1 if k == "elements" else n_img
        assert abs(v) <= 5 / math.sqrt(n), (k, v)


@pytest.mark.parametrize("reps", [1, 2, 3])
def test_noise_is_batch_invariant(kc, reps):
    n_img = 16 * 8 * 12
    alone = _noise(1, n_img, [7], 3, reps)[0]
    first = _noise(3, n_img, [7, 8, 9], 3, reps)[0]
    last = _noise(3, n_img, [8, 9, 7], 3, reps)[2]
    assert torch.equal(alone, first) and torch.equal(alone, last)


# ------------------------------------------------------------------------------------------------ the update
@pytest.mark.parametrize("dtype", [bf16, fp16])
@pytest.mark.parametrize("reps", [1, 2, 3])
def test_update_against_its_reference(kc, dtype, reps):
    from tests.sde_ref import ref_sde_step

    B, n_img = 3, 16 * 8 * 12
    cfg, slg = _cfg_slg(reps)
    seeds = _seeds([3, 2 ** 40 + 1, 99])
    for coef, keep in [((0.5, 0.4, 0.0, 0.3), False), ((0.5, 0.45, -0.05, 0.3), True), ((0.0, 1.0, 0.0, 0.0), True),
                       ((0.7, 0.3, 0.0, 0.0), True)]:
        x, xin, out = _inputs(dtype, B, n_img, reps, 2)
        d_prev = torch.randn_like(x) if keep else None
        want, den = ref_sde_step(x, d_prev, xin, out, 0.6875, *coef, cfg, slg, seeds, 5)
        got_prev = None if d_prev is None else d_prev.clone()
        got = _step(x.clone(), got_prev, xin, out, coef, seeds, 5, cfg=cfg, slg=slg)
        kc._assert_close(f"sde {coef} {reps}", got, want, 1e-6)
        if keep:
            kc._assert_close(f"sde d_prev {coef} {reps}", got_prev, den, 1e-6)


def test_c_zero_does_not_read_d_prev(kc):
    from tests.sde_ref import ref_sde_step

    x, xin, out = _inputs(bf16, 2, 1536, 1, 3)
    seeds = _seeds([1, 2])
    d_prev = torch.full_like(x, float("nan"))
    got = _step(x.clone(), d_prev, xin, out, (0.75, 0.25, 0.0, 0.5), seeds, 0)
    assert bool(torch.isfinite(got).all()) and bool(torch.isfinite(d_prev).all())
    kc._assert_close("sde c = 0", got, ref_sde_step(x, None, xin, out, 0.6875, 0.75, 0.25, 0.0, 0.5, 0.0, 0.0, seeds,
                                                    0)[0], 1e-6)


def test_update_at_the_c3_shape(kc):
    """SD3 under CFG 5, 4 x 1024^2 (latent 128^2), a second-order step with noise"""
    from tests.sde_ref import ref_sde_step

    x, xin, out = _inputs(fp16, 4, 128 * 128 * 16, 2, 4)
    d_prev = torch.randn_like(x)
    seeds = _seeds([0, 1, 2, 3])
    want, den = ref_sde_step(x, d_prev, xin, out, 0.3, 0.6, 0.5, -0.1, 0.2, 5.0, 0.0, seeds, 12)
    got = _step(x.clone(), d_prev, xin, out, (0.6, 0.5, -0.1, 0.2), seeds, 12, sigma=0.3, cfg=5.0)
    kc._assert_close("sde c3", got, want, 1e-6)
    kc._assert_close("sde c3 d_prev", d_prev, den, 1e-6)


def test_argument_errors_launch_nothing(kc):
    from diffusionkit_b200 import DkError, ops

    c = ops.ctx(0)
    seeds = _seeds([1])
    x, xin, out = _inputs(bf16, 1, 64, 1, 5)
    _, xin4, out4 = _inputs(bf16, 1, 64, 4, 5)
    _, xin3, out3 = _inputs(bf16, 1, 64, 3, 5)
    n0 = c.launches
    for args, msg in [((x, None, xin4, out4, (1.0, 0.0, 0.0, 0.0), seeds, 0), "reps must be"),
                      ((x, None, xin, out, (float("nan"), 0.0, 0.0, 0.0), seeds, 0), "finite"),
                      ((x, None, xin, out, (1.0, 0.0, 0.0, float("inf")), seeds, 0), "finite"),
                      ((x, None, xin3, out3, (1.0, 0.0, 0.0, 0.0), seeds, 0), "does not match"),
                      ((x, None, xin, out, (1.0, 0.0, 0.5, 0.0), seeds, 0), "needs d_prev")]:
        with pytest.raises(DkError, match=msg):
            _step(*args)
    with pytest.raises(DkError, match="skip-layer guidance needs reps = 3"):
        _step(x, None, xin, out, (1.0, 0.0, 0.0, 0.0), seeds, 0, slg=2.0)
    assert c.launches == n0


# ------------------------------------------------------------------------------------------------ pipelines
@pytest.fixture
def sde_census(kc, monkeypatch):
    """tests/launch_parity's census over every ops launch, plus pipeline.sampler_sde_step (sde_ref.census_check)"""
    from diffusionkit_b200 import pipeline
    from tests import launch_parity as lp
    from tests.sde_ref import census_check

    monkeypatch.setitem(lp.CHECKS, "sampler_sde_step", census_check)
    monkeypatch.setitem(lp.WRITES, "sampler_sde_step", ["x", "d_prev"])
    c = lp.Census()
    with lp.census(c):
        monkeypatch.setattr(pipeline, "sampler_sde_step", c._wrap("sampler_sde_step", pipeline.sampler_sde_step))
        yield c


def _flux():
    from tests.test_solvers_gpu import _weights

    return _weights("flux")


def _flux_pipe(p16, vp16=None, **kw):
    from tests.test_solvers_gpu import _pipe

    return _pipe("flux", p16, vp16, **kw)


def _flux_oracle(solver, cfg, p16, cond, pooled, eta=1.0, sig=None, x0s=None, steps=STEPS):
    from oracle import sampler_ref as sr
    from oracle.mmdit_ref import MMDiTRef
    from tests import sde_ref, solver_ref
    from tests.oracle_bridge import ref_config

    sampler = sr.FluxSamplerRef(1.0)
    sig = sr.get_sigmas(sampler, steps) if sig is None else sig
    outs = []
    for i, s in enumerate(SEEDS):
        ref = MMDiTRef(ref_config(cfg), {k: v.float() for k, v in p16.items()})
        x0 = (sampler.noise_scaling(float(sig[0]), sr.get_noise(s, *LAT), sr.get_empty_latent(*LAT))
              if x0s is None else x0s[i])
        args = (lambda xin, c, t: ref(xin, c, t), ref.cache_modulation_params, x0, sig, cond[[i]].float(),
                pooled[[i]].float(), 0.0, bf16)
        if solver == "euler":
            x = sr.sample_euler(*args)
        elif solver == "dpmpp_2m":
            x = solver_ref.sample_dpmpp_2m(*args)
        else:
            x = getattr(sde_ref, "sample_" + solver)(*args, seed=s, eta=eta)
        outs.append(sr.process_out(x, "flux"))
    return torch.cat(outs)


def _check(latent, want, what, img=None, floor=30.0):
    from tests.model_checks import psnr, rel_l2

    r = rel_l2(latent, want)
    msg = f"{what}: final latent rel_l2 {r:.3e}"
    if img is not None:
        ps = psnr(*img)
        msg += f", decoded psnr {ps:.1f} dB"
        assert ps >= floor, msg
    print(msg)
    assert r <= 5e-2, msg


@pytest.mark.parametrize("solver", SDE)
def test_flux_pipeline_against_the_oracle_under_a_census(sde_census, solver):
    from oracle.vae_ref import VAEDecoderRef, decode_latents_to_image

    cfg, p16, vp16 = _flux()
    pipe = _flux_pipe(p16, vp16)
    pipe.mmdit.use_cuda_graphs = pipe.decoder.use_cuda_graphs = False
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=16)
    sde_census.run = f"flux-{solver}"
    latent, it = pipe.denoise_latents(cond, pooled, num_steps=STEPS, latent_size=LAT, seed=SEEDS, solver=solver,
                                      eta=1.0)
    torch.cuda.synchronize()
    steps = [r for r in sde_census.records if r["op"] == "sampler_sde_step"]
    assert len(steps) == STEPS and len(it) == STEPS
    assert {r["info"]["d_prev"] for r in steps} == {solver == "dpmpp_2m_sde"}
    want = _flux_oracle(solver, cfg, p16, cond, pooled)
    img_want = decode_latents_to_image(VAEDecoderRef({k: v.float() for k, v in vp16.items()}), want.to(bf16).float())
    _check(latent, want, f"flux {solver} eta 1", (img_want, pipe.decode_latents_to_image(latent)))
    # the noise matters: eta = 1 is far from eta = 0 in the oracle
    from tests.model_checks import rel_l2

    print(f"flux {solver}: oracle eta 1 vs eta 0 rel_l2 {rel_l2(want, _flux_oracle(solver, cfg, p16, cond, pooled, 0.0)):.3e}")


@pytest.mark.parametrize("solver", SDE)
def test_sd35_medium_cfg_slg_against_the_oracle_under_a_census(sde_census, solver):
    from oracle import sampler_ref as sr
    from oracle.vae_ref import VAEDecoderRef, decode_latents_to_image
    from tests import test_sd35_medium_gpu as m
    from tests.sde_ref import sample_slg

    cfg = m._cfg()
    p16, vp16 = m._weights(cfg), m._vae_weights()
    pipe = m._pipe(cfg, p16, vp16)
    pipe.mmdit.use_cuda_graphs = pipe.decoder.use_cuda_graphs = False
    cond, pooled = m._cond(pipe)
    slg = m._slg()                                              # steps 1 and 2 of 4
    sde_census.run = f"sd35-{solver}"
    latent, _ = pipe.denoise_latents(cond, pooled, num_steps=STEPS, cfg_weight=m.CFGW, latent_size=LAT, seed=SEEDS,
                                     solver=solver, slg=slg)
    torch.cuda.synchronize()
    info = [r["info"] for r in sde_census.records if r["op"] == "sampler_sde_step"]
    assert [i["reps"] for i in info] == [2, 3, 3, 2] and all(i["cfg"] for i in info)
    smp = sr.ModelSamplingDiscreteFlowRef(3.0)
    sig = sr.get_sigmas(smp, STEPS)
    outs = []
    for i, s in enumerate(SEEDS):
        x0 = smp.noise_scaling(float(sig[0]), sr.get_noise(s, *LAT), sr.get_empty_latent(*LAT))
        idx = [i, i + len(SEEDS)]
        x = sample_slg(solver, m._xref(cfg, p16), x0, sig, cond[idx].float().cpu(), pooled[idx].float().cpu(), m.CFGW,
                       fp16, seed=s, scale=slg.scale, layers=slg.layers, start=slg.start, end=slg.end)
        outs.append(sr.process_out(x, "sd3"))
    want = torch.cat(outs)
    img_want = decode_latents_to_image(VAEDecoderRef({k: v.float() for k, v in vp16.items()}), want.to(fp16).float())
    _check(latent, want, f"sd35 cfg+slg {solver}", (img_want, pipe.decode_latents_to_image(latent)), floor=20.0)


def test_generate_image_logs_the_noise(kc):
    _, p16, vp16 = _flux()
    pipe = _flux_pipe(p16, vp16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=1, text_len=16)
    kw = dict(num_steps=STEPS, latent_size=LAT, verbose=False, conditioning=cond, pooled_conditioning=pooled)
    _, log = pipe.generate_image("", seed=5, solver="dpmpp_2m_sde", **kw)
    assert log["denoising"]["sde"] == {"solver": "dpmpp_2m_sde", "eta": 1.0, "seeds": [5]}
    assert log["denoising"]["solver"] == "dpmpp_2m_sde" and log["denoising"]["nfe"] == STEPS
    _, log = pipe.generate_image("", seed=None, solver="euler_ancestral", eta=0.5, **kw)
    assert log["denoising"]["sde"]["eta"] == 0.5 and len(log["denoising"]["sde"]["seeds"]) == 1
    _, log = pipe.generate_image("", seed=5, solver="dpmpp_2m", **kw)
    assert "sde" not in log["denoising"]


def test_seed_batches_reruns_and_graphs_are_reproducible(kc, monkeypatch):
    """[3, 7] together equal 3 alone and 7 alone bit for bit where the tiny forward is batch-invariant (checked first
    with Euler); graphs and eager give the same bits; reruns repeat"""
    _, p16, _ = _flux()
    runs = {}
    for graphs in ("1", "0"):
        monkeypatch.setenv("DK_CUDA_GRAPHS", graphs)
        pipe = _flux_pipe(p16)
        cond, pooled = pipe.synthetic_text_embeddings(n_images=2, text_len=16)

        def run(seeds, solver, rows):
            lat, _ = pipe.denoise_latents(cond[rows], pooled[rows], num_steps=STEPS, latent_size=LAT, seed=seeds,
                                          solver=solver)
            torch.cuda.synchronize()
            return lat.clone()

        invariant = all(torch.equal(run([3, 7], "euler", [0, 1])[k], run([s], "euler", [k])[0])
                        for k, s in enumerate([3, 7]))
        for solver in SDE:
            both = run([3, 7], solver, [0, 1])
            assert torch.equal(both, run([3, 7], solver, [0, 1])), (graphs, solver)
            runs[graphs, solver] = both
            if invariant:
                for k, s in enumerate([3, 7]):
                    assert torch.equal(both[k], run([s], solver, [k])[0]), (graphs, solver, s)
        print(f"graphs={graphs}: tiny forward batch-invariant: {invariant}")
        del pipe
    for solver in SDE:
        assert torch.equal(runs["1", solver], runs["0", solver]), solver


@pytest.mark.parametrize("kind", ["flux", "sd3"])
def test_eta_zero(kc, kind):
    """dpmpp_2m_sde at eta 0 is dpmpp_2m bit for bit; euler_ancestral at eta 0 is the oracle's Euler"""
    from tests import test_solvers_gpu as s

    cfg, p16, _ = s._weights(kind)
    pipe = s._pipe(kind, p16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=s.CASES[kind][5])
    two_m, _ = s._denoise(pipe, kind, cond, pooled, solver="dpmpp_2m")
    sde, _ = s._denoise(pipe, kind, cond, pooled, solver="dpmpp_2m_sde", eta=0.0)
    assert torch.equal(two_m, sde)
    anc, _ = s._denoise(pipe, kind, cond, pooled, solver="euler_ancestral", eta=0.0)
    _check(anc, s._oracle_latents(kind, "euler", cfg, p16, cond, pooled), f"{kind} euler_ancestral eta 0 vs euler")


def test_deterministic_solvers_are_unchanged(kc):
    """Euler, Heun and 2M launch no stochastic step and issue the same launches as before: the op list of each is
    the same with and without the stochastic solvers having run in the same process"""
    from diffusionkit_b200 import ops
    from tests import test_solvers_gpu as s

    _, p16, _ = s._weights("sd3")
    pipe = s._pipe("sd3", p16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=s.CASES["sd3"][5])

    def run(solver):
        n0 = ops.launch_count()
        lat, _ = s._denoise(pipe, "sd3", cond, pooled, solver=solver)
        return lat, ops.launch_count() - n0

    for k in ("euler", "heun", "dpmpp_2m"):                      # the first run of a shape captures the forward's graph
        run(k)
    first = {k: run(k) for k in ("euler", "heun", "dpmpp_2m")}
    for solver in SDE:
        run(solver)
    for k, (lat, n) in first.items():
        lat2, n2 = run(k)
        assert torch.equal(lat, lat2) and n == n2, k


# ------------------------------------------------------------------------------------------------ the rest of the stack
def test_img2img_against_the_oracle(kc):
    from diffusionkit_b200.config import VAEEncoderConfig
    from diffusionkit_b200.weights import init_params, vae_encoder_param_specs
    from oracle import sampler_ref as sr
    from oracle.vae_ref import VAEEncoderRef, encode_image_to_latents, read_image_array
    from tests.model_checks import _test_image

    cfg, p16, _ = _flux()
    ep16 = {k: v.to(bf16) for k, v in init_params(vae_encoder_param_specs(VAEEncoderConfig()), seed=9,
                                                   dtype=torch.float32).items()}
    pipe = _flux_pipe(p16, vae_encoder_params={k: v.to(DEV) for k, v in ep16.items()})
    img = _test_image(64, 128)                                  # both sides multiples of 64: no resize
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=16)
    steps, denoise = 5, 0.6
    trim = int(steps * (1 - denoise))
    sig = sr.get_sigmas(sr.FluxSamplerRef(1.0), steps)[trim:]
    enc_ref = VAEEncoderRef({k: v.float() for k, v in ep16.items()})
    image = read_image_array(torch.from_numpy(img))
    x0s = []
    for s in SEEDS:
        noise = sr.get_noise(s, 8, 16)
        x_T = (encode_image_to_latents(enc_ref, image, noise) - 0.1159) * 0.3611
        x0s.append(sr.FluxSamplerRef(1.0).noise_scaling(float(sig[0]), noise, x_T))
    for solver in SDE:
        latent, it = pipe.denoise_latents(cond, pooled, num_steps=steps, seed=SEEDS, image_path=img, denoise=denoise,
                                          solver=solver)
        assert latent.shape == (len(SEEDS), 8, 16, 16) and len(it) == steps - trim
        _check(latent, _flux_oracle(solver, cfg, p16, cond, pooled, sig=sig, x0s=x0s), f"img2img 0.6 {solver}")


def test_step_cache_fp8_and_lora(kc):
    from tests.lora_fixtures import kohya_dict, make_factors, upstream_modules
    from tests.model_checks import psnr

    cfg, p16, vp16 = _flux()
    pipe = _flux_pipe(p16, vp16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=16)

    def run(solver):
        lat, _ = pipe.denoise_latents(cond, pooled, num_steps=STEPS, latent_size=LAT, seed=SEEDS, solver=solver)
        torch.cuda.synchronize()
        return lat.clone()

    for solver in SDE:
        base = run(solver)
        pipe.set_step_cache(0.0)
        assert torch.equal(run(solver), base), f"step cache at threshold 0 under {solver}"
        assert not any(skipped for _, skipped in pipe.mmdit.step_cache_log)
        pipe.set_step_cache(None)
        pipe.set_fp8(True)
        got = run(solver)
        pipe.set_fp8(False)
        ps = psnr(pipe.decode_latents_to_image(base), pipe.decode_latents_to_image(got))
        print(f"fp8 {solver} vs 16-bit: decoded psnr {ps:.1f} dB")
        assert bool(torch.isfinite(got).all()) and ps >= 20.0
        name = pipe.load_lora_weights(kohya_dict(make_factors(upstream_modules(cfg), 4, seed=3)), scale=1.0)
        merged = run(solver)
        pipe.unload_lora_weights(name)
        assert bool(torch.isfinite(merged).all()) and not torch.equal(merged, base)
        assert torch.equal(run(solver), base), f"LoRA unloaded under {solver}"


def test_kontext_reference_and_redux_tokens(kc):
    from diffusionkit_b200.config import tiny_siglip_config
    from tests.test_solvers_gpu import _weights

    cfg, p16, _ = _weights("flux")
    pipe = _flux_pipe(p16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=16)
    ref = torch.randn((1, 8, 8, 16), generator=torch.Generator().manual_seed(2)).to(DEV)
    kw = dict(num_steps=STEPS, latent_size=LAT, seed=SEEDS)
    plain, _ = pipe.denoise_latents(cond, pooled, solver="dpmpp_2m_sde", **kw)
    plain = plain.clone()
    two_m, _ = pipe.denoise_latents(cond, pooled, solver="dpmpp_2m", reference_latents=ref, **kw)
    two_m = two_m.clone()
    sde0, _ = pipe.denoise_latents(cond, pooled, solver="dpmpp_2m_sde", eta=0.0, reference_latents=ref, **kw)
    assert torch.equal(sde0, two_m), "a Kontext reference under dpmpp_2m_sde at eta 0"
    with_ref, _ = pipe.denoise_latents(cond, pooled, solver="dpmpp_2m_sde", reference_latents=ref, **kw)
    assert bool(torch.isfinite(with_ref).all()) and not torch.equal(with_ref, plain)
    # Redux: redux_image= equals the same tokens passed as conditioning, bit for bit
    pipe.load_redux(siglip_config=tiny_siglip_config())
    from tests.model_checks import _test_image

    im = _test_image(pipe.siglip.config.image_size, pipe.siglip.config.image_size)
    got, _ = pipe.denoise_latents(cond, pooled, solver="euler_ancestral", redux_image=im, **kw)
    got = got.clone()
    tok = pipe.encode_redux(im)
    cat = torch.cat([cond.to(DEV), tok.expand(len(SEEDS), -1, -1)], dim=1)
    want, _ = pipe.denoise_latents(cat, pooled, solver="euler_ancestral", **kw)
    assert torch.equal(got, want)
