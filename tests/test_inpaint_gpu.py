"""GPU checks of masked inpainting (DESIGN.md §17): dk_inpaint_blend and dk_inpaint_paste against their references
(tests/inpaint_ref.py) and their argument errors; the tiny FLUX and SD3.5-medium (CFG + skip-layer guidance)
pipelines with every solver against the masked oracle under a launch census of their own; the exact invariants
(unmasked latents end at the encoded source and unmasked pixels are the source, with every solver and the rest of the
stack); reproducibility; and that a call without a mask launches nothing new."""
from dataclasses import replace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
bf16, fp16 = torch.bfloat16, torch.float16
SOLVERS = ["euler", "heun", "dpmpp_2m", "euler_ancestral", "dpmpp_2m_sde"]
SEEDS = [11, 12]
STEPS = 4
HP, WP = 64, 128                       # the source image; latent 8 x 16


@pytest.fixture(scope="module")
def kc():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    from tests import kernel_checks

    kernel_checks._setup()
    return kernel_checks


def _mask(H=HP, W=WP, value=255):
    """a rectangle plus a 3-pixel vertical line, white on black"""
    m = np.zeros((H, W), dtype=np.uint8)
    m[H // 4:H // 2 + 5, W // 5:W // 2] = value
    m[:, W - 27:W - 24] = value
    return m


def _source():
    from tests.model_checks import _test_image

    return _test_image(HP, WP)


# ------------------------------------------------------------------------------------------------ kernels
def _blend_inputs(shape, seed, p=0.4):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x, eps, x0 = (torch.randn(shape, generator=g, device=DEV) for _ in range(3))
    mask = (torch.rand(shape[1:3], generator=g, device=DEV) < p).to(torch.uint8)
    return x, eps, x0, mask


@pytest.mark.parametrize("shape", [(2, 8, 12, 16), (4, 128, 128, 16), (3, 5, 7, 4)])
def test_blend_against_its_reference(kc, shape):
    from diffusionkit_b200 import ops
    from diffusionkit_b200.inpaint import inpaint_blend
    from tests.inpaint_ref import ref_blend

    x, eps, x0, mask = _blend_inputs(shape, 1)
    rep = (mask != 0)[None, :, :, None].expand(shape)
    for a in (0.0, 0.3125, 0.75, 1.0):
        b = 1.0 - a
        got = inpaint_blend(x.clone(), eps, x0, mask, a, b)
        assert torch.equal(got[rep], x[rep]), "a repainted element changed"
        kc._assert_close(f"blend a={a}", got, ref_blend(x, eps, x0, mask, a, b), 1e-6)
        if a == 0.0:
            assert torch.equal(got[~rep], x0[~rep]), "a = 0, b = 1 must return x0 exactly"
        # rounding for rounding the img2img start (dk_axpby_f32) where nothing is repainted
        all_kept = inpaint_blend(x.clone(), eps, x0, torch.zeros_like(mask), a, b)
        assert torch.equal(all_kept, ops.axpby(eps, x0, a, b))


def test_paste_is_exact(kc):
    from diffusionkit_b200.inpaint import inpaint_paste
    from tests.inpaint_ref import ref_paste

    g = torch.Generator(device=DEV).manual_seed(2)
    for B, H, W in ((2, 64, 128), (4, 1024, 1024), (1, 8, 4)):
        img = torch.randint(0, 256, (B, H, W, 3), generator=g, device=DEV, dtype=torch.uint8)
        src = torch.randint(0, 256, (H, W, 3), generator=g, device=DEV, dtype=torch.uint8)
        for p in (0.0, 0.3, 1.0):
            mask = (torch.rand((H, W), generator=g, device=DEV) < p).to(torch.uint8)
            got = inpaint_paste(img.clone(), src, mask)
            assert torch.equal(got, ref_paste(img, src, mask)), (B, H, W, p)


def test_argument_errors_launch_nothing(kc):
    from diffusionkit_b200 import DkError, ops
    from diffusionkit_b200.inpaint import inpaint_blend, inpaint_paste

    c = ops.ctx(0)
    x, eps, x0, mask = _blend_inputs((1, 4, 4, 16), 3)
    x6, e6, z6, m6 = _blend_inputs((1, 4, 4, 6), 3)
    buf = torch.zeros(x.numel() + 1, device=DEV)
    off = buf[1:].view(x.shape)                                     # contiguous, 4 bytes past a 16-byte boundary
    img = torch.zeros((1, 3, 3, 3), dtype=torch.uint8, device=DEV)
    n0 = c.launches
    for args, msg in [((x6, e6, z6, m6, 0.5, 0.5), "multiple of 4"),
                      ((x, eps, x0, mask, float("nan"), 0.5), "finite"),
                      ((x, eps, x0, mask, 0.5, float("inf")), "finite"),
                      ((off, eps, x0, mask, 0.5, 0.5), "16-byte aligned")]:
        with pytest.raises(DkError, match=msg):
            inpaint_blend(*args)
    with pytest.raises(DkError, match="multiple of 4"):
        inpaint_paste(img, img[0].clone(), torch.zeros((3, 3), dtype=torch.uint8, device=DEV))
    assert c.launches == n0


# ------------------------------------------------------------------------------------------------ pipelines
def _census_wrap(monkeypatch, c):
    """tests/launch_parity's census plus the two inpaint launches (inpaint_ref.census_check_*), as test_sde_gpu does
    for its stochastic step"""
    from diffusionkit_b200 import inpaint, pipeline
    from tests import launch_parity as lp
    from tests import sde_ref
    from tests.inpaint_ref import census_check_blend, census_check_paste

    for name, check, writes in (("inpaint_blend", census_check_blend, ["x"]),
                                ("inpaint_paste", census_check_paste, ["img"]),
                                ("sampler_sde_step", sde_ref.census_check, ["x", "d_prev"])):
        monkeypatch.setitem(lp.CHECKS, name, check)
        monkeypatch.setitem(lp.WRITES, name, writes)
    monkeypatch.setattr(inpaint, "inpaint_blend", c._wrap("inpaint_blend", inpaint.inpaint_blend))
    monkeypatch.setattr(inpaint, "inpaint_paste", c._wrap("inpaint_paste", inpaint.inpaint_paste))
    monkeypatch.setattr(pipeline, "sampler_sde_step", c._wrap("sampler_sde_step", pipeline.sampler_sde_step))


def _encoder_weights(dtype):
    from diffusionkit_b200.config import VAEEncoderConfig
    from diffusionkit_b200.weights import init_params, vae_encoder_param_specs

    return {k: v.to(dtype) for k, v in init_params(vae_encoder_param_specs(VAEEncoderConfig()), seed=9,
                                                   dtype=torch.float32).items()}


def _oracle_starts(ep16, img, sig, lat, shift, scale):
    """per seed: (eps, x0 in process_in, the img2img start) from the oracle encoder"""
    from oracle import sampler_ref as sr
    from oracle.vae_ref import VAEEncoderRef, encode_image_to_latents, read_image_array

    enc = VAEEncoderRef({k: v.float() for k, v in ep16.items()})
    image = read_image_array(torch.from_numpy(img))
    out = []
    for s in SEEDS:
        eps = sr.get_noise(s, *lat)
        x0 = (encode_image_to_latents(enc, image, eps) - shift) * scale
        out.append((eps, x0, float(sig[0]) * eps + (1.0 - float(sig[0])) * x0))
    return out


def _check_masked(latent, want, dtype, vp16, pipe, pixmask, what, floor):
    from oracle.vae_ref import VAEDecoderRef, decode_latents_to_image
    from tests.model_checks import psnr, rel_l2

    r = rel_l2(latent, want)
    img_want = decode_latents_to_image(VAEDecoderRef({k: v.float() for k, v in vp16.items()}), want.to(dtype).float())
    got = pipe.decode_latents_to_image(latent)
    sel = torch.from_numpy(pixmask.astype(bool))
    ps = psnr(img_want[:, sel], got.cpu()[:, sel])
    msg = f"{what}: final latent rel_l2 {r:.3e}, decoded psnr on masked pixels {ps:.1f} dB"
    print(msg)
    assert r <= 5e-2 and ps >= floor, msg


def _flux_pipe(p16, vp16=None, **kw):
    from tests.test_solvers_gpu import _pipe

    return _pipe("flux", p16, vp16, vae_encoder_params={k: v.to(DEV) for k, v in _encoder_weights(bf16).items()},
                 **kw)


@pytest.mark.parametrize("denoise", [1.0, 0.6])
def test_flux_against_the_oracle_under_a_census(kc, monkeypatch, denoise):
    from diffusionkit_b200.inpaint import prepare_mask
    from oracle import sampler_ref as sr
    from oracle.mmdit_ref import MMDiTRef
    from tests import inpaint_ref
    from tests import launch_parity as lp
    from tests.oracle_bridge import ref_config
    from tests.test_solvers_gpu import _weights

    cfg, p16, vp16 = _weights("flux")
    pipe = _flux_pipe(p16, vp16)
    pipe.mmdit.use_cuda_graphs = pipe.decoder.use_cuda_graphs = False
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=16)
    img, mask = _source(), _mask()
    m = prepare_mask(mask, (WP, HP))
    hidden = pipe._encode_u8(img)                   # the VAE encoder runs before the census: not this feature's launches
    monkeypatch.setattr(pipe, "_encode_u8", lambda arr: hidden)
    steps = 5
    sig = sr.get_sigmas(sr.FluxSamplerRef(1.0), steps)[int(steps * (1 - denoise)):]
    starts = _oracle_starts(_encoder_weights(bf16), img, sig, (HP // 8, WP // 8), 0.1159, 0.3611)
    c = lp.Census()
    with lp.census(c):
        _census_wrap(monkeypatch, c)
        for solver in SOLVERS:
            c.run = f"flux-{solver}-{denoise}"
            n0 = len(c.records)
            latent, it = pipe.denoise_latents(cond, pooled, num_steps=steps, seed=SEEDS, image_path=img,
                                              denoise=denoise, solver=solver, mask_image=mask)
            torch.cuda.synchronize()
            blends = [r for r in c.records[n0:] if r["op"] == "inpaint_blend"]
            assert len(blends) == len(it) == len(sig) - 1
            outs = []
            for i, s in enumerate(SEEDS):
                ref = MMDiTRef(ref_config(cfg), {k: v.float() for k, v in p16.items()})
                eps, x0, start = starts[i]
                x = inpaint_ref.sample_model(solver, lambda xin, cc, t: ref(xin, cc, t), ref.cache_modulation_params,
                                             start, sig, cond[[i]].float(), pooled[[i]].float(), 0.0, bf16, eps=eps,
                                             x0=x0, mask=torch.from_numpy(m.latent), seed=s)
                outs.append(sr.process_out(x, "flux"))
            _check_masked(latent, torch.cat(outs), bf16, vp16, pipe, m.pixels, f"flux {solver} denoise {denoise}",
                          30.0)
        c.run = f"flux-generate-{denoise}"                     # the decode and the paste-back
        pipe.generate_image("", num_steps=steps, seed=SEEDS, image_path=img, denoise=denoise, mask_image=mask,
                            verbose=False, conditioning=cond, pooled_conditioning=pooled)
        assert [r["op"] for r in c.records].count("inpaint_paste") == 1
    print(c.table())


def test_sd35_medium_cfg_slg_against_the_oracle_under_a_census(kc, monkeypatch):
    from diffusionkit_b200.inpaint import prepare_mask
    from oracle import sampler_ref as sr
    from tests import inpaint_ref
    from tests import launch_parity as lp
    from tests import test_sd35_medium_gpu as m35

    cfg = m35._cfg()
    p16, vp16 = m35._weights(cfg), m35._vae_weights()
    ep16 = _encoder_weights(fp16)
    pipe = m35._pipe(cfg, p16, vp16, vae_encoder_params={k: v.to(DEV) for k, v in ep16.items()})
    pipe.mmdit.use_cuda_graphs = pipe.decoder.use_cuda_graphs = False
    cond, pooled = m35._cond(pipe)
    slg = m35._slg()
    img, mask = _source(), _mask()
    m = prepare_mask(mask, (WP, HP))
    hidden = pipe._encode_u8(img)
    monkeypatch.setattr(pipe, "_encode_u8", lambda arr: hidden)
    smp = sr.ModelSamplingDiscreteFlowRef(3.0)
    sig = sr.get_sigmas(smp, STEPS)
    starts = _oracle_starts(ep16, img, sig, (HP // 8, WP // 8), 0.0609, 1.5305)
    c = lp.Census()
    with lp.census(c):
        _census_wrap(monkeypatch, c)
        for solver in SOLVERS:
            c.run = f"sd35-{solver}"
            latent, _ = pipe.denoise_latents(cond, pooled, num_steps=STEPS, cfg_weight=m35.CFGW, seed=SEEDS,
                                             image_path=img, solver=solver, slg=slg, mask_image=mask)
            torch.cuda.synchronize()
            outs = []
            for i, s in enumerate(SEEDS):
                eps, x0, start = starts[i]
                idx = [i, i + len(SEEDS)]
                x = inpaint_ref.sample_slg(solver, m35._xref(cfg, p16), start, sig, cond[idx].float().cpu(),
                                           pooled[idx].float().cpu(), m35.CFGW, fp16, eps=eps, x0=x0,
                                           mask=torch.from_numpy(m.latent), seed=s, scale=slg.scale,
                                           layers=slg.layers, start=slg.start, end=slg.end)
                outs.append(sr.process_out(x, "sd3"))
            _check_masked(latent, torch.cat(outs), fp16, vp16, pipe, m.pixels, f"sd35 cfg+slg {solver}", 20.0)


# ------------------------------------------------------------------------------------------------ exact invariants
def _x0_out(pipe, img, seeds):
    """process_out(x0) of each seed with the pipeline's own kernels: the bits the unmasked latents must end at"""
    from diffusionkit_b200 import ops

    hidden = pipe._encode_u8(img)
    H, W = hidden.shape[1], hidden.shape[2]
    noise = pipe._get_noise_batch(list(seeds), pipe.get_empty_latent(H, W)).to(DEV).contiguous()
    lf = pipe.latent_format
    x0 = torch.empty_like(noise)
    for b in range(len(seeds)):
        ops.vae_sample_latent(hidden, noise[b:b + 1], lf.shift_factor, lf.scale_factor, out=x0[b:b + 1])
    return ops.axpb(x0, 1.0 / lf.scale_factor, lf.shift_factor)


def _assert_kept(latent, want, latent_mask, what):
    keep = torch.from_numpy(latent_mask == 0).to(DEV)[None, :, :, None].expand_as(latent)
    assert torch.equal(latent[keep], want[keep]), f"{what}: unmasked latents are not process_out(x0)"
    assert not torch.equal(latent[~keep], want[~keep]), f"{what}: the masked region was not regenerated"


@pytest.mark.parametrize("denoise", [1.0, 0.5])
def test_unmasked_latents_and_pixels_are_the_source(kc, denoise):
    from diffusionkit_b200.inpaint import prepare_mask
    from tests.test_solvers_gpu import _weights

    _, p16, vp16 = _weights("flux")
    pipe = _flux_pipe(p16, vp16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=16)
    img, mask = _source(), _mask()
    m = prepare_mask(mask, (WP, HP))
    want = _x0_out(pipe, img, SEEDS)
    kw = dict(num_steps=STEPS, seed=SEEDS, image_path=img, denoise=denoise, mask_image=mask)
    for solver in SOLVERS:
        lat, _ = pipe.denoise_latents(cond, pooled, solver=solver, **kw)
        _assert_kept(lat, want, m.latent, f"{solver} denoise {denoise}")
        images, log = pipe.generate_image("", verbose=False, conditioning=cond, pooled_conditioning=pooled,
                                          solver=solver, **kw)
        keep = m.pixels == 0
        for im in images:
            a = np.asarray(im)
            assert a.shape == img.shape and np.array_equal(a[keep], img[keep]), solver
        assert log["denoising"]["inpaint"] == {"latent_size": (HP // 8, WP // 8),
                                               "masked_fraction": float(m.latent.mean())}
    pipe.set_step_cache(float("inf"))
    lat, _ = pipe.denoise_latents(cond, pooled, solver="euler", **kw)
    assert any(s for _, s in pipe.mmdit.step_cache_log)
    _assert_kept(lat, want, m.latent, "step cache")
    pipe.set_step_cache(None)
    pipe.set_fp8(True)
    lat, _ = pipe.denoise_latents(cond, pooled, solver="dpmpp_2m", **kw)
    _assert_kept(lat, want, m.latent, "fp8")
    pipe.set_fp8(False)
    from tests.lora_fixtures import kohya_dict, make_factors, upstream_modules
    from tests.test_solvers_gpu import _weights as w

    name = pipe.load_lora_weights(kohya_dict(make_factors(upstream_modules(w("flux")[0]), 4, seed=3)), scale=1.0)
    lat, _ = pipe.denoise_latents(cond, pooled, solver="heun", **kw)
    _assert_kept(lat, want, m.latent, "lora")
    pipe.unload_lora_weights(name)
    ref = torch.randn((1, 8, 8, 16), generator=torch.Generator().manual_seed(2)).to(DEV)
    lat, _ = pipe.denoise_latents(cond, pooled, solver="euler_ancestral", reference_latents=ref, **kw)
    _assert_kept(lat, want, m.latent, "kontext reference")


def test_flux_dev_guidance(kc):
    import diffusionkit_b200 as dk
    from diffusionkit_b200.config import tiny_flux_config
    from diffusionkit_b200.inpaint import prepare_mask
    from diffusionkit_b200.weights import init_params, mmdit_param_specs

    cfg = replace(tiny_flux_config(), guidance_embed=True)
    p16 = {k: v.to(bf16) for k, v in init_params(mmdit_param_specs(cfg), seed=7, dtype=torch.float32).items()}
    pipe = dk.FluxPipeline(w16=True, a16=True, model_version="argmaxinc/mlx-FLUX.1-dev", mmdit_config=cfg,
                           params={k: v.to(DEV) for k, v in p16.items()}, load_decoder=False,
                           vae_encoder_params={k: v.to(DEV) for k, v in _encoder_weights(bf16).items()})
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=16)
    img, mask = _source(), _mask()
    lat, _ = pipe.denoise_latents(cond, pooled, num_steps=STEPS, seed=SEEDS, image_path=img, mask_image=mask,
                                  guidance=[2.0, 4.5], solver="dpmpp_2m_sde")
    _assert_kept(lat, _x0_out(pipe, img, SEEDS), prepare_mask(mask, (WP, HP)).latent, "flux.1-dev guidance")


def test_all_ones_is_img2img_and_all_zeros_is_the_source(kc):
    from tests.test_solvers_gpu import _weights

    _, p16, vp16 = _weights("flux")
    pipe = _flux_pipe(p16, vp16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=16)
    img = _source()
    kw = dict(num_steps=STEPS, seed=SEEDS, image_path=img, denoise=0.75, verbose=False, conditioning=cond,
              pooled_conditioning=pooled)
    for solver in ("heun", "dpmpp_2m_sde"):
        plain_lat, _ = pipe.denoise_latents(cond, pooled, num_steps=STEPS, seed=SEEDS, image_path=img, denoise=0.75,
                                            solver=solver)
        plain_lat = plain_lat.clone()
        ones_lat, _ = pipe.denoise_latents(cond, pooled, num_steps=STEPS, seed=SEEDS, image_path=img, denoise=0.75,
                                           solver=solver, mask_image=np.full((HP, WP), 255, np.uint8))
        assert torch.equal(ones_lat, plain_lat), solver
        plain, _ = pipe.generate_image("", solver=solver, **kw)
        ones, log = pipe.generate_image("", solver=solver, mask_image=np.full((HP, WP), 255, np.uint8), **kw)
        assert log["denoising"]["inpaint"]["masked_fraction"] == 1.0
        assert all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(plain, ones)), solver
        zeros, log = pipe.generate_image("", solver=solver, mask_image=np.zeros((HP, WP), np.uint8), **kw)
        assert log["denoising"]["inpaint"]["masked_fraction"] == 0.0
        assert all(np.array_equal(np.asarray(a), img) for a in zeros), solver


def test_reproducible_with_and_without_graphs(kc, monkeypatch):
    from tests.test_solvers_gpu import _weights

    _, p16, _ = _weights("flux")
    runs = {}
    for graphs in ("1", "0"):
        monkeypatch.setenv("DK_CUDA_GRAPHS", graphs)
        pipe = _flux_pipe(p16)
        cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=16)
        for solver in ("euler", "dpmpp_2m_sde"):
            got = []
            for _ in range(2):
                lat, _ = pipe.denoise_latents(cond, pooled, num_steps=STEPS, seed=SEEDS, image_path=_source(),
                                              solver=solver, mask_image=_mask())
                torch.cuda.synchronize()
                got.append(lat.clone())
            assert torch.equal(got[0], got[1]), (graphs, solver)
            runs[graphs, solver] = got[0]
        del pipe
    for solver in ("euler", "dpmpp_2m_sde"):
        assert torch.equal(runs["1", solver], runs["0", solver]), solver


def test_no_mask_launches_nothing_new(kc, monkeypatch):
    """without a mask the inpaint wrappers are never called and a call's launches are the same as before; with one, a
    denoise adds one blend per step and generate_image one paste"""
    from diffusionkit_b200 import inpaint, ops
    from tests.test_solvers_gpu import _weights

    calls = {"inpaint_blend": 0, "inpaint_paste": 0}
    for name in calls:
        fn = getattr(inpaint, name)

        def counted(*a, _fn=fn, _name=name, **k):
            calls[_name] += 1
            return _fn(*a, **k)

        monkeypatch.setattr(inpaint, name, counted)
    _, p16, vp16 = _weights("flux")
    pipe = _flux_pipe(p16, vp16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=1, text_len=16)
    img = _source()
    kw = dict(num_steps=STEPS, seed=3, image_path=img, denoise=0.75, verbose=False, conditioning=cond,
              pooled_conditioning=pooled, solver="heun")

    def launches(**extra):
        n0 = ops.launch_count()
        pipe.generate_image("", **kw, **extra)
        return ops.launch_count() - n0

    launches()                                                       # captures the graphs of these shapes
    plain = launches()
    assert calls == {"inpaint_blend": 0, "inpaint_paste": 0}
    assert launches(mask_image=None) == plain
    masked = launches(mask_image=_mask())
    steps = STEPS - int(STEPS * (1 - 0.75))
    assert calls == {"inpaint_blend": steps, "inpaint_paste": 1}
    assert masked == plain + steps + 1


def test_pipeline_argument_errors_launch_nothing(kc, tmp_path):
    from diffusionkit_b200 import ops
    from tests.test_solvers_gpu import _weights

    _, p16, vp16 = _weights("flux")
    pipe = _flux_pipe(p16, vp16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=1, text_len=16)
    img = _source()
    bad = tmp_path / "mask.png"
    bad.write_bytes(b"\x89PNG broken")
    cases = [(dict(mask_image=_mask()), "needs image_path"),
             (dict(image_path=img, mask_image=_mask(HP, WP - 64)), "same size"),
             (dict(image_path=img, mask_image=_mask().astype(np.int32)), "uint8"),
             (dict(image_path=img, mask_image=np.zeros((HP, WP, 2), np.uint8)), "uint8"),
             (dict(image_path=img, mask_image=str(tmp_path / "none.png")), "cannot be read"),
             (dict(image_path=img, mask_image=str(bad)), "cannot be read")]
    n0 = ops.launch_count()
    for extra, msg in cases:
        with pytest.raises(ValueError, match=msg):
            pipe.denoise_latents(cond, pooled, num_steps=STEPS, seed=3, **extra)
        with pytest.raises(ValueError, match=msg):
            pipe.generate_image("", num_steps=STEPS, seed=3, verbose=False, conditioning=cond,
                                pooled_conditioning=pooled, **extra)
    assert ops.launch_count() == n0
