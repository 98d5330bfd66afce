"""GPU checks of FLUX.1 Fill [dev] (DESIGN.md §18): dk_image_pre_masked and dk_fill_cond_rows bit for bit against
their references (tests/fill_ref.py) and their argument errors; a tiny Fill pipeline against the oracle with the
concatenated x-embedder under a launch census of its own; that the conditioning matters; a full-width forward under the
census; the per-step launches equal to FLUX.1-dev's; and the invariants (paste-back, reruns, CUDA graphs, LoRA, Redux,
the step cache, FP8), with §17's path unchanged on other models."""
from dataclasses import replace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
bf16, fp16 = torch.bfloat16, torch.float16
SEEDS = [11, 12]
STEPS = 4
T = 16
HP, WP = 64, 128                       # the source image; latent 8 x 16, 4 x 8 tokens


@pytest.fixture(scope="module")
def kc():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    from tests import kernel_checks

    kernel_checks._setup()
    return kernel_checks


def _cfg():
    from tests.test_fill_cpu import tiny_fill_config

    return tiny_fill_config()


def _mask(H=HP, W=WP, value=255):
    """a rectangle plus a 3-pixel vertical line, white on black"""
    m = np.zeros((H, W), dtype=np.uint8)
    m[H // 4:H // 2 + 5, W // 5:W // 2] = value
    m[:, W - 27:W - 24] = value
    return m


def _source():
    from tests.model_checks import _test_image

    return _test_image(HP, WP)


def _weights(cfg, seed=7):
    from diffusionkit_b200.weights import init_params, mmdit_param_specs
    from tests.kontext_ref import sharpen

    return {k: v.to(bf16) for k, v in sharpen(init_params(mmdit_param_specs(cfg), seed=seed,
                                                          dtype=torch.float32)).items()}


def _vae(encoder):
    from tests.test_kontext_gpu import _vae_weights

    return _vae_weights(encoder=encoder)


def _pipe(cfg, p16, vp16=None, **kw):
    from tests.test_kontext_gpu import _pipe as kpipe

    return kpipe(cfg, p16, vp16, _vae(True), **kw)


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("dtype", [bf16, fp16])
@pytest.mark.parametrize("H, W", [(64, 128), (1024, 1024)])
def test_kernels_bit_for_bit(kc, dtype, H, W):
    from diffusionkit_b200.fill import fill_cond_rows, image_pre_masked
    from tests.fill_ref import ref_cond_rows, ref_image_pre_masked

    g = torch.Generator(device=DEV).manual_seed(H + W)
    img = torch.randint(0, 256, (1, H, W, 4), generator=g, device=DEV, dtype=torch.uint8)
    lat = torch.randn(((H // 16) * (W // 16), 64), generator=g, device=DEV).to(dtype)
    for p in (0.0, 1.0 / 3.0, 1.0):
        mask = (torch.rand((H, W), generator=g, device=DEV) < p).to(torch.uint8) * 255
        got = image_pre_masked(img, mask, dtype)
        assert torch.equal(got, ref_image_pre_masked(img, mask, dtype)), (H, W, p)
        if p == 0.0:
            from diffusionkit_b200 import ops

            assert torch.equal(got, ops.image_pre(img, dtype)), "no mask: dk_image_pre's bits"
        rows = fill_cond_rows(lat, mask)
        assert torch.equal(rows, ref_cond_rows(lat, mask)), (H, W, p)


def test_kernel_argument_errors_launch_nothing(kc):
    from diffusionkit_b200 import DkError, ops
    from diffusionkit_b200._lib import ptr

    c = ops.ctx(0)
    img = torch.zeros((1, 32, 32, 3), dtype=torch.uint8, device=DEV)
    mask = torch.zeros((32, 32), dtype=torch.uint8, device=DEV)
    out = torch.empty(32 * 32 * 64 + 8, dtype=bf16, device=DEV)
    lat = torch.empty(4 * 64 + 8, dtype=bf16, device=DEV)
    rows = torch.empty(4 * 320 + 8, dtype=bf16, device=DEV)
    n0 = c.launches
    for args, msg in [(("dk_image_pre_masked", 0, ptr(img), ptr(mask), ptr(out[1:]), 32, 32, 3, 64), "aligned"),
                      (("dk_image_pre_masked", 0, ptr(img), None, ptr(out), 32, 32, 3, 64), "required"),
                      (("dk_image_pre_masked", 0, ptr(img), ptr(mask), ptr(out), 32, 24, 3, 64), "multiples of 16"),
                      (("dk_image_pre_masked", 5, ptr(img), ptr(mask), ptr(out), 32, 32, 3, 64), "bad dtype"),
                      (("dk_fill_cond_rows", 0, ptr(lat[1:]), ptr(mask), ptr(rows), 32, 32), "aligned"),
                      (("dk_fill_cond_rows", 0, ptr(lat), ptr(mask), ptr(rows[1:]), 32, 32), "aligned"),
                      (("dk_fill_cond_rows", 0, ptr(lat), ptr(mask), None, 32, 32), "required"),
                      (("dk_fill_cond_rows", 0, ptr(lat), ptr(mask), ptr(rows), 40, 32), "multiples of 16"),
                      (("dk_fill_cond_rows", 9, ptr(lat), ptr(mask), ptr(rows), 32, 32), "bad dtype")]:
        with pytest.raises(DkError, match=msg):
            c.call(*args)
    assert c.launches == n0


# ------------------------------------------------------------------------------------------------ pipelines
def _census_wrap(monkeypatch, c):
    """tests/launch_parity's census plus the two Fill launches and the stochastic step (tests/sde_ref)"""
    from diffusionkit_b200 import fill, pipeline
    from tests import launch_parity as lp
    from tests import sde_ref
    from tests.fill_ref import census_check_cond_rows, census_check_image_pre_masked

    for name, check, writes in (("image_pre_masked", census_check_image_pre_masked, []),
                                ("fill_cond_rows", census_check_cond_rows, ["out"]),
                                ("sampler_sde_step", sde_ref.census_check, ["x", "d_prev"])):
        monkeypatch.setitem(lp.CHECKS, name, check)
        monkeypatch.setitem(lp.WRITES, name, writes)
    monkeypatch.setattr(fill, "image_pre_masked", c._wrap("image_pre_masked", fill.image_pre_masked))
    monkeypatch.setattr(fill, "fill_cond_rows", c._wrap("fill_cond_rows", fill.fill_cond_rows))
    monkeypatch.setattr(pipeline, "sampler_sde_step", c._wrap("sampler_sde_step", pipeline.sampler_sde_step))


def _oracle(cfg, p16, img, mask_u8, cond, pooled, sig, guidance, solver):
    """the oracle Fill pipeline: img2img starts and conditioning rows from the fp32 oracle encoder"""
    from oracle import sampler_ref as sr
    from oracle.vae_ref import VAEEncoderRef, encode_image_to_latents, read_image_array
    from tests.fill_ref import FillMMDiTRef, fill_pipeline_latents, oracle_cond_rows
    from tests.oracle_bridge import ref_config

    enc = VAEEncoderRef({k: v.float() for k, v in _vae(True).items()})
    m01 = (mask_u8 >= 128).astype(np.uint8)
    rows = oracle_cond_rows(enc, img, m01, 0.1159, 0.3611, bf16)
    image = read_image_array(torch.from_numpy(img))
    x0s = []
    for s in SEEDS:
        eps = sr.get_noise(s, HP // 8, WP // 8)
        x0 = (encode_image_to_latents(enc, image, eps) - 0.1159) * 0.3611
        x0s.append(float(sig[0]) * eps + (1.0 - float(sig[0])) * x0)
    params = {k: v.float() for k, v in p16.items()}
    return fill_pipeline_latents(lambda: FillMMDiTRef(ref_config(cfg), params), solver, sig, x0s, rows, cond, pooled,
                                 guidance, 0.0, bf16, SEEDS)


def _compare(pipe, vp16, latent, want, what):
    from oracle.vae_ref import VAEDecoderRef, decode_latents_to_image
    from tests.model_checks import psnr, rel_l2

    r = rel_l2(latent, want)
    img_want = decode_latents_to_image(VAEDecoderRef({k: v.float() for k, v in vp16.items()}), want.to(bf16).float())
    ps = psnr(img_want, pipe.decode_latents_to_image(latent))
    print(f"{what}: final latent rel_l2 {r:.3e}, decoded psnr {ps:.1f} dB")
    assert r <= 5e-2 and ps >= 30.0, f"{what}: rel_l2 {r:.3e}, psnr {ps:.1f}"
    return r


@pytest.mark.parametrize("denoise", [1.0, 0.6])
def test_tiny_pipeline_against_the_oracle_under_a_census(kc, monkeypatch, denoise):
    from oracle import sampler_ref as sr
    from tests import launch_parity as lp
    from tests.model_checks import rel_l2

    cfg = _cfg()
    p16, vp16 = _weights(cfg), _vae(False)
    pipe = _pipe(cfg, p16, vp16)
    pipe.mmdit.use_cuda_graphs = pipe.decoder.use_cuda_graphs = False
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
    img, mask = _source(), _mask()
    sig = sr.get_sigmas(sr.FluxSamplerRef(1.0), STEPS)[int(STEPS * (1 - denoise)):]
    guidance = [30.0, 12.0]
    c = lp.Census()
    with lp.census(c):
        _census_wrap(monkeypatch, c)
        for solver in ("euler", "dpmpp_2m", "dpmpp_2m_sde"):
            c.run = f"fill-{solver}-{denoise}"
            n0 = len(c.records)
            lat, it = pipe.denoise_latents(cond, pooled, num_steps=STEPS, seed=SEEDS, image_path=img, denoise=denoise,
                                           solver=solver, mask_image=mask, guidance=guidance)
            torch.cuda.synchronize()
            ops_run = [r["op"] for r in c.records[n0:]]
            assert ops_run.count("image_pre_masked") == 1 and ops_run.count("fill_cond_rows") == 1
            assert len(it) == len(sig) - 1
            want = _oracle(cfg, p16, img, mask, cond, pooled, sig, guidance, solver)
            _compare(pipe, vp16, lat, want, f"fill {solver} denoise {denoise}")
            if solver == "euler":
                other = _mask()[::-1, ::-1].copy()
                moved = rel_l2(_oracle(cfg, p16, img, other, cond, pooled, sig, guidance, solver), want)
                print(f"another mask moves the oracle by rel_l2 {moved:.3e}")
                assert moved > 5e-2, "the conditioning must matter beyond the pipeline bound"
    print(c.table())


def test_fullwidth_forward_under_a_census(kc):
    """FLUX.1-dev's width (h = 3072), 1 double + 1 single block, a 64 x 64 latent, T = 512, B = 2 with per-image
    guidance, eager under the launch census: the K = 320 conditioning GEMM with bias once, the K = 64 x-embedder GEMM
    with the batch-broadcast residual and no bias every forward"""
    from diffusionkit_b200 import MMDiT, ops
    from diffusionkit_b200.config import FLUX_FILL_DEV
    from tests import launch_parity as lp
    from tests.fill_ref import FillMMDiTRef
    from tests.oracle_bridge import ref_config
    from tests.test_kontext_gpu import _check

    cfg = replace(FLUX_FILL_DEV, depth_multimodal=1, depth_unified=1)
    B, lat, guidance = 2, (64, 64), [30.0, 10.0]
    N = (lat[0] // 2) * (lat[1] // 2)
    p16 = _weights(cfg)
    g = torch.Generator().manual_seed(5)
    latent = torch.randn((B, *lat, 16), generator=g).to(bf16)
    text = torch.randn((B, 512, cfg.token_level_text_embed_dim), generator=g).to(bf16)
    pooled = torch.randn((B, cfg.pooled_text_embed_dim), generator=g).to(bf16)
    rows = torch.cat([torch.randn((N, 64), generator=g), (torch.rand((N, 256), generator=g) < 0.4).float()],
                     dim=1).to(bf16)
    m = MMDiT(cfg, {k: v.to(DEV) for k, v in p16.items()})
    m.use_cuda_graphs = False
    m.cache_modulation_params(pooled.to(DEV), [752.0], guidance)
    c = lp.Census()
    c.run = "fill-fullwidth"
    with lp.census(c):
        m.cache_fill_conditioning(rows.to(DEV))
        got = m(latent.to(DEV), text.to(DEV), timestep=752.0)
        torch.cuda.synchronize()
        got = got.clone()
    print(c.table())
    sigs = [r["info"] for r in c.records if r["op"] == "gemm" and r["info"]["K"] in (64, 320)]
    assert [(s["K"], s["M"], s["epi"]) for s in sigs] == [(320, N, "bias"), (64, B * N, "res")], sigs
    assert sigs[1]["res_batch_rows"] == 0
    del m
    torch.cuda.empty_cache()
    ref = FillMMDiTRef(ref_config(cfg), {k: v.float() for k, v in p16.items()})
    ref.cond = rows.float()
    t = torch.tensor([752.0])
    ref.cache_modulation_params(pooled.float(), t, guidance)
    _check(got, ref(latent.float(), text.float(), t.repeat(B)), "fill full width, 64x64, T = 512, B = 2")


def test_per_step_launches_equal_flux_dev(kc):
    """a Fill forward launches exactly what a FLUX.1-dev forward of the same shape launches"""
    from diffusionkit_b200 import MMDiT, ops

    cfg = _cfg()
    dev = replace(cfg, x_embedder_cond_channels=0)
    g = torch.Generator().manual_seed(3)
    latent = torch.randn((2, 8, 16, 16), generator=g).to(bf16).to(DEV)
    text = torch.randn((2, T, cfg.token_level_text_embed_dim), generator=g).to(bf16).to(DEV)
    pooled = torch.randn((2, cfg.pooled_text_embed_dim), generator=g).to(bf16).to(DEV)
    counts = []
    for c in (cfg, dev):
        m = MMDiT(c, {k: v.to(DEV) for k, v in _weights(c).items()})
        m.use_cuda_graphs = False
        m.cache_modulation_params(pooled, [500.0], [3.5, 3.5])
        if c.x_embedder_cond_channels:
            m.cache_fill_conditioning(torch.zeros((32, 320), dtype=bf16, device=DEV))
        m(latent, text, timestep=500.0)
        n0 = ops.launch_count()
        m(latent, text, timestep=500.0)
        counts.append(ops.launch_count() - n0)
    assert counts[0] == counts[1], counts


# ------------------------------------------------------------------------------------------------ invariants
def test_invariants(kc):
    cfg = _cfg()
    p16, vp16 = _weights(cfg), _vae(False)
    pipe = _pipe(cfg, p16, vp16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
    img, mask = _source(), _mask()
    kw = dict(num_steps=STEPS, seed=SEEDS, image_path=img, mask_image=mask)

    def run(**extra):
        lat, _ = pipe.denoise_latents(cond, pooled, **kw, **extra)
        torch.cuda.synchronize()
        return lat.clone()

    base = run()
    assert torch.equal(run(), base), "a rerun repeats"
    pipe.mmdit.use_cuda_graphs = False
    assert torch.equal(run(), base), "CUDA graphs equal eager"
    pipe.mmdit.use_cuda_graphs = True
    assert torch.equal(run(guidance=30.0), base), "guidance None is 30 on Fill"
    # paste-back and the log
    images, log = pipe.generate_image("", verbose=False, conditioning=cond, pooled_conditioning=pooled, **kw)
    keep = mask < 128
    for im in images:
        assert np.array_equal(np.asarray(im)[keep], img[keep])
    f = log["denoising"]["fill"]
    assert f["latent_size"] == (HP // 8, WP // 8) and "inpaint" not in log["denoising"] and f["time"] >= 0
    # LoRA on the x-embedder and the blocks: load, rescale and unload restore every bit
    from tests.lora_fixtures import kohya_dict, make_factors, upstream_modules

    name = pipe.load_lora_weights(kohya_dict(make_factors(upstream_modules(cfg), 4, seed=3)), scale=1.0)
    with_lora = run()
    assert not torch.equal(with_lora, base)
    pipe.set_lora_scale(name, 0.0)
    assert torch.equal(run(), base), "scale 0"
    pipe.set_lora_scale(name, 1.0)
    assert torch.equal(run(), with_lora), "scale back"
    pipe.unload_lora_weights(name)
    assert torch.equal(run(), base), "unloaded"
    # step cache: threshold 0 never skips and changes no bit; infinity skips and keeps the pasted pixels
    pipe.set_step_cache(0.0)
    assert torch.equal(run(), base)
    pipe.set_step_cache(float("inf"))
    run()
    assert any(s for _, s in pipe.mmdit.step_cache_log)
    pipe.set_step_cache(None)
    # FP8 decodes close to 16-bit
    from tests.model_checks import psnr

    want = pipe.decode_latents_to_image(base)
    pipe.set_fp8(True)
    got = pipe.decode_latents_to_image(run())
    pipe.set_fp8(False)
    ps = psnr(want.cpu(), got.cpu())
    print(f"fp8 vs 16-bit decoded psnr {ps:.1f} dB")
    assert ps >= 25.0
    # a batch with CFG shares the one conditioning buffer: per-seed results do not depend on the batch
    lat1, _ = pipe.denoise_latents(cond[[1]], pooled[[1]], num_steps=STEPS, seed=SEEDS[1], image_path=img,
                                   mask_image=mask)
    assert torch.equal(lat1[0], base[1])


def test_redux_tokens_equal_conditioning(kc):
    from diffusionkit_b200.config import tiny_siglip_config

    cfg = _cfg()
    pipe = _pipe(cfg, _weights(cfg))
    pipe.load_redux(siglip_config=tiny_siglip_config())
    cond, pooled = pipe.synthetic_text_embeddings(n_images=1, text_len=T)
    img, mask = _source(), _mask()
    prompt = np.roll(img, 17, axis=1)
    kw = dict(num_steps=STEPS, seed=5, image_path=img, mask_image=mask)
    a, _ = pipe.denoise_latents(cond, pooled, redux_image=prompt, **kw)
    a = a.clone()
    tokens = pipe.encode_redux(prompt)
    b, _ = pipe.denoise_latents(torch.cat([cond.to(DEV), tokens], dim=1), pooled, **kw)
    assert torch.equal(a, b)


def test_errors_and_other_models(kc, monkeypatch):
    """argument errors launch nothing; a non-Fill model given mask_image runs §17 and never the Fill path"""
    from diffusionkit_b200 import fill, ops
    from tests.test_inpaint_gpu import _flux_pipe
    from tests.test_solvers_gpu import _weights as sw

    cfg = _cfg()
    pipe = _pipe(cfg, _weights(cfg))
    cond, pooled = pipe.synthetic_text_embeddings(n_images=1, text_len=T)
    img, mask = _source(), _mask()
    n0 = ops.launch_count()
    for kw, msg in [(dict(image_path=img), "needs image_path and mask_image"),
                    (dict(mask_image=mask), "needs image_path and mask_image"),
                    (dict(image_path=img, mask_image=mask, reference_latents=torch.zeros(1, 8, 8, 16, device=DEV)),
                     "Kontext")]:
        with pytest.raises(ValueError, match=msg):
            pipe.denoise_latents(cond, pooled, num_steps=STEPS, seed=3, **kw)
        with pytest.raises(ValueError, match=msg):
            pipe.generate_image("", num_steps=STEPS, seed=3, verbose=False, conditioning=cond,
                                pooled_conditioning=pooled, **kw)
    assert ops.launch_count() == n0
    calls = []
    for name in ("image_pre_masked", "fill_cond_rows", "conditioning_rows"):
        fn = getattr(fill, name)
        monkeypatch.setattr(fill, name, lambda *a, _fn=fn, _n=name, **k: calls.append(_n) or _fn(*a, **k))
    _, p16, vp16 = sw("flux")
    other = _flux_pipe(p16, vp16)
    c2, pl2 = other.synthetic_text_embeddings(n_images=1, text_len=T)
    _, log = other.generate_image("", num_steps=STEPS, seed=3, verbose=False, conditioning=c2, pooled_conditioning=pl2,
                                  image_path=img, mask_image=mask)
    assert calls == [] and "inpaint" in log["denoising"] and "fill" not in log["denoising"]
