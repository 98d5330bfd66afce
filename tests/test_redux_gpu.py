"""GPU checks of FLUX.1 Redux image prompts (DESIGN.md §15): dk_image_patches bit for bit, the tanh-GELU epilogue and
dk_act, the SigLIP forward and the Redux tokens against tests/redux_ref.py (a launch census of the real-width run), the
tiny pipelines against the oracle pipeline, the bit-identities the concatenation promises, and the argument errors.

The MMDiT weights go through kontext_ref.sharpen: with the synthetic initialiser's flat attention two different image
prompts move the tiny pipeline's final latents only 6.8 % apart (the bound is 5 %); sharpened, about 14 %."""
from dataclasses import replace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
bf16, fp16 = torch.bfloat16, torch.float16
LAT = (8, 12)
SEEDS = [11, 12]
STEPS = 4
T = 16


@pytest.fixture(scope="module")
def kc():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    from tests import kernel_checks

    kernel_checks._setup()
    return kernel_checks


def _check(got, want, what):
    from tests.model_checks import psnr, rel_l2

    got = got.float().cpu()
    assert got.shape == want.shape and bool(torch.isfinite(got).all())
    r, ps = rel_l2(got, want), psnr(want, got)
    print(f"{what}: rel_l2 {r:.3e}, psnr {ps:.1f} dB")
    assert r <= 2e-2 and ps >= 35.0, f"{what}: rel_l2={r:.3e} psnr={ps:.1f}"


def _images(n, size, seed=1):
    from tests.model_checks import _test_image

    return [_test_image(size, size, seed=seed + i) for i in range(n)]


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("dtype", [bf16, fp16])
def test_image_patches_bit_exact(kc, dtype):
    from diffusionkit_b200.image_encoders import image_patches
    from tests.redux_ref import ref_image_patches

    g = torch.Generator().manual_seed(0)
    for B, H, W, C, p, kp in [(1, 384, 384, 3, 14, 592), (2, 98, 98, 3, 14, 592), (3, 100, 113, 4, 14, 592),
                              (4, 30, 45, 3, 7, 152), (2, 16, 16, 3, 2, 16)]:
        img = torch.randint(0, 256, (B, H, W, C), generator=g, dtype=torch.uint8).to(DEV)
        got = image_patches(img, dtype, p, kp)
        assert got.shape == (B * (H // p) * (W // p), kp)
        assert torch.equal(got, ref_image_patches(img, dtype, p, kp)), (B, H, W, C, p, kp, dtype)


def test_tanh_gelu_epilogue_and_act(kc):
    import torch.nn.functional as F

    from diffusionkit_b200 import ops
    from diffusionkit_b200._lib import ACT_GELU_TANH
    from tests.redux_ref import with_gelu_tanh

    ref_gemm = with_gelu_tanh(kc.ref_gemm)
    for M, N, K, dt in [(1458, 4304, 1152, bf16), (729, 4304, 1152, fp16), (200, 304, 144, bf16)]:
        A = kc._rand((M, K), dt)
        W = kc._rand((N, K), dt, K ** -0.5)
        b = kc._rand((N,), dt, 0.5)
        got = ops.gemm(A, W, bias=b, act=ACT_GELU_TANH)
        kc._assert_close(f"gemm gelu_tanh {M}x{N}x{K}", got, ref_gemm(A, W, b, ACT_GELU_TANH), 4e-3)
    for dt in (bf16, fp16):
        x = kc._rand((4096, 72), dt, 3.0)
        kc._assert_close(f"act gelu_tanh {dt}", ops.act(x, ACT_GELU_TANH), F.gelu(x.float(), approximate="tanh"),
                         4e-3)


# ------------------------------------------------------------------------------------------------ encoder
def _encoder_weights(scfg, txt_dim, seed=3):
    """bf16-rounded SigLIP (engine layout) and Redux weights, generated in fp32 on the host"""
    from diffusionkit_b200.image_encoders import init_siglip_params, redux_param_specs
    from diffusionkit_b200.weights import init_params

    sp = {k: v.to(bf16) for k, v in init_siglip_params(scfg, seed=seed, dtype=torch.float32).items()}
    rp = {k: v.to(bf16) for k, v in init_params(redux_param_specs(scfg.hidden_size, txt_dim), seed=seed + 1,
                                                 dtype=torch.float32).items()}
    return sp, rp


def _encode(scfg, sp, rp, imgs):
    from diffusionkit_b200.image_encoders import ReduxImageEncoder, SiglipVisionModel

    sig = SiglipVisionModel({k: v.to(DEV) for k, v in sp.items()}, scfg)
    red = ReduxImageEncoder({k: v.to(DEV) for k, v in rp.items()})
    img = torch.from_numpy(np.stack(imgs)).to(DEV)
    h = sig(img)
    tok = red(h.reshape(-1, h.shape[2]), h.shape[1])
    torch.cuda.synchronize()
    return h.clone(), tok.reshape(h.shape[0], h.shape[1], -1).clone()


def test_tiny_siglip_and_redux_against_the_oracle(kc):
    from diffusionkit_b200.config import tiny_siglip_config
    from tests.redux_ref import SiglipVisionRef, redux_project

    for scfg in (tiny_siglip_config(layers=4), tiny_siglip_config(image_size=100, layers=4)):
        sp, rp = _encoder_weights(scfg, 128)
        imgs = _images(3, scfg.image_size)
        h, tok = _encode(scfg, sp, rp, imgs)
        want = SiglipVisionRef(sp, scfg)(torch.from_numpy(np.stack(imgs)))
        _check(h, want, f"tiny SigLIP {scfg.image_size}^2, 4 layers")
        _check(tok, redux_project(rp, want), f"tiny Redux tokens {scfg.image_size}^2")


def _c_image_patches(L, a, s, r, census):
    from tests.redux_ref import ref_image_patches

    L.exact("rows", r, ref_image_patches(s["img_u8"], a["dtype"], a["p"], a["kp"]))
    L.own(r)
    L.sig.update(shape=tuple(s["img_u8"].shape), p=a["p"], kp=a["kp"], dtype=str(a["dtype"])[6:])


def _c_attention_scaled(L, a, s, r, census):
    """tests/launch_parity's attention check with the launch's own softmax scale (SigLIP passes 72^-0.5 at d = 128)"""
    from tests import launch_parity as lp
    from tests.redux_ref import ref_attention

    B, S, heads, hd = a["B"], a["S"], a["heads"], a["d"]
    assert a["split"] is None and a["out1"] is None
    h = heads * hd
    scale = a["scale"] if a["scale"] is not None else hd ** -0.5
    o0 = a["out0"]
    L.close("out0", o0[:B * S, :h], ref_attention(s["qkv"], B, S, heads, hd, scale), lp.TOL_ATT, lp.BLK_ATT, bc=hd)
    L.own(o0, (slice(0, B * S), slice(0, h)))
    L.sig.update(B=B, S=S, heads=heads, d=hd, scale=round(scale, 6), ld0=o0.stride(0), dtype=str(o0.dtype)[6:])


@pytest.fixture
def redux_census(kc, monkeypatch):
    """tests/launch_parity's census over the encoder: every ops launch, plus image_encoders.image_patches, with the
    references it lacks supplied here (tanh-GELU in the GEMM reference, attention at a given scale, the patch rows)"""
    from diffusionkit_b200 import image_encoders
    from tests import launch_parity as lp
    from tests.redux_ref import with_gelu_tanh

    monkeypatch.setattr(kc, "ref_gemm", with_gelu_tanh(kc.ref_gemm))
    monkeypatch.setitem(lp.CHECKS, "attention", _c_attention_scaled)
    monkeypatch.setitem(lp.CHECKS, "image_patches", _c_image_patches)
    monkeypatch.setitem(lp.WRITES, "image_patches", ["out"])
    c = lp.Census()
    with lp.census(c):
        monkeypatch.setattr(image_encoders, "image_patches", c._wrap("image_patches", image_encoders.image_patches))
        yield c


def test_real_width_against_the_oracle_under_a_census(redux_census):
    """SigLIP so400m's width (1152 / 16 heads / 4304) at 384^2, 3 layers, B = 2, and the 1152 -> 12288 -> 4096 Redux
    projector, eagerly under the launch census"""
    from diffusionkit_b200.config import SIGLIP_SO400M_PATCH14_384
    from tests.redux_ref import SiglipVisionRef, redux_project

    scfg = replace(SIGLIP_SO400M_PATCH14_384, num_hidden_layers=3)
    sp, rp = _encoder_weights(scfg, 4096)
    imgs = _images(2, 384)
    c = redux_census
    c.run = "redux-realwidth"
    h, tok = _encode(scfg, sp, rp, imgs)
    print(c.table())
    seen = {r["op"] for r in c.records}
    assert {"image_patches", "gemm", "layernorm", "attention"} <= seen, seen
    atts = [r["info"] for r in c.records if r["op"] == "attention"]
    assert len(atts) == 3 and all((a["S"], a["heads"], a["d"]) == (729, 16, 128) for a in atts), atts
    want = SiglipVisionRef(sp, scfg)(torch.from_numpy(np.stack(imgs)))
    _check(h, want, "SigLIP so400m width, 3 layers, B = 2")
    _check(tok, redux_project(rp, want), "Redux tokens, 4096 wide")


# ------------------------------------------------------------------------------------------------ pipelines
def _mmdit_weights(cfg, seed=7):
    from diffusionkit_b200.weights import init_params, mmdit_param_specs
    from tests.kontext_ref import sharpen

    p = sharpen(init_params(mmdit_param_specs(cfg), seed=seed, dtype=torch.float32))
    return {k: v.to(bf16) for k, v in p.items()}


def _vae_weights():
    from diffusionkit_b200.config import VAEDecoderConfig
    from diffusionkit_b200.weights import init_params, vae_decoder_param_specs

    return {k: v.to(bf16) for k, v in init_params(vae_decoder_param_specs(VAEDecoderConfig()), seed=8,
                                                   dtype=torch.float32).items()}


def _pipe(cfg, p16, vp16=None, redux=True, **kw):
    import diffusionkit_b200 as dk
    from diffusionkit_b200.config import tiny_siglip_config

    def dev(p):
        return None if p is None else {k: v.to(DEV) for k, v in p.items()}

    pipe = dk.FluxPipeline(w16=True, a16=True, shift=1.0, mmdit_config=cfg, params=dev(p16), vae_params=dev(vp16),
                           load_decoder=vp16 is not None, **kw)
    if redux:
        scfg = tiny_siglip_config()
        sp, rp = _encoder_weights(scfg, cfg.token_level_text_embed_dim)
        pipe.load_redux(sp, rp, siglip_config=scfg)
        pipe._test_encoder = (scfg, sp, rp)
    return pipe


def _oracle_pipeline(pipe, cfg, p16, cond, pooled, imgs, guidance, solver="euler"):
    """the oracle pipeline on cat(T5 rows, oracle Redux tokens of the host-resized image) per seed"""
    from oracle import sampler_ref as sr
    from tests import solver_ref
    from tests.kontext_ref import KontextMMDiTRef
    from tests.oracle_bridge import ref_config
    from tests.redux_ref import redux_pipeline_latents, redux_tokens

    scfg, sp, rp = pipe._test_encoder
    arrs = torch.from_numpy(np.stack([pipe._redux_image_u8(im) for im in imgs]))
    tokens = redux_tokens(sp, rp, scfg, arrs)
    sample = {"euler": sr.sample_euler, "dpmpp_2m": solver_ref.sample_dpmpp_2m}[solver]
    sampler = sr.FluxSamplerRef(1.0)
    sig = sr.get_sigmas(sampler, STEPS)
    H, W = LAT
    x0s = [sampler.noise_scaling(float(sig[0]), sr.get_noise(s, H, W), sr.get_empty_latent(H, W)) for s in SEEDS]
    params = {k: v.float() for k, v in p16.items()}
    return redux_pipeline_latents(lambda: KontextMMDiTRef(ref_config(cfg), params), sample, sig, x0s, cond, pooled,
                                  [tokens[i if len(imgs) > 1 else 0] for i in range(len(SEEDS))], guidance, bf16)


def _compare(pipe, vp16, latent, want, what):
    from oracle.vae_ref import VAEDecoderRef, decode_latents_to_image
    from tests.model_checks import psnr, rel_l2

    r = rel_l2(latent, want)
    img_want = decode_latents_to_image(VAEDecoderRef({k: v.float() for k, v in vp16.items()}), want.to(bf16).float())
    ps = psnr(img_want, pipe.decode_latents_to_image(latent))
    print(f"{what}: final latent rel_l2 {r:.3e}, decoded psnr {ps:.1f} dB")
    assert r <= 5e-2, f"{what}: final latent rel_l2 {r:.3e}"
    assert ps >= 30.0, f"{what}: decoded RGB psnr {ps:.1f}"


def _configs():
    from diffusionkit_b200.config import tiny_flux_config
    from tests.test_guidance_cpu import tiny_dev_config

    return {"schnell": tiny_flux_config(), "dev": tiny_dev_config()}


@pytest.mark.parametrize("model, solver, per_seed", [("dev", "euler", False), ("dev", "dpmpp_2m", True),
                                                     ("schnell", "euler", True), ("schnell", "dpmpp_2m", False)])
def test_tiny_pipeline_against_the_oracle(kc, model, solver, per_seed):
    from tests.model_checks import rel_l2

    cfg = _configs()[model]
    p16, vp16 = _mmdit_weights(cfg), _vae_weights()
    pipe = _pipe(cfg, p16, vp16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=1, text_len=T)
    imgs = _images(2, 150, seed=4) if per_seed else _images(1, 120, seed=4)
    guidance = 3.0 if cfg.guidance_embed else None
    lat, it = pipe.denoise_latents(cond, pooled, num_steps=STEPS, latent_size=LAT, seed=SEEDS, solver=solver,
                                   guidance=guidance, redux_image=imgs if per_seed else imgs[0])
    torch.cuda.synchronize()
    assert lat.shape == (len(SEEDS), *LAT, 16) and len(it) == STEPS
    cond2, pooled2 = cond.repeat(2, 1, 1), pooled.repeat(2, 1)
    want = _oracle_pipeline(pipe, cfg, p16, cond2, pooled2, imgs, [guidance] * 2, solver)
    _compare(pipe, vp16, lat, want, f"{model} {solver} {'one image per seed' if per_seed else 'one shared image'}")
    # the check sees the image: another prompt image moves the oracle's latents well past the 5e-2 bound
    other = _oracle_pipeline(pipe, cfg, p16, cond2, pooled2, _images(len(imgs), 150, seed=40), [guidance] * 2, solver)
    sep = rel_l2(other, want)
    print(f"another image prompt: oracle latents {sep:.3e} apart")
    assert sep >= 0.1, sep


def test_redux_image_is_the_concatenated_conditioning(kc):
    """redux_image= gives bit for bit what conditioning=cat(cond, encode_redux(img)) gives, shared and per seed, with
    and without a Kontext reference, with CUDA graphs and eagerly; reruns are bit-identical; generate_image logs it"""
    from tests.test_guidance_cpu import tiny_dev_config

    cfg = tiny_dev_config()
    pipe = _pipe(cfg, _mmdit_weights(cfg))
    cond, pooled = pipe.synthetic_text_embeddings(n_images=1, text_len=T)
    imgs = _images(2, 130, seed=6)
    g = torch.Generator().manual_seed(21)
    refs = torch.randn((1, 8, 8, 16), generator=g).to(DEV)
    kw = dict(num_steps=STEPS, latent_size=LAT, seed=SEEDS, guidance=3.0)
    results = {}
    for graphs in (True, False):
        pipe.mmdit.use_cuda_graphs = graphs
        for ref in (None, refs):
            for per_seed in (False, True):
                prompt = imgs if per_seed else imgs[0]
                a, _ = pipe.denoise_latents(cond, pooled, redux_image=prompt, reference_latents=ref, **kw)
                a = a.clone()
                tok = pipe.encode_redux(prompt)
                assert tok.shape == (len(imgs) if per_seed else 1, 49, 128) and tok.dtype == bf16
                cat = torch.cat([cond.to(DEV).repeat(2, 1, 1), tok.expand(2, -1, -1)], dim=1)
                b, _ = pipe.denoise_latents(cat, pooled.repeat(2, 1), reference_latents=ref, **kw)
                assert torch.equal(a, b), (graphs, ref is not None, per_seed)
                again, _ = pipe.denoise_latents(cond, pooled, redux_image=prompt, reference_latents=ref, **kw)
                assert torch.equal(again, a)
                results[(graphs, ref is not None, per_seed)] = a
    for key in [k for k in results if k[0]]:
        assert torch.equal(results[key], results[(False,) + key[1:]])
    assert not torch.equal(results[(True, False, False)], results[(True, False, True)])


def test_generate_image_logs_the_encode(kc):
    from tests.test_guidance_cpu import tiny_dev_config

    cfg = tiny_dev_config()
    pipe = _pipe(cfg, _mmdit_weights(cfg), _vae_weights())
    cond, pooled = pipe.synthetic_text_embeddings(n_images=1, text_len=T)
    imgs = _images(2, 130, seed=6)
    out, log = pipe.generate_image("", num_steps=STEPS, latent_size=LAT, seed=SEEDS, verbose=False, conditioning=cond,
                                   pooled_conditioning=pooled, redux_image=imgs[0])
    red = log["denoising"]["redux"]
    assert red["images"] == 1 and red["tokens"] == 49 and red["time"] >= 0.0 and len(out) == 2
    _, log = pipe.generate_image("", num_steps=STEPS, latent_size=LAT, seed=SEEDS, verbose=False, conditioning=cond,
                                 pooled_conditioning=pooled, redux_image=imgs)
    assert log["denoising"]["redux"]["images"] == 2
    _, log = pipe.generate_image("", num_steps=STEPS, latent_size=LAT, seed=SEEDS, verbose=False, conditioning=cond,
                                 pooled_conditioning=pooled)
    assert "redux" not in log["denoising"]


def test_no_redux_path_is_unchanged(kc):
    """without an image prompt, outputs and the op list equal those of a pipeline that never loaded Redux"""
    from tests.test_kontext_gpu import _op_list
    from tests.test_guidance_cpu import tiny_dev_config

    cfg = tiny_dev_config()
    p16 = _mmdit_weights(cfg)
    with_redux, plain = _pipe(cfg, p16), _pipe(cfg, p16, redux=False)
    cond, pooled = plain.synthetic_text_embeddings(n_images=1, text_len=T)
    kw = dict(num_steps=STEPS, latent_size=LAT, seed=SEEDS, guidance=3.0)
    with_redux.denoise_latents(cond, pooled, redux_image=_images(1, 100)[0], **kw)      # an image prompt came before
    outs = []
    for graphs in (True, False):
        for pipe in (with_redux, plain):
            pipe.mmdit.use_cuda_graphs = graphs
            lat, _ = pipe.denoise_latents(cond, pooled, **kw)
            outs.append(lat.clone())
    assert all(torch.equal(o, outs[0]) for o in outs[1:])
    g = torch.Generator().manual_seed(5)
    latent = torch.randn((2, *LAT, 16), generator=g).to(bf16)
    text = torch.randn((2, T, cfg.token_level_text_embed_dim), generator=g).to(bf16)
    pooled_m = torch.randn((2, cfg.pooled_text_embed_dim), generator=g).to(bf16).to(DEV)
    lists = []
    for pipe in (with_redux, plain):
        pipe.mmdit.cache_modulation_params(pooled_m, [752.0, 0.0], [3.5, 3.5])
        lists.append(_op_list(pipe.mmdit, latent, text))
    assert lists[0] == lists[1] and len(lists[0]) > 0


def test_errors_launch_nothing(kc):
    from diffusionkit_b200 import DkError, ops
    from diffusionkit_b200.config import tiny_siglip_config
    from tests.test_guidance_cpu import tiny_dev_config

    cfg = tiny_dev_config()
    p16 = _mmdit_weights(cfg)
    pipe, bare = _pipe(cfg, p16), _pipe(cfg, p16, redux=False)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=1, text_len=T)
    img = _images(1, 100)[0]
    base = dict(num_steps=STEPS, latent_size=LAT, seed=SEEDS)
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    for p, kw, err in [(pipe, dict(redux_image=img, cfg_weight=2.0), ValueError),
                       (pipe, dict(redux_image=[img]), ValueError),
                       (pipe, dict(redux_image=[img, img, img]), ValueError),
                       (pipe, dict(redux_image=np.zeros((64, 64, 2), np.uint8)), ValueError),
                       (bare, dict(redux_image=img), DkError)]:
        c = torch.cat([cond, cond]) if kw.get("cfg_weight") else cond
        pc = torch.cat([pooled, pooled]) if kw.get("cfg_weight") else pooled
        with pytest.raises(err):
            p.denoise_latents(c, pc, **base, **kw)
        with pytest.raises(err):
            p.generate_image("", verbose=False, conditioning=c, pooled_conditioning=pc, **base, **kw)
    with pytest.raises(DkError):
        bare.encode_redux(img)
    scfg = tiny_siglip_config()
    sp, rp = _encoder_weights(scfg, 256)
    with pytest.raises(ValueError, match="token_level_text_embed_dim"):     # a projector for another text width
        bare.load_redux(sp, rp, siglip_config=scfg)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0
