"""GPU checks of FLUX.1 Kontext editing (DESIGN.md §14): the MMDiT with reference tokens against the ids-driven oracle
(tests/kontext_ref.py) at tiny and full width, a launch census of the full-width run, the no-reference path unchanged,
the tiny pipelines against the oracle pipeline, composition with the step cache, FP8 and LoRA, the checkpoint preset,
and the argument errors.  Weights go through kontext_ref.sharpen, so that the reference's position matters enough for
the bounds to see it."""
import math
import os
import tempfile
from dataclasses import replace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
bf16 = torch.bfloat16
KONTEXT = "black-forest-labs/FLUX.1-Kontext-dev"
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


def _dev():
    from tests.test_guidance_cpu import tiny_dev_config

    return tiny_dev_config()


def _weights(cfg, seed=7):
    """generated in fp32 on the host, sharpened and rounded, so the oracle sees exactly the device's weights"""
    from diffusionkit_b200.weights import init_params, mmdit_param_specs
    from tests.kontext_ref import sharpen

    p = sharpen(init_params(mmdit_param_specs(cfg), seed=seed, dtype=torch.float32))
    return {k: v.to(bf16) for k, v in p.items()}


def _vae_weights(encoder=False, seed=None):
    from diffusionkit_b200.config import VAEDecoderConfig, VAEEncoderConfig
    from diffusionkit_b200.weights import init_params, vae_decoder_param_specs, vae_encoder_param_specs

    specs = vae_encoder_param_specs(VAEEncoderConfig()) if encoder else vae_decoder_param_specs(VAEDecoderConfig())
    return {k: v.to(bf16) for k, v in init_params(specs, seed=seed or (9 if encoder else 8),
                                                   dtype=torch.float32).items()}


def _pipe(cfg, p16, vp16=None, ep16=None, **kw):
    import diffusionkit_b200 as dk

    def dev(p):
        return None if p is None else {k: v.to(DEV) for k, v in p.items()}

    return dk.FluxPipeline(w16=True, a16=True, shift=1.0, mmdit_config=cfg, params=dev(p16), vae_params=dev(vp16),
                           vae_encoder_params=dev(ep16), load_decoder=vp16 is not None, **kw)


def _inputs(cfg, B, lat, ref, T_txt, seed=5):
    """bf16 host tensors: latent, reference (one per sequence), text, pooled"""
    g = torch.Generator().manual_seed(seed)
    latent = torch.randn((B, lat[0], lat[1], 16), generator=g).to(bf16)
    reference = torch.randn((B, ref[0], ref[1], 16), generator=g).to(bf16)
    text = torch.randn((B, T_txt, cfg.token_level_text_embed_dim), generator=g).to(bf16)
    pooled = torch.randn((B, cfg.pooled_text_embed_dim), generator=g).to(bf16)
    return latent, reference, text, pooled


def _oracle_forward(cfg, p16, latent, reference, text, pooled, tval, guidance):
    from tests.kontext_ref import KontextMMDiTRef
    from tests.oracle_bridge import ref_config

    t = torch.tensor([tval])
    ref = KontextMMDiTRef(ref_config(cfg), {k: v.float() for k, v in p16.items()})
    ref.cache_modulation_params(pooled.float(), t, guidance)
    return ref(latent.float(), text.float(), t.repeat(latent.shape[0]),
               reference=None if reference is None else reference.float())


def _engine(cfg, p16, pooled, guidance, tval=752.0):
    import diffusionkit_b200 as dk

    m = dk.MMDiT(cfg, {k: v.to(DEV) for k, v in p16.items()})
    m.cache_modulation_params(pooled.to(DEV), [tval, 0.0], guidance)
    return m


def _fwd(m, latent, text, reference=None, tval=752.0):
    out = m(latent.to(DEV), text.to(DEV), timestep=tval, reference=None if reference is None else reference.to(DEV))
    torch.cuda.synchronize()
    return out.clone()


def _check(got, want, what):
    from tests.model_checks import psnr, rel_l2

    got = got.float().cpu()
    assert got.shape == want.shape and bool(torch.isfinite(got).all())
    r, ps = rel_l2(got, want), psnr(want, got)
    print(f"{what}: rel_l2 {r:.3e}, psnr {ps:.1f} dB")
    assert r <= 2e-2 and ps >= 35.0, f"{what}: rel_l2={r:.3e} psnr={ps:.1f}"


# ------------------------------------------------------------------------------------------------ MMDiT
@pytest.mark.parametrize("B, lat, ref, guidance", [
    (1, (8, 8), (8, 8), [3.5]),                      # reference of the target's size
    (2, (16, 16), (16, 32), [2.5, 5.0]),             # another shape, per-image guidance
    (2, (8, 12), (8, 12), [3.5, 3.5]),               # two different references, one per seed
])
def test_tiny_forward_against_the_oracle(kc, B, lat, ref, guidance):
    cfg = _dev()
    p16 = _weights(cfg)
    latent, reference, text, pooled = _inputs(cfg, B, lat, ref, T)
    want = _oracle_forward(cfg, p16, latent, reference, text, pooled, 752.0, guidance)
    m = _engine(cfg, p16, pooled, guidance)
    _check(_fwd(m, latent, text, reference), want, f"B={B} target {lat} reference {ref}")


def test_fullwidth_against_the_oracle_under_a_census(kc):
    """FLUX.1-dev's width (h = 3072), 1 double + 1 single block, target 64 x 64, reference 64 x 128, T = 512, B = 2,
    eager under the launch census; the x-embedder remap and the final-layer gather are seen in it"""
    from diffusionkit_b200 import ops
    from diffusionkit_b200.config import FLUX_DEV
    from tests import launch_parity as lp

    cfg = replace(FLUX_DEV, depth_multimodal=1, depth_unified=1)
    assert cfg.hidden_size == 3072 and cfg.guidance_embed
    B, lat, ref, guidance = 2, (64, 64), (64, 128), [3.5, 5.0]
    p16 = _weights(cfg)
    latent, reference, text, pooled = _inputs(cfg, B, lat, ref, 512)
    Nx, Nr = (lat[0] // 2) * (lat[1] // 2), (ref[0] // 2) * (ref[1] // 2)
    m = _engine(cfg, p16, pooled, guidance)
    m.use_cuda_graphs = False
    c = lp.Census()
    c.run = "kontext-fullwidth"
    x_embeds = []
    with lp.census(c):
        checked_gemm = ops.gemm

        def spy(A, W, *args, **kw):
            if W.data_ptr() == m.w_x.data_ptr():
                x_embeds.append((A.shape[0], kw.get("rows_per_batch"), kw.get("out_batch_rows"),
                                 kw.get("out_row_off")))
            return checked_gemm(A, W, *args, **kw)

        ops.gemm = spy
        got = _fwd(m, latent, text, reference)
    print(c.table())
    assert x_embeds == [(B * Nx, Nx, Nx + Nr, 0), (B * Nr, Nr, Nx + Nr, Nx)], x_embeds
    gathers = [r for r in c.records if r["op"] == "copy_rows" and r["info"].get("src") == (Nx + Nr, 0)
               and r["info"].get("dst") == (Nx, 0) and r["info"].get("rows") == Nx]
    assert len(gathers) == 1, "the final layer's target-row gather"
    del m
    torch.cuda.empty_cache()
    want = _oracle_forward(cfg, p16, latent, reference, text, pooled, 752.0, guidance)
    _check(got, want, "full width, target 64x64, reference 64x128")


def test_no_reference_path_is_unchanged(kc):
    """plain -> Kontext -> plain -> Kontext at another reference size -> again: plain outputs bit-identical, Kontext
    outputs bit-identical per shape, with graphs and eagerly; and a plain forward issues exactly the ops of a fresh
    MMDiT that never saw a reference"""
    cfg = _dev()
    p16 = _weights(cfg)
    latent, ref_a, text, pooled = _inputs(cfg, 2, LAT, (8, 12), T)
    _, ref_b, _, _ = _inputs(cfg, 2, LAT, (16, 8), T, seed=6)
    runs = {}
    for graphs in (True, False):
        m = _engine(cfg, p16, pooled, [3.5, 3.5])
        m.use_cuda_graphs = graphs
        seq = [None, ref_a, None, ref_b, ref_a, ref_b, None]
        outs = [_fwd(m, latent, text, r) for r in seq]
        assert torch.equal(outs[0], outs[2]) and torch.equal(outs[0], outs[6])
        assert torch.equal(outs[1], outs[4]) and torch.equal(outs[3], outs[5])
        assert not torch.equal(outs[0], outs[1]) and not torch.equal(outs[1], outs[3])
        runs[graphs] = outs[:4]
        del m
    for a, b in zip(runs[True], runs[False]):
        assert torch.equal(a, b)
    # the op list of a plain forward
    m_seen = _engine(cfg, p16, pooled, [3.5, 3.5])
    _fwd(m_seen, latent, text, ref_a)
    fresh = _engine(cfg, p16, pooled, [3.5, 3.5])
    lists = [_op_list(mm, latent, text) for mm in (m_seen, fresh)]
    assert lists[0] == lists[1] and len(lists[0]) > 0
    assert torch.equal(_fwd(m_seen, latent, text), runs[True][0])


def _op_list(m, latent, text):
    """every ops function the forward calls, with its tensor shapes / strides and other arguments, eagerly"""
    import inspect

    from diffusionkit_b200 import ops

    m.use_cuda_graphs = False
    calls = []
    saved = {n: f for n, f in vars(ops).items() if inspect.isfunction(f) and f.__module__ == ops.__name__}

    def wrap(name, fn):
        def w(*args, **kw):
            desc = [(tuple(a.shape), tuple(a.stride()), str(a.dtype)) if torch.is_tensor(a) else
                    (tuple(x.shape if torch.is_tensor(x) else x for x in a) if isinstance(a, tuple) else a)
                    for a in list(args) + [kw[k] for k in sorted(kw)]]
            calls.append((name, sorted(kw), repr(desc)))
            return fn(*args, **kw)
        return w

    try:
        for n, f in saved.items():
            setattr(ops, n, wrap(n, f))
        _fwd(m, latent, text)
    finally:
        for n, f in saved.items():
            setattr(ops, n, f)
    return calls


# ------------------------------------------------------------------------------------------------ pipelines
def _ref_latents(cfg, n, Hr, Wr, seed=21):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((n, Hr, Wr, 16), generator=g)


def _oracle_pipeline(cfg, p16, cond, pooled, refs, guidance, solver="euler", cfgw=0.0, x0s=None, sig=None,
                     decisions=None):
    from oracle import sampler_ref as sr
    from tests import solver_ref
    from tests.kontext_ref import KontextMMDiTRef, KontextSplitRef, kontext_pipeline_latents
    from tests.oracle_bridge import ref_config
    from tests.step_cache_ref import StepCacheRef

    sample = {"euler": sr.sample_euler, "dpmpp_2m": solver_ref.sample_dpmpp_2m}[solver]
    sampler = sr.FluxSamplerRef(1.0)
    if sig is None:
        sig = sr.get_sigmas(sampler, STEPS)
    if x0s is None:
        H, W = LAT
        x0s = [sampler.noise_scaling(float(sig[0]), sr.get_noise(s, H, W), sr.get_empty_latent(H, W)) for s in SEEDS]
    params = {k: v.float() for k, v in p16.items()}
    refs16 = [None if r is None else r.to(bf16).float()[None] for r in refs]
    if decisions is None:
        return kontext_pipeline_latents(lambda: KontextMMDiTRef(ref_config(cfg), params), sample, sig, x0s, cond,
                                        pooled, refs16, guidance, cfgw, bf16)
    outs = []                                       # the step cache: replay the engine's decisions per image
    for i, s in enumerate(SEEDS):
        split = KontextSplitRef(ref_config(cfg), params)
        split.reference = refs16[i]
        sc = StepCacheRef(split, decisions=decisions)
        x = sample(lambda xin, c, t, sc=sc: sc(xin, c, t), sc.cache_modulation_params, x0s[i], sig,
                   cond[[i]].float(), pooled[[i]].float(), cfgw, bf16)
        outs.append(sr.process_out(x, "flux"))
    return torch.cat(outs)


def _compare(pipe, vp16, latent, want, what):
    from oracle.vae_ref import VAEDecoderRef, decode_latents_to_image
    from tests.model_checks import psnr, rel_l2

    r = rel_l2(latent, want)
    img_want = decode_latents_to_image(VAEDecoderRef({k: v.float() for k, v in vp16.items()}), want.to(bf16).float())
    ps = psnr(img_want, pipe.decode_latents_to_image(latent))
    print(f"{what}: final latent rel_l2 {r:.3e}, decoded psnr {ps:.1f} dB")
    assert r <= 5e-2, f"{what}: final latent rel_l2 {r:.3e}"
    assert ps >= 30.0, f"{what}: decoded RGB psnr {ps:.1f}"


@pytest.mark.parametrize("solver, cfgw, per_seed", [("euler", 0.0, True), ("dpmpp_2m", 0.0, False),
                                                    ("euler", 2.0, True)])
def test_tiny_pipeline_against_the_oracle(kc, solver, cfgw, per_seed):
    cfg = _dev()
    p16, vp16 = _weights(cfg), _vae_weights()
    pipe = _pipe(cfg, p16, vp16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
    if cfgw > 0:                                                # [positive x B | negative x B]
        cond2, pooled2 = pipe.synthetic_text_embeddings(n_images=len(SEEDS), seed=99, text_len=T)
        cond, pooled = torch.cat([cond, cond2]), torch.cat([pooled, pooled2])
    refs = _ref_latents(cfg, 2 if per_seed else 1, 8, 16)
    guidance = 2.5 if cfgw == 0 else [2.5, 4.0]
    lat, it = pipe.denoise_latents(cond, pooled, num_steps=STEPS, cfg_weight=cfgw, latent_size=LAT, seed=SEEDS,
                                   solver=solver, guidance=guidance, reference_latents=refs.to(DEV))
    torch.cuda.synchronize()
    assert lat.shape == (len(SEEDS), *LAT, 16) and len(it) == STEPS
    per_image = [guidance] * 2 if not isinstance(guidance, list) else guidance
    want = _oracle_pipeline(cfg, p16, cond, pooled, [refs[i if per_seed else 0] for i in range(2)], per_image, solver,
                            cfgw)
    _compare(pipe, vp16, lat, want, f"{solver} cfg {cfgw}")
    plain, _ = pipe.denoise_latents(cond, pooled, num_steps=STEPS, cfg_weight=cfgw, latent_size=LAT, seed=SEEDS,
                                    solver=solver, guidance=guidance)
    assert not torch.equal(plain, lat)


@pytest.mark.parametrize("img2img", [False, True])
def test_tiny_pipeline_with_a_reference_image(kc, img2img):
    """reference_image through the VAE encoder (its posterior mean), optionally with img2img at denoise 0.6"""
    from oracle import sampler_ref as sr
    from oracle.vae_ref import VAEEncoderRef, encode_image_to_latents, read_image_array
    from tests.model_checks import _test_image

    cfg = _dev()
    p16, vp16, ep16 = _weights(cfg), _vae_weights(), _vae_weights(encoder=True)
    pipe = _pipe(cfg, p16, vp16, ep16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
    ref_img = _test_image(64, 128, seed=7)
    src_img = _test_image(128, 64, seed=8)                     # target latent 16 x 8
    kw = dict(image_path=src_img, denoise=0.6) if img2img else dict(latent_size=LAT)
    lat, it = pipe.denoise_latents(cond, pooled, num_steps=STEPS, seed=SEEDS, guidance=3.0, reference_image=ref_img,
                                   **kw)
    torch.cuda.synchronize()
    enc = VAEEncoderRef({k: v.float() for k, v in ep16.items()})
    mean = encode_image_to_latents(enc, read_image_array(torch.from_numpy(ref_img)), torch.zeros(1, 8, 16, 16))
    reference = ((mean - 0.1159) * 0.3611)[0]                  # FluxLatentFormat.process_in
    sampler = sr.FluxSamplerRef(1.0)
    sig = sr.get_sigmas(sampler, STEPS)
    x0s = None
    if img2img:
        sig = sig[int(STEPS * (1 - 0.6)):]
        image = read_image_array(torch.from_numpy(src_img))
        x0s = []
        for s in SEEDS:
            noise = sr.get_noise(s, 16, 8)
            x_T = (encode_image_to_latents(enc, image, noise) - 0.1159) * 0.3611
            x0s.append(sampler.noise_scaling(float(sig[0]), noise, x_T))
    assert len(it) == len(sig) - 1
    want = _oracle_pipeline(cfg, p16, cond, pooled, [reference, reference], [3.0, 3.0], x0s=x0s, sig=sig)
    _compare(pipe, vp16, lat, want, f"reference image, img2img {img2img}")
    out, log = pipe.generate_image("", num_steps=STEPS, seed=SEEDS, verbose=False, conditioning=cond,
                                   pooled_conditioning=pooled, guidance=3.0, reference_image=ref_img, **kw)
    assert log["denoising"]["reference"] == {"latent_size": (8, 16), "tokens": 32}
    got = pipe.decode_latents_to_image(lat)
    assert len(out) == 2 and np.asarray(out[0]).shape == tuple(got.shape[1:])


# ------------------------------------------------------------------------------------------------ composition
def test_step_cache_with_a_reference(kc):
    """threshold 0 is bit-identical to the cache off; threshold inf with cap 1 matches the oracle replaying the same
    decisions, the rule running over target and reference tokens"""
    from diffusionkit_b200.config import tiny_flux_config

    cfg = tiny_flux_config()
    p16, vp16 = _weights(cfg), _vae_weights()
    pipe = _pipe(cfg, p16, vp16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
    refs = _ref_latents(cfg, 2, 8, 8)
    kw = dict(num_steps=STEPS, latent_size=LAT, seed=SEEDS, reference_latents=refs.to(DEV))
    off, _ = pipe.denoise_latents(cond, pooled, **kw)
    off = off.clone()
    pipe.set_step_cache(0.0)
    zero, _ = pipe.denoise_latents(cond, pooled, **kw)
    assert torch.equal(zero, off)
    pipe.set_step_cache(math.inf, 1)
    cached, _ = pipe.denoise_latents(cond, pooled, **kw)
    torch.cuda.synchronize()
    decisions = [s for _, s in pipe.mmdit.step_cache_log]
    assert decisions == [False, True, False, True], decisions
    want = _oracle_pipeline(cfg, p16, cond, pooled, [refs[0], refs[1]], [None, None], decisions=decisions)
    _compare(pipe, vp16, cached, want, "step cache inf, cap 1")


def test_fp8_with_a_reference(kc):
    from tests.model_checks import psnr

    cfg = _dev()
    p16, vp16 = _weights(cfg), _vae_weights()
    pipe = _pipe(cfg, p16, vp16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
    kw = dict(num_steps=STEPS, latent_size=LAT, seed=SEEDS, reference_latents=_ref_latents(cfg, 1, 8, 12).to(DEV))
    a, _ = pipe.denoise_latents(cond, pooled, **kw)
    a = a.clone()
    pipe.set_fp8(True)
    b, _ = pipe.denoise_latents(cond, pooled, **kw)
    ps = psnr(pipe.decode_latents_to_image(a), pipe.decode_latents_to_image(b))
    print(f"fp8 vs 16-bit with a reference: decoded psnr {ps:.1f} dB")
    assert ps >= 20.0


def test_lora_unload_restores_the_kontext_output(kc):
    from tests.lora_fixtures import make_factors, peft_dict

    cfg = _dev()
    p16 = _weights(cfg)
    pipe = _pipe(cfg, p16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
    kw = dict(num_steps=STEPS, latent_size=LAT, seed=SEEDS, reference_latents=_ref_latents(cfg, 2, 8, 12).to(DEV))
    base, _ = pipe.denoise_latents(cond, pooled, **kw)
    base = base.clone()
    h = cfg.hidden_size
    factors = make_factors({"double_blocks.0.img_attn.proj": (h, h), "single_blocks.0.linear2": (h, 5 * h)}, rank=4,
                           seed=6, gain=0.5)
    pipe.load_lora_weights(peft_dict(factors, "diffusion_model."), scale=1.0, adapter_name="k")
    merged, _ = pipe.denoise_latents(cond, pooled, **kw)
    assert not torch.equal(merged, base)
    pipe.unload_lora_weights()
    again, _ = pipe.denoise_latents(cond, pooled, **kw)
    assert torch.equal(again, base)


def test_checkpoint_under_the_kontext_preset(kc):
    import diffusionkit_b200 as dk
    from safetensors.torch import save_file

    from tests.test_guidance_cpu import dev_upstream

    cfg = _dev()
    p16 = _weights(cfg)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "flux1-kontext-dev.safetensors")
        save_file({k: v.contiguous() for k, v in dev_upstream(p16, cfg).items()}, path)
        a = dk.FluxPipeline(w16=True, a16=True, shift=1.0, model_version=KONTEXT, mmdit_config=cfg, local_ckpt=path,
                            load_decoder=False)
    b = _pipe(cfg, p16, model_version=KONTEXT)
    cond, pooled = a.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
    kw = dict(num_steps=STEPS, latent_size=LAT, seed=SEEDS, reference_latents=_ref_latents(cfg, 1, 8, 12).to(DEV))
    la, _ = a.denoise_latents(cond, pooled, **kw)
    la = la.clone()
    lb, _ = b.denoise_latents(cond, pooled, **kw)
    assert torch.equal(la, lb)


# ------------------------------------------------------------------------------------------------ errors
def test_errors_launch_nothing(kc):
    import diffusionkit_b200 as dk
    from diffusionkit_b200 import ops
    from diffusionkit_b200.config import tiny_sd3_config, tiny_sd35_medium_config
    from diffusionkit_b200.weights import init_params, mmdit_param_specs

    cfg = _dev()
    pipe = _pipe(cfg, _weights(cfg))
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
    latent, reference, text, pooled_m = _inputs(cfg, 2, LAT, (8, 12), T)
    m = pipe.mmdit
    m.cache_modulation_params(pooled_m.to(DEV), [752.0], [3.5, 3.5])
    sd3 = []
    for c in (tiny_sd3_config(), tiny_sd35_medium_config()):
        mm = dk.MMDiT(c, init_params(mmdit_param_specs(c), seed=0, dtype=torch.float16, device=DEV))
        g = torch.Generator().manual_seed(1)
        mm.cache_modulation_params(torch.randn((2, c.pooled_text_embed_dim), generator=g).half().to(DEV), [752.0])
        sd3.append((mm, torch.randn((2, T, c.token_level_text_embed_dim), generator=g).half().to(DEV)))
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    lat_d, ref_d, text_d = latent.to(DEV), reference.to(DEV), text.to(DEV)
    for mm, tt in sd3:                                              # SD3 / SD3.5
        with pytest.raises(ValueError, match="FLUX-shaped"):
            mm(lat_d.half(), tt, timestep=752.0, reference=ref_d.half())
    for bad in (ref_d[:, :7], ref_d[:, :, :11], ref_d[:1], ref_d[..., :8]):     # odd Hr, odd Wr, batch, channels
        with pytest.raises(ValueError):
            m(lat_d, text_d, timestep=752.0, reference=bad)
    base = dict(num_steps=STEPS, latent_size=LAT, seed=SEEDS)
    cases = [dict(reference_latents=torch.zeros((1, 7, 12, 16), device=DEV)),
             dict(reference_latents=torch.zeros((1, 8, 13, 16), device=DEV)),
             dict(reference_latents=torch.zeros((3, 8, 12, 16), device=DEV)),
             dict(reference_latents=torch.zeros((1, 8, 12, 16), device=DEV),
                  reference_image=np.zeros((64, 64, 3), dtype=np.uint8)),
             dict(reference_image=np.zeros((64, 64), dtype=np.uint8))]
    from PIL import Image

    cases.append(dict(reference_image=Image.new("L", (64, 64))))
    for kw in cases:
        with pytest.raises(ValueError):
            pipe.denoise_latents(cond, pooled, **base, **kw)
        with pytest.raises(ValueError):
            pipe.generate_image("", verbose=False, conditioning=cond, pooled_conditioning=pooled, **base, **kw)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0
    assert not hasattr(pipe, "encoder")                             # nothing was encoded either
