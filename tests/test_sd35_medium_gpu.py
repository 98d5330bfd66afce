"""GPU checks of SD3.5 Medium (MMDiT-X) and skip-layer guidance (DESIGN.md §13): the MMDiT against the oracle
(tests/sd35_medium_ref.py) tiny and at full width, the skip forward, the four *_slg solver kernels, the tiny pipeline
under every solver with SLG off and on, the checkpoint file, LoRA on attn2, FP8, determinism and the argument errors."""
import os
import tempfile
from dataclasses import replace

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
bf16, fp16 = torch.bfloat16, torch.float16
LAT = (8, 12)
SEEDS = [11, 12]
STEPS = 6
T = 24
CFGW = 4.5
MEDIUM = "stabilityai/stable-diffusion-3.5-medium"


@pytest.fixture(scope="module")
def kc():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    from tests import kernel_checks

    kernel_checks._setup()
    return kernel_checks


def _cfg(dtype=fp16):
    from diffusionkit_b200.config import tiny_sd35_medium_config

    cfg = tiny_sd35_medium_config()
    return cfg if dtype == fp16 else replace(cfg, dtype=dtype, float16_dtype=dtype)


def _weights(cfg, dtype=fp16, seed=7):
    """generated in fp32 on the host and rounded, so the oracle sees exactly the device's weights"""
    from diffusionkit_b200.weights import init_params, mmdit_param_specs

    return {k: v.to(dtype) for k, v in init_params(mmdit_param_specs(cfg), seed=seed, dtype=torch.float32).items()}


def _vae_weights():
    from diffusionkit_b200.config import VAEDecoderConfig
    from diffusionkit_b200.weights import init_params, vae_decoder_param_specs

    return {k: v.to(fp16) for k, v in init_params(vae_decoder_param_specs(VAEDecoderConfig()), seed=8,
                                                   dtype=torch.float32).items()}


def _xref(cfg, p16):
    from tests.oracle_bridge import ref_config
    from tests.sd35_medium_ref import MMDiTXRef

    return MMDiTXRef(ref_config(cfg), {k: v.float() for k, v in p16.items()}, x_layers=cfg.x_block_self_attn_layers,
                     k_bias=cfg.attn_k_bias)


def _pipe(cfg, p16, vp16=None, **kw):
    import diffusionkit_b200 as dk

    return dk.DiffusionPipeline(w16=True, a16=True, shift=3.0, model_version=MEDIUM, mmdit_config=cfg,
                                params={k: v.to(DEV) for k, v in p16.items()},
                                vae_params=None if vp16 is None else {k: v.to(DEV) for k, v in vp16.items()},
                                load_decoder=vp16 is not None, **kw)


def _cond(pipe):
    """[positive x B | negative x B] synthetic text embeddings"""
    return pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)


def _denoise(pipe, cond, pooled, **kw):
    lat, it = pipe.denoise_latents(cond, pooled, num_steps=STEPS, cfg_weight=CFGW, latent_size=LAT, seed=SEEDS, **kw)
    torch.cuda.synchronize()
    return lat.clone(), it


def _slg(**kw):
    from diffusionkit_b200.sampler import SkipLayerGuidance

    return SkipLayerGuidance(**{**dict(scale=2.5, layers=(1,), start=0.1, end=0.7), **kw})   # steps 1..4 of 6


# ------------------------------------------------------------------------------------------------ MMDiT
def _mmdit_vs_oracle(cfg, dtype, B, lat, T_txt, skip_layers=(), seed=7):
    import diffusionkit_b200 as dk
    from tests.model_checks import psnr, rel_l2

    p16 = _weights(cfg, dtype, seed)
    gen = torch.Generator().manual_seed(5)
    latent = torch.randn((B, lat[0], lat[1], 16), generator=gen).to(dtype)
    text = torch.randn((B, T_txt, cfg.token_level_text_embed_dim), generator=gen).to(dtype)
    pooled = torch.randn((B, cfg.pooled_text_embed_dim), generator=gen).to(dtype)
    tval = 752.0
    t = torch.tensor([tval])
    ref = _xref(cfg, p16)
    ref.cache_modulation_params(pooled.float(), t)
    want = ref(latent.float(), text.float(), t.repeat(B), skip_layers=skip_layers)
    del ref
    m = dk.MMDiT(cfg, {k: v.to(DEV) for k, v in p16.items()})
    del p16
    if skip_layers:
        # the skip rows trail a leading copy of themselves: [rows | rows skipping]
        m.cache_modulation_params(torch.cat([pooled, pooled]).to(DEV), [tval], skip_batch=B)
        got = m(latent_image_embeddings=torch.cat([latent, latent]).to(DEV),
                token_level_text_embeddings=torch.cat([text, text]).to(DEV), timestep=tval,
                skip_layers=skip_layers, skip_batch=B)[B:].float().cpu()
    else:
        m.cache_modulation_params(pooled.to(DEV), [tval, 0.0])
        got = m(latent_image_embeddings=latent.to(DEV), token_level_text_embeddings=text.to(DEV).unsqueeze(2),
                timestep=torch.full((B,), tval)).float().cpu()
    torch.cuda.synchronize()
    del m
    assert got.shape == want.shape and bool(torch.isfinite(got).all())
    r, ps = rel_l2(got, want), psnr(want, got)
    print(f"{dtype} B={B} lat={lat} T={T_txt} skip={skip_layers}: mmdit rel_l2 {r:.3e}, psnr {ps:.1f} dB")
    assert r <= 2e-2 and ps >= 35.0, f"mmdit rel_l2={r:.3e} psnr={ps:.1f}"


@pytest.mark.parametrize("dtype", [fp16, bf16])
@pytest.mark.parametrize("B", [1, 2])
def test_tiny_mmdit_against_the_oracle(kc, dtype, B):
    _mmdit_vs_oracle(_cfg(dtype), dtype, B, LAT, T)


def test_fullwidth_truncated_depth_against_the_oracle(kc):
    """SD3.5 Medium at its real width (h = 1536, 24 heads) through 3 joint blocks, x-layers 0 and 1 (the last text
    block pre-only), 1024^2 (latent 128^2) and the SD3 text length 77 + 512"""
    from diffusionkit_b200.config import SD35_MEDIUM

    cfg = replace(SD35_MEDIUM, depth_multimodal=3, hidden_size_override=1536, x_block_self_attn_layers=(0, 1))
    assert cfg.hidden_size == 1536 and cfg.num_heads == 24
    _mmdit_vs_oracle(cfg, fp16, 2, (128, 128), 589)


def test_skip_forward(kc):
    """a 3B skip forward: its leading 2B sequences are bit-identical to the 2B forward, its trailing B are the oracle
    forward that skips the listed blocks"""
    import diffusionkit_b200 as dk

    cfg = _cfg()
    _mmdit_vs_oracle(cfg, fp16, 2, LAT, T, skip_layers=(1,))
    _mmdit_vs_oracle(cfg, fp16, 1, LAT, T, skip_layers=(0, 2))
    p16 = _weights(cfg)
    m = dk.MMDiT(cfg, {k: v.to(DEV) for k, v in p16.items()})
    B = 2
    g = torch.Generator().manual_seed(9)
    x = torch.randn((3 * B, *LAT, 16), generator=g).to(fp16).to(DEV)
    text = torch.randn((3 * B, T, cfg.token_level_text_embed_dim), generator=g).to(fp16).to(DEV)
    pooled = torch.randn((3 * B, cfg.pooled_text_embed_dim), generator=g).to(fp16).to(DEV)
    m.cache_modulation_params(pooled, [500.0], skip_batch=B)
    for graphs in (True, False):
        m.use_cuda_graphs = graphs
        two = m(x[:2 * B], text[:2 * B], 500.0).clone()
        three = m(x, text, 500.0, skip_layers=(1,), skip_batch=B).clone()
        assert torch.equal(three[:2 * B], two), graphs
        assert not torch.equal(three[2 * B:], three[:B])
    # a forward whose batch matches neither the cache nor its leading rows is refused
    with pytest.raises(dk.DkError, match="modulation cache"):
        m(x[:B], text[:B], 500.0)


# ------------------------------------------------------------------------------------------------ kernels
N_ODD = 3 * 4099


def _inputs(dtype, n, seed, reps=3):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn((n,), generator=g, device=DEV)
    xin = torch.randn((reps * n,), generator=g, device=DEV).to(dtype)
    out = torch.randn((reps * n,), generator=g, device=DEV).to(dtype)
    return x, xin, out


def _ref_d(xin, out, sigma, cfg, slg, n):
    den = xin.float() - out.float() * sigma
    pos, neg, skip = den[:n], den[n:2 * n], den[2 * n:]
    return neg + cfg * (pos - neg) + slg * (pos - skip)


@pytest.mark.parametrize("dtype", [fp16, bf16])
def test_slg_kernels(kc, dtype):
    from diffusionkit_b200 import ops

    n, sigma, sigma_next, w, s = N_ODD, 0.6875, 0.5, 4.5, 2.5
    x, xin, out = _inputs(dtype, n, 1)
    D = _ref_d(xin, out, sigma, w, s, n)
    kc._assert_close("step_slg", ops.sampler_step(x.clone(), xin, out, sigma, sigma_next, w, slg=s),
                     x + (x - D) / sigma * (sigma_next - sigma), 1e-6)
    d, x2 = ops.sampler_heun_predict(x, xin, out, sigma, sigma_next, w, slg=s)
    kc._assert_close("heun_predict_slg_d", d, (x - D) / sigma, 1e-6)
    kc._assert_close("heun_predict_slg_x2", x2, x + (x - D) / sigma * (sigma_next - sigma), 1e-6)
    _, xin2, out2 = _inputs(dtype, n, 2)
    d2 = (x2 - _ref_d(xin2, out2, sigma_next, w, s, n)) / sigma_next
    kc._assert_close("heun_correct_slg", ops.sampler_heun_correct(x.clone(), d, x2, xin2, out2, sigma, sigma_next, w,
                                                                  slg=s), x + (d + d2) / 2 * (sigma_next - sigma), 1e-6)
    a, b, c = 0.75, 0.3, -0.05
    d_prev = torch.randn((n,), device=DEV)
    got_prev = d_prev.clone()
    got = ops.sampler_dpmpp_2m(x.clone(), got_prev, xin, out, sigma, a, b, c, w, slg=s)
    kc._assert_close("dpmpp_2m_slg", got, a * x + b * D + c * d_prev, 1e-6)
    kc._assert_close("dpmpp_2m_slg_d_prev", got_prev, D, 1e-6)


@pytest.mark.parametrize("dtype", [fp16, bf16])
def test_slg_kernels_at_zero_are_the_plain_ones(kc, dtype):
    from diffusionkit_b200 import ops
    from diffusionkit_b200._lib import dtype_code, ptr

    c = ops.ctx(0)
    n, sigma, sigma_next, w = N_ODD, 0.6875, 0.5, 4.5
    x, xin, out = _inputs(dtype, n, 3)
    dt = dtype_code(dtype)

    def both(fn):
        a, b = fn(None), fn(0.0)
        for u, v in zip(a, b):
            assert torch.equal(u, v)

    def step(slg):
        y = x.clone()
        args = (dt, ptr(y), ptr(xin), ptr(out), n, sigma, sigma_next, w)
        c.call("dk_sampler_step", *args) if slg is None else c.call("dk_sampler_step_slg", *args, slg)
        return (y,)

    def predict(slg):
        d, x2 = torch.empty_like(x), torch.empty_like(x)
        args = (dt, ptr(x), ptr(xin), ptr(out), ptr(d), ptr(x2), n, sigma, sigma_next, w)
        c.call("dk_sampler_heun_predict", *args) if slg is None else c.call("dk_sampler_heun_predict_slg", *args, slg)
        return d, x2

    d, x2 = predict(None)

    def correct(slg):
        y = x.clone()
        args = (dt, ptr(y), ptr(d), ptr(x2), ptr(xin), ptr(out), n, sigma, sigma_next, w)
        c.call("dk_sampler_heun_correct", *args) if slg is None else c.call("dk_sampler_heun_correct_slg", *args, slg)
        return (y,)

    d_prev = torch.randn((n,), device=DEV)

    def dpm(slg):
        y, p = x.clone(), d_prev.clone()
        args = (dt, ptr(y), ptr(p), ptr(xin), ptr(out), n, sigma, 0.75, 0.3, -0.05, w)
        c.call("dk_sampler_dpmpp_2m", *args) if slg is None else c.call("dk_sampler_dpmpp_2m_slg", *args, slg)
        return y, p

    for fn in (step, predict, correct, dpm):
        both(fn)
    torch.cuda.synchronize()


def test_slg_kernels_refuse_no_cfg(kc):
    from diffusionkit_b200 import DkError, ops

    c = ops.ctx(0)
    x, xin, out = _inputs(fp16, 64, 4)
    n0 = c.launches
    with pytest.raises(DkError, match="needs CFG"):
        ops.sampler_step(x, xin, out, 0.5, 0.25, 0.0, slg=2.5)
    with pytest.raises(DkError, match="finite"):
        ops.sampler_dpmpp_2m(x, x.clone(), xin, out, 0.5, 1.0, 0.5, 0.0, 4.5, slg=float("inf"))
    assert c.launches == n0


# ------------------------------------------------------------------------------------------------ pipelines
def _oracle_latents(cfg, p16, cond, pooled, solver, slg=None):
    """the oracle pipeline one image at a time ([pos, neg] rows) -> process_out latents"""
    from oracle import sampler_ref as sr
    from tests.sd35_medium_ref import sample

    smp = sr.ModelSamplingDiscreteFlowRef(3.0)
    sig = sr.get_sigmas(smp, STEPS)
    H, W = LAT
    n = len(SEEDS)
    kw = {} if slg is None else dict(scale=slg.scale, layers=slg.layers, start=slg.start, end=slg.end)
    outs = []
    for i, s in enumerate(SEEDS):
        ref = _xref(cfg, p16)
        x0 = smp.noise_scaling(float(sig[0]), sr.get_noise(s, H, W), sr.get_empty_latent(H, W))
        idx = [i, i + n]
        x = sample(solver, ref, x0, sig, cond[idx].float().cpu(), pooled[idx].float().cpu(), CFGW, fp16, **kw)
        outs.append(sr.process_out(x, "sd3"))
    return torch.cat(outs)


@pytest.mark.parametrize("solver", ["euler", "heun", "dpmpp_2m"])
def test_tiny_pipeline_against_the_oracle(kc, solver):
    from oracle.vae_ref import VAEDecoderRef, decode_latents_to_image
    from tests.model_checks import psnr, rel_l2

    cfg = _cfg()
    p16, vp16 = _weights(cfg), _vae_weights()
    pipe = _pipe(cfg, p16, vp16)
    cond, pooled = _cond(pipe)
    vae_ref = VAEDecoderRef({k: v.float() for k, v in vp16.items()})
    results = {}
    for slg in (None, _slg()):
        latent, it = _denoise(pipe, cond, pooled, solver=solver, slg=slg)
        assert latent.shape == (len(SEEDS), *LAT, 16) and len(it) == STEPS
        want = _oracle_latents(cfg, p16, cond, pooled, solver, slg)
        r = rel_l2(latent, want)
        ps = psnr(decode_latents_to_image(vae_ref, want.to(fp16).float()), pipe.decode_latents_to_image(latent))
        print(f"{solver} slg={slg}: final latent rel_l2 {r:.3e}, decoded psnr {ps:.1f} dB")
        assert r <= 5e-2, f"final latent rel_l2 {r:.3e}"
        assert ps >= 20.0, f"decoded RGB psnr {ps:.1f}"
        results[slg is None] = (latent, want)
    (on, want_on), (off, want_off) = results[False], results[True]
    print(f"{solver}: oracle slg on vs off rel_l2 {rel_l2(want_on, want_off):.3e}")
    assert not torch.equal(on, off)
    # slg=None is omitting it
    plain, _ = _denoise(pipe, cond, pooled, solver=solver)
    assert torch.equal(plain, off)
    # generate_image under CUDA graphs, and its log
    image, log = pipe.generate_image("", num_steps=STEPS, cfg_weight=CFGW, latent_size=LAT, seed=SEEDS[0],
                                     verbose=False, conditioning=cond[[0, len(SEEDS)]],
                                     pooled_conditioning=pooled[[0, len(SEEDS)]], solver=solver, slg=_slg())
    assert pipe.mmdit.use_cuda_graphs and image.size == (LAT[1] * 8, LAT[0] * 8)
    assert log["denoising"]["skip_layer_guidance"] == {"scale": 2.5, "layers": [1], "steps": [1, 2, 3, 4]}


def test_local_checkpoint(kc):
    from safetensors.torch import save_file

    from tests.test_sd35_medium_cpu import medium_upstream

    cfg = _cfg()
    p16 = _weights(cfg)
    import diffusionkit_b200 as dk

    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "sd3.5_medium.safetensors")
        save_file({k: v.contiguous() for k, v in medium_upstream(p16, cfg, vae=False).items()}, path)
        a = dk.DiffusionPipeline(w16=True, a16=True, shift=3.0, model_version=MEDIUM, mmdit_config=cfg,
                                 local_ckpt=path, load_decoder=False)
    b = _pipe(cfg, p16)
    cond, pooled = _cond(a)
    la, _ = _denoise(a, cond, pooled, slg=_slg())
    lb, _ = _denoise(b, cond, pooled, slg=_slg())
    assert torch.equal(la, lb)


def test_lora_on_attn2(kc):
    from diffusionkit_b200.lora import load_lora
    from tests.lora_fixtures import make_factors, merge_lora, peft_dict
    from tests.model_checks import psnr, rel_l2

    cfg = _cfg()
    p16 = _weights(cfg)
    pipe = _pipe(cfg, p16)
    m = pipe.mmdit
    h = cfg.hidden_size
    s0, s1 = m.attn2[0], m.attn2[1]
    w_qkv0, w_o1 = s0.w_qkv.clone(), s1.w_o.clone()
    factors = make_factors({"joint_blocks.0.x_block.attn2.qkv": (3 * h, h),
                            "joint_blocks.1.x_block.attn2.proj": (h, h)}, rank=4, seed=6, gain=0.5)
    sd = peft_dict(factors, "model.diffusion_model.")
    g = torch.Generator().manual_seed(3)
    B = 2
    latent = torch.randn((B, *LAT, 16), generator=g).to(fp16)
    text = torch.randn((B, T, cfg.token_level_text_embed_dim), generator=g).to(fp16)
    pooled = torch.randn((B, cfg.pooled_text_embed_dim), generator=g).to(fp16)

    def forward():
        m.cache_modulation_params(pooled.to(DEV), [600.0])
        return m(latent.to(DEV), text.to(DEV), 600.0).float().cpu()

    base = forward()
    pipe.load_lora_weights(sd, scale=0.8, adapter_name="x")
    assert not torch.equal(s0.w_qkv, w_qkv0) and not torch.equal(s1.w_o, w_o1)
    merged = forward()
    lora = load_lora(sd, cfg)
    ref = _xref(cfg, {k: v.to(fp16) for k, v in merge_lora(p16, [(lora.targets, 0.8)]).items()})
    ref.cache_modulation_params(pooled.float(), torch.tensor([600.0]))
    want = ref(latent.float(), text.float(), torch.full((B,), 600.0))
    r, ps = rel_l2(merged, want), psnr(want, merged)
    print(f"LoRA on attn2: rel_l2 {r:.3e}, psnr {ps:.1f} dB; merged vs base rel_l2 {rel_l2(merged, base):.3e}")
    assert r <= 2e-2 and ps >= 35.0 and rel_l2(merged, base) >= 10 * r
    pipe.unload_lora_weights()
    assert torch.equal(s0.w_qkv, w_qkv0) and torch.equal(s1.w_o, w_o1)
    assert torch.equal(forward(), base)


def test_fp8_with_attn2_and_slg(kc):
    from diffusionkit_b200.mmdit import fp8_covered_linears
    from tests.model_checks import psnr, rel_l2

    cfg = _cfg()
    p16, vp16 = _weights(cfg), _vae_weights()
    pipe = _pipe(cfg, p16, vp16)
    cond, pooled = _cond(pipe)
    keys = {(id(s), a) for s, a in [(pipe.mmdit.attn2[0], "w_qkv"), (pipe.mmdit.attn2[1], "w_o")]}
    ref, _ = _denoise(pipe, cond, pooled, slg=_slg())
    pipe.set_fp8(True)
    assert keys <= set(pipe.mmdit._fp8_w) and len(pipe.mmdit._fp8_packed()) > 0
    assert any(".attn2." in n for n in fp8_covered_linears(cfg))
    got, _ = _denoise(pipe, cond, pooled, slg=_slg())
    ps = psnr(pipe.decode_latents_to_image(ref), pipe.decode_latents_to_image(got))
    print(f"fp8 vs 16-bit with SLG: latent rel_l2 {rel_l2(got, ref):.3e}, decoded psnr {ps:.1f} dB")
    assert bool(torch.isfinite(got).all()) and ps >= 20.0 and not torch.equal(got, ref)
    pipe.set_fp8(False)


# ------------------------------------------------------------------------------------------------ determinism
@pytest.mark.parametrize("solver", ["euler", "heun", "dpmpp_2m"])
def test_step_cache_threshold_zero_changes_nothing(kc, solver):
    cfg = _cfg()
    pipe = _pipe(cfg, _weights(cfg))
    cond, pooled = _cond(pipe)
    for slg in (None, _slg()):
        pipe.set_step_cache(None)
        off, _ = _denoise(pipe, cond, pooled, solver=solver, slg=slg)
        pipe.set_step_cache(0.0)
        on, _ = _denoise(pipe, cond, pooled, solver=solver, slg=slg)
        assert torch.equal(on, off), slg
        assert not any(s for _, s in pipe.mmdit.step_cache_log)
    pipe.set_step_cache(None)


def test_graphs_eager_and_reruns_are_bit_identical(kc, monkeypatch):
    cfg = _cfg()
    p16 = _weights(cfg)
    runs = {}
    for graphs in ("1", "0"):
        monkeypatch.setenv("DK_CUDA_GRAPHS", graphs)
        pipe = _pipe(cfg, p16)
        assert pipe.mmdit.use_cuda_graphs == (graphs == "1")
        cond, pooled = _cond(pipe)
        for solver in ("euler", "heun", "dpmpp_2m"):
            a, _ = _denoise(pipe, cond, pooled, solver=solver, slg=_slg())
            b, _ = _denoise(pipe, cond, pooled, solver=solver, slg=_slg())
            assert torch.equal(a, b) and bool(torch.isfinite(a).all()), (graphs, solver)
            runs[graphs, solver] = a
        del pipe
    for solver in ("euler", "heun", "dpmpp_2m"):
        assert torch.equal(runs["1", solver], runs["0", solver]), solver


# ------------------------------------------------------------------------------------------------ errors
def test_errors_launch_nothing(kc):
    from diffusionkit_b200 import ops
    from diffusionkit_b200.sampler import SkipLayerGuidance

    cfg = _cfg()
    pipe = _pipe(cfg, _weights(cfg))
    cond, pooled = _cond(pipe)
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    cases = [(0.0, _slg()), (CFGW, _slg(layers=())), (CFGW, _slg(layers=(3,))), (CFGW, _slg(layers=(1, 1))),
             (CFGW, _slg(start=0.5, end=0.5)), (CFGW, _slg(scale=float("nan"))), (CFGW, SkipLayerGuidance()),
             (CFGW, (1,))]
    for cfgw, slg in cases:
        with pytest.raises(ValueError):
            pipe.denoise_latents(cond, pooled, num_steps=STEPS, cfg_weight=cfgw, latent_size=LAT, seed=SEEDS, slg=slg)
        with pytest.raises(ValueError):
            pipe.generate_image("", num_steps=STEPS, cfg_weight=cfgw, latent_size=LAT, seed=SEEDS, verbose=False,
                                conditioning=cond, pooled_conditioning=pooled, slg=slg)
    with pytest.raises(ValueError):
        pipe.mmdit(torch.zeros((2, *LAT, 16), dtype=fp16, device=DEV), cond[:2].to(DEV), 1000.0, skip_layers=(5,),
                   skip_batch=1)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0
