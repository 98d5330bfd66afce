"""GPU checks of FLUX.1-dev's guidance embedder (DESIGN.md §12): the MMDiT and the tiny pipelines against the oracle
with per-row guidance (tests/guidance_ref.py), a zero embedder bit-identical to FLUX.1-schnell, the per-step launch
count unchanged, graphs and determinism, the checkpoint loader, LoRA on the embedder and the argument errors."""
import os
import tempfile
from dataclasses import replace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
bf16 = torch.bfloat16
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


def _configs():
    from diffusionkit_b200.config import tiny_flux_config

    schnell = tiny_flux_config()
    return schnell, replace(schnell, guidance_embed=True)


def _weights(cfg, seed=7):
    """generated in fp32 on the host and rounded, so the oracle sees exactly the device's weights"""
    from diffusionkit_b200.weights import init_params, mmdit_param_specs

    return {k: v.to(bf16) for k, v in init_params(mmdit_param_specs(cfg), seed=seed, dtype=torch.float32).items()}


def _vae_weights():
    from diffusionkit_b200.config import VAEDecoderConfig
    from diffusionkit_b200.weights import init_params, vae_decoder_param_specs

    return {k: v.to(bf16) for k, v in init_params(vae_decoder_param_specs(VAEDecoderConfig()), seed=8,
                                                   dtype=torch.float32).items()}


def _pipe(cfg, p16, vp16=None, **kw):
    import diffusionkit_b200 as dk

    return dk.FluxPipeline(w16=True, a16=True, shift=1.0, mmdit_config=cfg,
                           params={k: v.to(DEV) for k, v in p16.items()},
                           vae_params=None if vp16 is None else {k: v.to(DEV) for k, v in vp16.items()},
                           load_decoder=vp16 is not None, **kw)


def _denoise(pipe, cond, pooled, cfgw=0.0, **kw):
    lat, it = pipe.denoise_latents(cond, pooled, num_steps=STEPS, cfg_weight=cfgw, latent_size=LAT, seed=SEEDS, **kw)
    torch.cuda.synchronize()
    return lat.clone(), it


# ------------------------------------------------------------------------------------------------ MMDiT
def _mmdit_vs_oracle(cfg, B, lat, T_txt, guidance):
    """one forward at t = 752 with per-row guidance against GuidanceMMDiTRef -> (got, want, oracle, inputs)"""
    import diffusionkit_b200 as dk
    from tests.guidance_ref import GuidanceMMDiTRef
    from tests.model_checks import psnr, rel_l2
    from tests.oracle_bridge import ref_config

    p16 = _weights(cfg)
    gen = torch.Generator().manual_seed(5)
    latent = torch.randn((B, lat[0], lat[1], 16), generator=gen).to(bf16)
    text = torch.randn((B, T_txt, cfg.token_level_text_embed_dim), generator=gen).to(bf16)
    pooled = torch.randn((B, cfg.pooled_text_embed_dim), generator=gen).to(bf16)
    tval = 752.0
    t = torch.tensor([tval])
    ref = GuidanceMMDiTRef(ref_config(cfg), {k: v.float() for k, v in p16.items()})
    ref.cache_modulation_params(pooled.float(), t, guidance)
    want = ref(latent.float(), text.float(), t.repeat(B))
    m = dk.MMDiT(cfg, {k: v.to(DEV) for k, v in p16.items()})
    del p16
    m.cache_modulation_params(pooled.to(DEV), [tval, 0.0], guidance)
    got = m(latent_image_embeddings=latent.to(DEV), token_level_text_embeddings=text.to(DEV).unsqueeze(2),
            timestep=torch.full((B,), tval)).float().cpu()
    torch.cuda.synchronize()
    del m
    assert got.shape == want.shape and bool(torch.isfinite(got).all())
    r, ps = rel_l2(got, want), psnr(want, got)
    print(f"guidance {guidance}: mmdit rel_l2 {r:.3e}, psnr {ps:.1f} dB")
    assert r <= 2e-2 and ps >= 35.0, f"mmdit rel_l2={r:.3e} psnr={ps:.1f}"
    return got, want, ref, (latent, text, pooled, t)


def test_tiny_mmdit_against_the_oracle(kc):
    from tests.model_checks import rel_l2

    _, dev = _configs()
    g = [1.0, 3.5, 5.0]
    got, want, ref, (latent, text, pooled, t) = _mmdit_vs_oracle(dev, 3, (8, 12), T, g)
    # the check tells guidance values apart: row 1 of the oracle at 3.5 against the same row at 5.0
    ref.cache_modulation_params(pooled.float(), t, [1.0, 5.0, 5.0])
    at5 = ref(latent.float(), text.float(), t.repeat(3))
    sep = rel_l2(want[1], at5[1])
    print(f"oracle 3.5 vs 5.0: rel_l2 {sep:.3e}")
    assert sep >= 10 * 2e-2, sep


def test_fullwidth_truncated_depth_against_the_oracle(kc):
    """FLUX.1-dev at its real width (h = 3072) through 1 double + 1 single block, the C5 text length"""
    from diffusionkit_b200.config import FLUX_DEV

    cfg = replace(FLUX_DEV, depth_multimodal=1, depth_unified=1)
    assert cfg.hidden_size == 3072 and cfg.head_dim == 128 and cfg.guidance_embed
    _mmdit_vs_oracle(cfg, 2, (128, 64), 512, [3.5, 5.0])


# ------------------------------------------------------------------------------------------------ pipelines
def test_zero_embedder_is_bit_identical_to_schnell(kc):
    schnell, dev = _configs()
    p16 = _weights(dev)
    p16["guidance_in.mlp.layers.2.weight"].zero_()
    p16["guidance_in.mlp.layers.2.bias"].zero_()
    plain = {k: v for k, v in p16.items() if not k.startswith("guidance_in.")}
    vp16 = _vae_weights()
    a, b = _pipe(dev, p16, vp16), _pipe(schnell, plain, vp16)
    cond, pooled = a.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
    la, _ = _denoise(a, cond, pooled, guidance=[2.0, 5.0])
    lb, _ = _denoise(b, cond, pooled)
    assert torch.equal(la, lb)
    kw = dict(num_steps=STEPS, latent_size=LAT, seed=SEEDS, verbose=False, conditioning=cond,
              pooled_conditioning=pooled)
    ia, log = a.generate_image("", guidance=4.0, **kw)
    ib, _ = b.generate_image("", **kw)
    assert log["denoising"]["guidance"] == [4.0, 4.0]
    for x, y in zip(ia, ib):
        assert np.array_equal(np.asarray(x), np.asarray(y))


def test_per_step_launch_count_is_unchanged(kc):
    from diffusionkit_b200 import ops

    schnell, dev = _configs()
    p16 = _weights(dev)
    counts = {}
    for name, cfg in (("schnell", schnell), ("dev", dev)):
        pipe = _pipe(cfg, {k: v for k, v in p16.items() if cfg.guidance_embed or not k.startswith("guidance_in.")})
        cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
        _denoise(pipe, cond, pooled)                            # captures the forward's graph
        per_run = []
        for steps in (2, 4):
            n0 = ops.launch_count()
            pipe.denoise_latents(cond, pooled, num_steps=steps, latent_size=LAT, seed=SEEDS)
            torch.cuda.synchronize()
            per_run.append(ops.launch_count() - n0)
        n0 = ops.launch_count()
        pipe.mmdit.cache_modulation_params(pooled.to(DEV), [1000.0, 500.0], [3.5, 3.5] if cfg.guidance_embed else None)
        torch.cuda.synchronize()
        counts[name] = ((per_run[1] - per_run[0]) / 2, per_run[0], ops.launch_count() - n0)
        del pipe
    print(counts)
    (step_s, run_s, cache_s), (step_d, run_d, cache_d) = counts["schnell"], counts["dev"]
    assert step_d == step_s                                     # every denoise step is untouched
    assert cache_d - cache_s == 2                               # the embedder's two GEMMs, once per call
    assert run_d - run_s == 2


def _oracle_latents(cfg, p16, cond, pooled, guidance, solver="euler", cfgw=0.0):
    """the oracle pipeline one image at a time (CFG doubles it), image i at guidance[i] -> process_out latents"""
    from oracle import sampler_ref as sr
    from tests import solver_ref
    from tests.guidance_ref import GuidanceMMDiTRef
    from tests.oracle_bridge import ref_config

    sample = {"euler": sr.sample_euler, "dpmpp_2m": solver_ref.sample_dpmpp_2m}[solver]
    sampler = sr.FluxSamplerRef(1.0)
    sig = sr.get_sigmas(sampler, STEPS)
    H, W = LAT
    n = len(SEEDS)
    reps = 2 if cfgw > 0 else 1
    outs = []
    for i, s in enumerate(SEEDS):
        ref = GuidanceMMDiTRef(ref_config(cfg), {k: v.float() for k, v in p16.items()})
        idx = [i + k * n for k in range(reps)]
        x0 = sampler.noise_scaling(float(sig[0]), sr.get_noise(s, H, W), sr.get_empty_latent(H, W))
        x = sample(lambda xin, c, t: ref(xin, c, t),
                   lambda p, ts, g=guidance[i]: ref.cache_modulation_params(p, ts, [g] * reps),
                   x0, sig, cond[idx].float(), pooled[idx].float(), cfgw, bf16)
        outs.append(sr.process_out(x, "flux"))
    return torch.cat(outs)


@pytest.mark.parametrize("solver, cfgw, guidance", [("euler", 0.0, 3.5), ("dpmpp_2m", 0.0, 3.5),
                                                     ("euler", 2.0, [2.0, 5.0])])
def test_tiny_pipeline_against_the_oracle(kc, solver, cfgw, guidance):
    from oracle.vae_ref import VAEDecoderRef, decode_latents_to_image
    from tests.model_checks import psnr, rel_l2

    _, dev = _configs()
    p16, vp16 = _weights(dev), _vae_weights()
    pipe = _pipe(dev, p16, vp16)
    reps = 2 if cfgw > 0 else 1
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
    if reps == 2:                                               # [positive x B | negative x B]
        cond2, pooled2 = pipe.synthetic_text_embeddings(n_images=len(SEEDS), seed=99, text_len=T)
        cond, pooled = torch.cat([cond, cond2]), torch.cat([pooled, pooled2])
    latent, iter_time = _denoise(pipe, cond, pooled, cfgw=cfgw, solver=solver, guidance=guidance)
    assert latent.shape == (len(SEEDS), *LAT, 16) and len(iter_time) == STEPS
    per_image = guidance if isinstance(guidance, list) else [guidance] * len(SEEDS)
    want = _oracle_latents(dev, p16, cond, pooled, per_image, solver, cfgw)
    r = rel_l2(latent, want)
    img_want = decode_latents_to_image(VAEDecoderRef({k: v.float() for k, v in vp16.items()}), want.to(bf16).float())
    ps = psnr(img_want, pipe.decode_latents_to_image(latent))
    print(f"{solver} cfg {cfgw} guidance {guidance}: final latent rel_l2 {r:.3e}, decoded psnr {ps:.1f} dB")
    assert r <= 5e-2, f"final latent rel_l2 {r:.3e}"
    assert ps >= 30.0, f"decoded RGB psnr {ps:.1f}"
    # the default (None) is 3.5
    if guidance == 3.5:
        default, _ = _denoise(pipe, cond, pooled, cfgw=cfgw, solver=solver)
        assert torch.equal(default, latent)


def test_graphs_and_determinism(kc, monkeypatch):
    _, dev = _configs()
    p16 = _weights(dev)
    runs = {}
    for graphs in ("1", "0"):
        monkeypatch.setenv("DK_CUDA_GRAPHS", graphs)
        pipe = _pipe(dev, p16)
        assert pipe.mmdit.use_cuda_graphs == (graphs == "1")
        cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
        a, _ = _denoise(pipe, cond, pooled, guidance=2.0)
        b, _ = _denoise(pipe, cond, pooled, guidance=[4.0, 6.0])
        a2, _ = _denoise(pipe, cond, pooled, guidance=2.0)
        b2, _ = _denoise(pipe, cond, pooled, guidance=[4.0, 6.0])
        assert torch.equal(a, a2) and torch.equal(b, b2), graphs
        assert not torch.equal(a, b)
        del pipe
        for g, want in ((2.0, a), ([4.0, 6.0], b)):
            fresh = _pipe(dev, p16)
            got, _ = _denoise(fresh, cond, pooled, guidance=g)
            assert torch.equal(got, want), (graphs, g)
            del fresh
        runs[graphs] = (a, b)
    assert torch.equal(runs["1"][0], runs["0"][0]) and torch.equal(runs["1"][1], runs["0"][1])


def test_local_checkpoint_with_the_embedder(kc):
    from safetensors.torch import save_file

    from tests.test_guidance_cpu import dev_upstream

    _, dev = _configs()
    p16 = _weights(dev)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "flux1-dev.safetensors")
        save_file({k: v.contiguous() for k, v in dev_upstream(p16, dev).items()}, path)
        a = _pipe_ckpt(dev, path)
    b = _pipe(dev, p16)
    cond, pooled = a.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
    la, _ = _denoise(a, cond, pooled, guidance=[3.0, 4.5])
    lb, _ = _denoise(b, cond, pooled, guidance=[3.0, 4.5])
    assert torch.equal(la, lb)


def _pipe_ckpt(cfg, path):
    import diffusionkit_b200 as dk

    return dk.FluxPipeline(w16=True, a16=True, shift=1.0, mmdit_config=cfg, local_ckpt=path, load_decoder=False)


def test_lora_on_the_embedder(kc):
    from tests.lora_fixtures import make_factors, peft_dict

    _, dev = _configs()
    p16 = _weights(dev)
    pipe = _pipe(dev, p16)
    m = pipe.mmdit
    slots = m.lora_weight_slots()
    assert "guidance_in.mlp.layers.0.weight" in slots and "guidance_in.mlp.layers.2.weight" in slots
    g0, g2 = m.g0[0].clone(), m.g2[0].clone()
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
    base, _ = _denoise(pipe, cond, pooled)
    h, f = dev.hidden_size, dev.frequency_embed_dim
    factors = make_factors({"guidance_in.in_layer": (h, f), "guidance_in.out_layer": (h, h)}, rank=4, seed=6,
                           gain=0.5)
    name = pipe.load_lora_weights(peft_dict(factors, "diffusion_model."), scale=1.0, adapter_name="g")
    lora = pipe._loras[name][0]
    for attr, ref_name, orig in (("g0", "guidance_in.mlp.layers.0.weight", g0),
                                 ("g2", "guidance_in.mlp.layers.2.weight", g2)):
        up, down = lora.targets[ref_name]
        want = orig.float().cpu() + up @ down
        got = getattr(m, attr)[0].float().cpu()
        assert (got - want).abs().max() <= 2 ** -7 * want.abs().max(), attr    # one bf16 rounding
        assert not torch.equal(getattr(m, attr)[0], orig)
    merged, _ = _denoise(pipe, cond, pooled)
    assert not torch.equal(merged, base)
    pipe.unload_lora_weights()
    assert torch.equal(m.g0[0], g0) and torch.equal(m.g2[0], g2)
    again, _ = _denoise(pipe, cond, pooled)
    assert torch.equal(again, base)


def test_errors_launch_nothing(kc):
    from diffusionkit_b200 import ops

    schnell, dev = _configs()
    p16 = _weights(dev)
    a = _pipe(dev, p16)
    b = _pipe(schnell, {k: v for k, v in p16.items() if not k.startswith("guidance_in.")})
    cond, pooled = a.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
    torch.cuda.synchronize()
    n0 = ops.launch_count()
    cases = [(b, dict(guidance=3.5)), (b, dict(guidance=[3.5, 3.5])), (a, dict(guidance=[3.5])),
             (a, dict(guidance=[3.5, 4.0, 5.0])), (a, dict(guidance=float("nan"))), (a, dict(guidance=[1.0, float("inf")]))]
    for pipe, kw in cases:
        with pytest.raises(ValueError):
            pipe.denoise_latents(cond, pooled, num_steps=STEPS, latent_size=LAT, seed=SEEDS, **kw)
        with pytest.raises(ValueError):
            pipe.generate_image("", num_steps=STEPS, latent_size=LAT, seed=SEEDS, verbose=False, conditioning=cond,
                                pooled_conditioning=pooled, **kw)
    with pytest.raises(ValueError):
        a.mmdit.cache_modulation_params(pooled.to(DEV), [1000.0])
    with pytest.raises(ValueError):
        b.mmdit.cache_modulation_params(pooled.to(DEV), [1000.0], [3.5, 3.5])
    torch.cuda.synchronize()
    assert ops.launch_count() == n0
