"""-m gpu: the launch census (tests/launch_parity.py) over every shipped model at its real width and truncated depth,
eager, on synthetic weights: each kernel launch against the fp32 reference of that launch, plus the bytes around its
output.  The last test checks that the runs together reached every launching op and the layouts this census exists
for, and prints the census table (one row per op and signature; run with -s to see it)."""
from dataclasses import replace

import pytest
import torch

from tests import launch_parity as lp

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
bf16, fp16 = torch.bfloat16, torch.float16


@pytest.fixture(scope="session")
def the_census():
    return lp.Census()


def _fullwidth(cfg, depth_mm, depth_uni=0, **over):
    return replace(cfg, depth_multimodal=depth_mm, depth_unified=depth_uni, hidden_size_override=cfg.hidden_size,
                   **over)


def _mmdit(cfg, dtype, B, lat, T, guidance=None, fp8=False, slg_layers=(), skip_batch=0, seed=7):
    import diffusionkit_b200 as dk
    from diffusionkit_b200.weights import init_params, mmdit_param_specs

    m = dk.MMDiT(cfg, init_params(mmdit_param_specs(cfg), seed=seed, dtype=dtype, device=DEV))
    m.use_cuda_graphs = False
    if fp8:
        m.set_fp8(True)
    g = torch.Generator(device=DEV).manual_seed(5)
    latent = torch.randn((B, lat[0], lat[1], 16), generator=g, device=DEV).to(dtype)
    text = torch.randn((B, T, cfg.token_level_text_embed_dim), generator=g, device=DEV).to(dtype)
    pooled = torch.randn((B, cfg.pooled_text_embed_dim), generator=g, device=DEV).to(dtype)
    m.cache_modulation_params(pooled, [752.0, 500.0], guidance, skip_batch=skip_batch)
    m(latent, text, timestep=752.0, skip_layers=slg_layers, skip_batch=skip_batch)
    torch.cuda.synchronize()


def run_flux_schnell():
    from diffusionkit_b200.config import FLUX_SCHNELL

    cfg = _fullwidth(FLUX_SCHNELL, 1, 1)
    _mmdit(cfg, bf16, 1, (128, 128), 256)
    _mmdit(cfg, bf16, 2, (128, 128), 512)


def run_flux_dev():
    from diffusionkit_b200.config import FLUX_DEV

    _mmdit(_fullwidth(FLUX_DEV, 1, 1), bf16, 2, (128, 128), 512, guidance=[3.5, 5.0])


def run_sd3_medium():
    from diffusionkit_b200.config import SD3_2b

    _mmdit(_fullwidth(SD3_2b, 2), fp16, 2, (128, 128), 589)


def run_sd35_medium():
    from diffusionkit_b200.config import SD35_MEDIUM

    cfg = _fullwidth(SD35_MEDIUM, 3, x_block_self_attn_layers=(0, 1))
    _mmdit(cfg, fp16, 2, (128, 128), 589)
    _mmdit(cfg, fp16, 3, (128, 128), 589, slg_layers=(1,), skip_batch=1)


def run_sd35_large():
    from diffusionkit_b200.config import SD3_8b

    cfg = _fullwidth(SD3_8b, 2)
    assert cfg.hidden_size == 2432 and cfg.num_heads == 38
    _mmdit(cfg, cfg.dtype, 2, (128, 128), 589)


def run_fp8():
    from diffusionkit_b200.config import FLUX_SCHNELL, SD3_8b

    _mmdit(_fullwidth(FLUX_SCHNELL, 1, 1), bf16, 1, (128, 128), 256, fp8=True)
    cfg = _fullwidth(SD3_8b, 2)
    _mmdit(cfg, cfg.dtype, 2, (128, 128), 589, fp8=True)


def run_vae_decoder():
    import diffusionkit_b200 as dk
    from diffusionkit_b200.config import VAEDecoderConfig
    from diffusionkit_b200.weights import init_params, vae_decoder_param_specs

    dec = dk.VAEDecoder(init_params(vae_decoder_param_specs(VAEDecoderConfig()), seed=8, dtype=bf16, device=DEV))
    dec.use_cuda_graphs = False
    g = torch.Generator(device=DEV).manual_seed(2)
    for lat in (64, 128):
        dec(torch.randn((1, lat, lat, 16), generator=g, device=DEV).to(bf16))
        torch.cuda.synchronize()


def run_vae_encoder():
    import diffusionkit_b200 as dk
    from diffusionkit_b200.config import VAEEncoderConfig
    from diffusionkit_b200.weights import init_params, vae_encoder_param_specs

    enc = dk.VAEEncoder(init_params(vae_encoder_param_specs(VAEEncoderConfig()), seed=9, dtype=bf16, device=DEV))
    g = torch.Generator(device=DEV).manual_seed(3)
    enc(torch.randint(0, 256, (1, 512, 512, 3), generator=g, device=DEV, dtype=torch.uint8))
    torch.cuda.synchronize()


def run_text_encoders():
    from diffusionkit_b200.config import CLIP_G, CLIP_L, T5EncoderConfig
    from diffusionkit_b200.text_encoders import CLIPTextModel, SD3T5Encoder, clip_param_specs, t5_param_specs
    from diffusionkit_b200.weights import init_params

    g = torch.Generator().manual_seed(9)
    for cfg in (CLIP_L, CLIP_G):
        cfg = replace(cfg, num_layers=2)
        m = CLIPTextModel(init_params(clip_param_specs(cfg), seed=41, dtype=fp16, device=DEV), cfg)
        tokens = torch.randint(1, 49406, (2, 77), generator=g)
        tokens[:, 30] = 49407
        m(tokens)
        del m
    cfg = replace(T5EncoderConfig(), num_layers=2)
    assert cfg.num_heads == 64 and cfg.d_ff == 10240
    t5 = SD3T5Encoder(init_params(t5_param_specs(cfg), seed=42, dtype=bf16, device=DEV), cfg)
    t5(torch.randint(0, 32128, (2, 512), generator=g))
    torch.cuda.synchronize()


def _tiny_pipe(kind):
    import diffusionkit_b200 as dk
    from diffusionkit_b200.config import VAEDecoderConfig, tiny_flux_config, tiny_sd35_medium_config
    from diffusionkit_b200.weights import init_params, mmdit_param_specs, vae_decoder_param_specs

    if kind == "flux":
        cfg, dt, cls, mv = tiny_flux_config(), bf16, dk.FluxPipeline, "argmaxinc/mlx-FLUX.1-schnell"
    else:
        cfg, dt, cls, mv = (tiny_sd35_medium_config(), fp16, dk.DiffusionPipeline,
                            "argmaxinc/mlx-stable-diffusion-3-medium")
    vp = init_params(vae_decoder_param_specs(VAEDecoderConfig()), seed=8, dtype=dt, device=DEV) if kind != "flux" else None
    pipe = cls(w16=True, a16=True, shift=3.0, model_version=mv, mmdit_config=cfg,
               params=init_params(mmdit_param_specs(cfg), seed=7, dtype=dt, device=DEV), vae_params=vp,
               load_decoder=vp is not None)
    pipe.mmdit.use_cuda_graphs = False
    if vp is not None:
        pipe.decoder.use_cuda_graphs = False
    return pipe


def run_pipelines():
    from diffusionkit_b200.sampler import SkipLayerGuidance

    flux = _tiny_pipe("flux")
    flux.set_step_cache(float("inf"))
    cond, pooled = flux.synthetic_text_embeddings(n_images=1, text_len=16)
    for solver in ("euler", "heun", "dpmpp_2m"):
        flux.denoise_latents(cond, pooled, num_steps=3, cfg_weight=0.0, latent_size=(128, 128), seed=[11],
                             solver=solver)
    sd = _tiny_pipe("sd35")
    sd.set_step_cache(float("inf"))
    cond, pooled = sd.synthetic_text_embeddings(n_images=2, text_len=24)
    slg = SkipLayerGuidance(scale=2.5, layers=(1,), start=0.0, end=1.0)
    for solver in ("euler", "heun", "dpmpp_2m"):
        lat, _ = sd.denoise_latents(cond, pooled, num_steps=3, cfg_weight=5.0, latent_size=(8, 12), seed=[11, 12],
                                    solver=solver, slg=slg)
    sd.decode_latents_to_image(lat)
    torch.cuda.synchronize()


RUNS = {"flux_schnell": run_flux_schnell, "flux_dev": run_flux_dev, "sd3_medium": run_sd3_medium,
        "sd35_medium": run_sd35_medium, "sd35_large": run_sd35_large, "fp8": run_fp8, "vae_decoder": run_vae_decoder,
        "vae_encoder": run_vae_encoder, "text_encoders": run_text_encoders, "pipelines": run_pipelines}


@pytest.mark.parametrize("run", list(RUNS))
def test_launch_parity(cuda, the_census, run):
    the_census.run = run
    n0 = len(the_census.records)
    with lp.census(the_census):
        RUNS[run]()
    assert len(the_census.records) > n0, f"{run}: no launch was checked"
    torch.cuda.empty_cache()


def _hits(census, run=None, op="gemm", **pred):
    return [r for r in census.records if r["op"] == op and (run is None or r["run"] == run)
            and all(f(r["info"]) for f in pred.values())]


def test_census_coverage(cuda, the_census):
    """the runs above checked every launching op but NOT_REACHED and the layouts the census exists for"""
    print("\n" + the_census.table())
    done = {r["run"] for r in the_census.records}
    assert done == set(RUNS), f"census runs missing (run the whole file): {sorted(set(RUNS) - done)}"
    seen = {r["op"] for r in the_census.records}
    missing = [n for n in lp.launching_ops() if n not in seen and n not in lp.NOT_REACHED]
    assert not missing, f"launching ops no run checked: {missing}"
    # SD3.5-large: the fused QK-norm GEMM (N = 3 * 2432) whose q | k boundary falls inside a 256-wide n-block, and a
    # gate + residual GEMM ending in a half-empty 256-wide tile
    assert _hits(the_census, "sd35_large", qk=lambda i: i.get("qk_hd") is not None and (i["N"] // 3) % 256 != 0)
    assert _hits(the_census, "sd35_large", g=lambda i: "gate" in i["epi"] and "res" in i["epi"] and i["n256"] == 128)
    # the VAE's P V product: W given N-major with K = S >= 4096
    assert _hits(the_census, "vae_decoder", nm=lambda i: "n_major" in i["epi"] and i["K"] >= 4096)
    assert _hits(the_census, "vae_decoder", nm=lambda i: "n_major" in i["epi"] and i["K"] == 16384)
    # a gate read through the modulation table's row stride, and a residual broadcast to every batch
    assert _hits(the_census, g=lambda i: i["gate_ld"] is not None and i["gate_ld"] != i["N"])
    assert _hits(the_census, r=lambda i: i["res_batch_rows"] == 0)
    # T5-XXL's 64-head attention with the relative bias at L = 512
    assert _hits(the_census, "text_encoders", op="attention_small",
                 t=lambda i: i["heads"] == 64 and i["S"] == 512 and i["rel_bias"])
    # FP8 GEMMs on the FLUX single-block concat buffer (K = 5h)
    assert _hits(the_census, "fp8", f=lambda i: "fp8" in i["epi"] and i["K"] == 5 * 3072)
