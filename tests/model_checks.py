"""GPU checks of the assembled models (MMDiT forward, denoise loop, VAE decode, pipeline API) against the fp32 CPU
oracle on the same synthetic weights and inputs.

Tolerances (stated per SURVEY.md §8c): 16-bit kernels vs the fp32 oracle —
  MMDiT forward     rel-L2 <= 2e-2 and PSNR >= 35 dB (the reference's own converter gate, tests/torch2coreml/test_mmdit.py:27)
  final latent      rel-L2 <= 5e-2
  decoded RGB       PSNR >= 30 dB (4-step FLUX), >= 20 dB (reference e2e floor) for CFG runs
"""
import math
import os
from dataclasses import replace

import numpy as np
import torch

import diffusionkit_b200 as dk
from diffusionkit_b200 import ops
from diffusionkit_b200.config import (VAEDecoderConfig, VAEEncoderConfig, tiny_flux_config, tiny_sd3_config,
                                      tiny_sd35_config)
from diffusionkit_b200.weights import (init_params, mmdit_param_specs, vae_decoder_param_specs,
                                       vae_encoder_param_specs)
from oracle import sampler_ref as sr
from oracle.mmdit_ref import MMDiTRef
from oracle.vae_ref import (VAEDecoderRef, VAEEncoderRef, decode_latents_to_image, encode_image_to_latents,
                            read_image_array, to_uint8)
from tests.oracle_bridge import ref_config

DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def psnr(ref, got):
    return sr.compute_psnr(ref.float().cpu().numpy(), got.float().cpu().numpy())


def _mmdit_case(cfg, dtype, B, lat, T, seed=7, from_golden=None):
    p32 = init_params(mmdit_param_specs(cfg), seed=seed, dtype=torch.float32)
    p16 = {k: v.to(dtype) for k, v in p32.items()}
    # the oracle sees the same (16-bit-rounded) weights as the GPU
    ref = MMDiTRef(ref_config(cfg), {k: v.float() for k, v in p16.items()})
    if from_golden is not None:
        g = np.load(os.path.join(GOLD, from_golden))
        latent, text, pooled = [torch.from_numpy(g[k]) for k in ("latent", "text", "pooled")]
        tval = float(g["timestep"][0])
    else:
        gen = torch.Generator().manual_seed(5)
        latent = torch.randn((B, lat[0], lat[1], 16), generator=gen)
        text = torch.randn((B, T, cfg.token_level_text_embed_dim), generator=gen)
        pooled = torch.randn((B, cfg.pooled_text_embed_dim), generator=gen)
        tval = 752.0
    latent, text, pooled = [t.to(dtype) for t in (latent, text, pooled)]
    t = torch.tensor([tval])
    ref.cache_modulation_params(pooled.float(), t)
    want = ref(latent.float(), text.float(), t.repeat(latent.shape[0]))
    m = dk.MMDiT(cfg, {k: v.to(DEV) for k, v in p16.items()})
    m.cache_modulation_params(pooled.to(DEV), [tval, 0.0])
    got = m(latent_image_embeddings=latent.to(DEV), token_level_text_embeddings=text.to(DEV).unsqueeze(2),
            timestep=torch.full((latent.shape[0],), tval))
    torch.cuda.synchronize()
    assert got.shape == want.shape and bool(torch.isfinite(got.float()).all())
    r, ps = rel_l2(got, want), psnr(want, got)
    assert r <= 2e-2 and ps >= 35.0, f"mmdit rel_l2={r:.3e} psnr={ps:.1f}"
    # modulation table sanity: every block's rows agree with the oracle
    return {"rel_l2": r, "psnr": ps}


def check_mmdit_flux_tiny():
    return _mmdit_case(tiny_flux_config(), torch.bfloat16, 2, (8, 12), 16, from_golden="tiny_flux_mmdit.npz")


def check_mmdit_sd3_tiny():
    return _mmdit_case(tiny_sd3_config(), torch.float16, 2, (8, 8), 24, from_golden="tiny_sd3_mmdit.npz")


def check_mmdit_flux_ragged():
    """sequence lengths that are not tile multiples: N = 14*18 = 252 image tokens + 77 text tokens, head dim 128"""
    return _mmdit_case(tiny_flux_config(hidden=256, heads=2, depth_mm=2, depth_uni=3), torch.bfloat16, 3, (28, 36), 77)


def check_mmdit_sd3_d64_long():
    return _mmdit_case(tiny_sd3_config(hidden=192, heads=3, depth_mm=3), torch.float16, 2, (32, 40), 154)


def check_mmdit_sd35_tiny():
    """SD3.5 shape of the block: learned positional embedding + QK-RMSNorm, fp16 activations, bf16 sinusoid"""
    return _mmdit_case(tiny_sd35_config(), torch.float16, 2, (8, 12), 24)


def _vae_case(dtype, B, lat, tol_psnr):
    vp32 = init_params(vae_decoder_param_specs(VAEDecoderConfig()), seed=8, dtype=torch.float32)
    vp16 = {k: v.to(dtype) for k, v in vp32.items()}
    gen = torch.Generator().manual_seed(4)
    z = torch.randn((B, lat[0], lat[1], 16), generator=gen).to(dtype)
    want = decode_latents_to_image(VAEDecoderRef({k: v.float() for k, v in vp16.items()}), z.float())
    dec = dk.VAEDecoder({k: v.to(DEV) for k, v in vp16.items()})
    raw = dec(z.to(DEV))
    Bo, Ho, Wo, _ = raw.shape
    padded = raw.as_strided((Bo, Ho, Wo, raw.stride(2)), (raw.stride(0), raw.stride(1), raw.stride(2), 1))
    f, u8 = ops.image_post(padded)
    torch.cuda.synchronize()
    assert f.shape == want.shape
    ps = psnr(want, f)
    du8 = (u8.cpu().int() - to_uint8(want).int()).abs()
    assert ps >= tol_psnr, f"vae psnr {ps:.1f}"
    return {"psnr": ps, "u8_max_diff": int(du8.max()), "u8_mean_diff": float(du8.float().mean())}


def check_vae_decode_tiny():
    return _vae_case(torch.bfloat16, 1, (8, 8), 30.0)


def check_vae_decode_batch_fp16():
    return _vae_case(torch.float16, 2, (8, 12), 40.0)


def _test_image(H, W, seed=5):
    """a smooth synthetic RGB picture (low-frequency sinusoids + a little noise), uint8 (H, W, 3)"""
    rng = np.random.RandomState(seed)
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    chans = [0.5 + 0.4 * np.sin(2 * np.pi * (a * xx + b * yy) + c) for a, b, c in rng.uniform(0.5, 3.0, (3, 3))]
    img = np.stack(chans, axis=-1) + 0.03 * rng.randn(H, W, 3)
    return (np.clip(img, 0, 1) * 255).astype(np.uint8)


def _vae_encode_case(dtype, B, size, tol):
    ep32 = init_params(vae_encoder_param_specs(VAEEncoderConfig()), seed=9, dtype=torch.float32)
    ep16 = {k: v.to(dtype) for k, v in ep32.items()}
    imgs = torch.from_numpy(np.stack([_test_image(size[0], size[1], seed=5 + i) for i in range(B)]))
    want = torch.cat([VAEEncoderRef({k: v.float() for k, v in ep16.items()})(read_image_array(im)) for im in imgs])
    enc = dk.VAEEncoder({k: v.to(DEV) for k, v in ep16.items()})
    got = enc(imgs.to(DEV))
    torch.cuda.synchronize()
    assert got.shape == want.shape == (B, size[0] // 8, size[1] // 8, 32)
    r = rel_l2(got, want)
    assert r <= tol, f"vae encoder hidden rel_l2 {r:.3e}"
    again = enc(imgs.to(DEV))
    assert torch.equal(got, again), "encoder is not deterministic"
    return {"hidden_rel_l2": r}


def check_vae_encode_tiny():
    return _vae_encode_case(torch.bfloat16, 1, (64, 64), 3e-2)


def check_vae_encode_batch_fp16():
    return _vae_encode_case(torch.float16, 2, (64, 128), 5e-3)


def check_pipeline_img2img():
    """image -> VAE encoder -> posterior sample -> process_in -> trimmed schedule -> Euler loop, vs the oracle
    (reference denoise_latents :270-285 + encode_image_to_latents :586-594); then generate_image on a PNG file whose
    size is not a multiple of 64 (read_image's LANCZOS resize rule)."""
    import tempfile

    from PIL import Image

    cfg, dtype, steps, shift, T = tiny_flux_config(), torch.bfloat16, 4, 1.0, 16
    p16 = {k: v.to(dtype) for k, v in init_params(mmdit_param_specs(cfg), seed=7, dtype=torch.float32).items()}
    vp16 = {k: v.to(dtype) for k, v in init_params(vae_decoder_param_specs(VAEDecoderConfig()), seed=8,
                                                    dtype=torch.float32).items()}
    ep16 = {k: v.to(dtype) for k, v in init_params(vae_encoder_param_specs(VAEEncoderConfig()), seed=9,
                                                    dtype=torch.float32).items()}
    pipe = dk.FluxPipeline(w16=True, a16=True, shift=shift, mmdit_config=cfg,
                           params={k: v.to(DEV) for k, v in p16.items()},
                           vae_params={k: v.to(DEV) for k, v in vp16.items()},
                           vae_encoder_params={k: v.to(DEV) for k, v in ep16.items()})
    assert not hasattr(pipe, "encoder")                      # built on first use
    img = _test_image(64, 128)
    H, W = 8, 16
    seeds, denoise = [11, 12], 0.5
    n = len(seeds)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=n, text_len=T)
    latent, iter_time = pipe.denoise_latents(cond, pooled, num_steps=steps, cfg_weight=0.0, latent_size=(2, 2),
                                             seed=seeds, image_path=img, denoise=denoise)
    assert latent.shape == (n, H, W, 16) and len(iter_time) == steps - int(steps * (1 - denoise))
    sampler = sr.FluxSamplerRef(shift)
    sig = sr.get_sigmas(sampler, steps)[int(steps * (1 - denoise)):]
    enc_ref = VAEEncoderRef({k: v.float() for k, v in ep16.items()})
    image = read_image_array(torch.from_numpy(img))
    outs, zs = [], []
    for i, s in enumerate(seeds):
        ref = MMDiTRef(ref_config(cfg), {k: v.float() for k, v in p16.items()})
        noise = sr.get_noise(s, H, W)
        z = encode_image_to_latents(enc_ref, image, noise)
        zs.append(z)
        x_T = (z - 0.1159) * 0.3611                                        # FluxLatentFormat.process_in
        x0 = sampler.noise_scaling(float(sig[0]), noise, x_T)
        x = sr.sample_euler(lambda xin, c, t: ref(xin, c, t), ref.cache_modulation_params, x0, sig,
                            cond[[i]].float(), pooled[[i]].float(), 0.0, dtype)
        outs.append(sr.process_out(x, "flux"))
    r = rel_l2(latent, torch.cat(outs))
    assert r <= 5e-2, f"img2img final latent rel_l2 {r:.3e}"
    z_got = pipe.encode_image_to_latents(img, seeds[0])
    rz = rel_l2(z_got, zs[0])
    assert rz <= 3e-2, f"encode_image_to_latents rel_l2 {rz:.3e}"
    # denoise = 1.0 with an image still starts from the image-derived x_T (sigma0 = 1 -> pure noise): equals txt2img
    full, _ = pipe.denoise_latents(cond, pooled, num_steps=steps, seed=seeds, image_path=img, denoise=1.0)
    plain, _ = pipe.denoise_latents(cond, pooled, num_steps=steps, seed=seeds, latent_size=(H, W))
    assert torch.equal(full, plain)
    # file path + resize rule: 100 x 150 -> 64 x 128
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "in.png")
        Image.fromarray(_test_image(100, 150)).save(path)
        ri = pipe.read_image(path)
        assert tuple(ri.shape) == (1, 64, 128, 3) and float(ri.min()) >= -1.0 and float(ri.max()) <= 1.0
        out, log = pipe.generate_image("", num_steps=steps, seed=seeds[0], verbose=False, conditioning=cond[[0]],
                                       pooled_conditioning=pooled[[0]], image_path=path, denoise=0.75)
    assert out.size == (128, 64) and len(log["denoising"]["iter_time"]) == 3
    return {"latent_rel_l2": r, "posterior_rel_l2": rz}


def _pipeline_case(kind):
    """Full denoise loop + decode through the public API vs the oracle loop (same seeds, steps, shift, cfg)."""
    vp32 = init_params(vae_decoder_param_specs(VAEDecoderConfig()), seed=8, dtype=torch.float32)
    if kind == "flux":
        cfg, dtype, steps, cfgw, shift, T, fmt = tiny_flux_config(), torch.bfloat16, 4, 0.0, 1.0, 16, "flux"
    else:
        cfg, dtype, steps, cfgw, shift, T, fmt = tiny_sd3_config(), torch.float16, 6, 5.0, 3.0, 24, "sd3"
    p32 = init_params(mmdit_param_specs(cfg), seed=7, dtype=torch.float32)
    p16 = {k: v.to(dtype) for k, v in p32.items()}
    vp16 = {k: v.to(dtype) for k, v in vp32.items()}
    Pipe = dk.FluxPipeline if kind == "flux" else dk.DiffusionPipeline
    mv = "argmaxinc/mlx-FLUX.1-schnell" if kind == "flux" else "argmaxinc/mlx-stable-diffusion-3-medium"
    pipe = Pipe(w16=True, a16=True, shift=shift, model_version=mv, mmdit_config=cfg,
                params={k: v.to(DEV) for k, v in p16.items()}, vae_params={k: v.to(DEV) for k, v in vp16.items()})
    seeds = [11, 12]
    n = len(seeds)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=n, text_len=T)
    H, W = 8, 12
    latent, iter_time = pipe.denoise_latents(cond, pooled, num_steps=steps, cfg_weight=cfgw, latent_size=(H, W),
                                             seed=seeds)
    assert latent.shape == (n, H, W, 16) and latent.dtype == torch.float32 and len(iter_time) == steps
    # oracle loop, one image at a time exactly like the reference (batch 1, CFG doubles it)
    sampler = sr.FluxSamplerRef(shift) if kind == "flux" else sr.ModelSamplingDiscreteFlowRef(shift)
    sig = sr.get_sigmas(sampler, steps)
    outs = []
    reps = 2 if cfgw > 0 else 1
    for i, s in enumerate(seeds):
        ref = MMDiTRef(ref_config(cfg), {k: v.float() for k, v in p16.items()})
        idx = [i + k * n for k in range(reps)]
        c_i, p_i = cond[idx].float(), pooled[idx].float()
        x0 = sampler.noise_scaling(float(sig[0]), sr.get_noise(s, H, W), sr.get_empty_latent(H, W))
        x = sr.sample_euler(lambda xin, c, t: ref(xin, c, t), ref.cache_modulation_params, x0, sig, c_i, p_i, cfgw, dtype)
        outs.append(sr.process_out(x, fmt))
    want = torch.cat(outs)
    r = rel_l2(latent, want)
    assert r <= 5e-2, f"{kind} final latent rel_l2 {r:.3e}"
    img_want = decode_latents_to_image(VAEDecoderRef({k: v.float() for k, v in vp16.items()}), want.to(dtype).float())
    img_got = pipe.decode_latents_to_image(latent)
    ps = psnr(img_want, img_got)
    assert ps >= (30.0 if kind == "flux" else 20.0), f"{kind} decoded RGB psnr {ps:.1f}"
    # public generate_image: returns (PIL image, log) for a scalar seed, list for a list of seeds
    c1, p1 = cond[[0] + ([n] if reps == 2 else [])], pooled[[0] + ([n] if reps == 2 else [])]
    image, log = pipe.generate_image("", num_steps=steps, cfg_weight=cfgw, latent_size=(H, W), seed=seeds[0],
                                     verbose=False, conditioning=c1, pooled_conditioning=p1)
    assert image.size == (W * 8, H * 8)
    for k in ("text_encoding", "denoising", "decoding", "peak_memory", "total_time"):
        assert k in log
    assert len(log["denoising"]["iter_time"]) == steps
    u8 = np.asarray(image)
    want_u8 = to_uint8(img_want[0]).numpy()
    return {"latent_rel_l2": r, "rgb_psnr": ps, "u8_mean_abs_diff": float(np.abs(u8.astype(int) - want_u8.astype(int)).mean())}


def check_pipeline_flux_tiny():
    return _pipeline_case("flux")


def check_pipeline_sd3_cfg_tiny():
    return _pipeline_case("sd3")


def check_pipeline_errors():
    cfg = tiny_flux_config()
    pipe = dk.FluxPipeline(w16=True, a16=True, mmdit_config=cfg, load_decoder=False)
    cond, pooled = pipe.synthetic_text_embeddings(text_len=8)
    try:
        pipe.generate_image("x", latent_size=(7, 8), conditioning=cond, pooled_conditioning=pooled)
        raise RuntimeError("odd latent size accepted")
    except AssertionError:
        pass
    try:
        pipe.encode_text("a prompt")
        raise RuntimeError("encode_text without attached encoders should refuse")
    except dk.DkError:
        pass
    try:
        pipe.mmdit(torch.zeros(1, 8, 16, dtype=torch.bfloat16, device=DEV), cond.to(DEV), 0.0)
        raise RuntimeError("rank-3 latent accepted")
    except ValueError:
        pass
    return {}


def check_pipeline_local_ckpt():
    """`local_ckpt=` (upstream BFL-layout .safetensors) produces the same latents as passing the parameter tree"""
    import tempfile

    from safetensors.torch import save_file

    from tests.test_model_io_cpu import _flux_upstream, _vae_upstream

    cfg = tiny_flux_config()
    p32 = init_params(mmdit_param_specs(cfg), seed=7, dtype=torch.float32)
    v32 = init_params(vae_decoder_param_specs(VAEDecoderConfig()), seed=8, dtype=torch.float32)
    p16 = {k: v.to(torch.bfloat16) for k, v in p32.items()}
    v16 = {k: v.to(torch.bfloat16) for k, v in v32.items()}
    with tempfile.TemporaryDirectory() as d:
        mm, va = os.path.join(d, "flux.safetensors"), os.path.join(d, "ae.safetensors")
        save_file({k: v.contiguous() for k, v in _flux_upstream(p16, cfg).items()}, mm)
        save_file({k: v.contiguous() for k, v in _vae_upstream(v16, prefix="decoder.").items()}, va)
        a = dk.FluxPipeline(w16=True, a16=True, mmdit_config=cfg, local_ckpt={"mmdit": mm, "vae": va})
    b = dk.FluxPipeline(w16=True, a16=True, mmdit_config=cfg, params={k: v.to(DEV) for k, v in p16.items()},
                        vae_params={k: v.to(DEV) for k, v in v16.items()})
    cond, pooled = a.synthetic_text_embeddings(text_len=16)
    la, _ = a.denoise_latents(cond, pooled, num_steps=2, latent_size=(8, 8), seed=3)
    lb, _ = b.denoise_latents(cond, pooled, num_steps=2, latent_size=(8, 8), seed=3)
    assert torch.equal(la, lb)
    assert torch.equal(a.decode_latents_to_image(la), b.decode_latents_to_image(lb))
    return {}


def check_pipeline_q4_ckpt():
    """`*-4bit-quantized` model versions: a checkpoint in the reference's saved layout (final names, MLX 4-bit triples
    for every Linear) loads to exactly the latents of the same weights dequantised by the oracle."""
    import tempfile

    from safetensors.torch import save_file

    from oracle import quant_ref as qr

    out = {}
    for kind in ("flux", "sd35"):
        if kind == "flux":
            cfg, dtype, Pipe = tiny_flux_config(), torch.bfloat16, dk.FluxPipeline
            mv, prefix = "argmaxinc/mlx-FLUX.1-schnell-4bit-quantized", ""
        else:
            cfg, dtype, Pipe = tiny_sd35_config(), torch.float16, dk.DiffusionPipeline
            mv, prefix = "argmaxinc/mlx-stable-diffusion-3.5-large-4bit-quantized", "model.diffusion_model."
        p32 = init_params(mmdit_param_specs(cfg), seed=7, dtype=torch.float32)
        v16 = {k: v.to(dtype) for k, v in init_params(vae_decoder_param_specs(VAEDecoderConfig()), seed=8,
                                                       dtype=torch.float32).items()}
        file, dense = {}, {}
        nq = 0
        for k, v in p32.items():
            if k.endswith(".weight") and v.dim() == 2 and "pos_embed" not in k:      # nn.Linear -> QuantizedLinear
                wq, sc, bi = qr.quantize_q4(v.numpy())
                sc16, bi16 = torch.from_numpy(sc).to(dtype), torch.from_numpy(bi).to(dtype)
                file[prefix + k] = torch.from_numpy(wq.view(np.int32)).view(torch.uint32)
                file[prefix + k[:-7] + ".scales"], file[prefix + k[:-7] + ".biases"] = sc16, bi16
                dense[k] = torch.from_numpy(qr.dequantize_q4(wq, sc16.float().numpy(), bi16.float().numpy())).to(dtype)
                nq += 1
            else:
                file[prefix + k] = dense[k] = v.to(dtype)
        if kind == "sd35":                                # single file: the (dense) VAE rides along, already renamed
            file.update({"first_stage_model.decoder." + k: v for k, v in v16.items()})
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "q4.safetensors")
            save_file({k: v.contiguous() for k, v in file.items()}, path)
            a = Pipe(w16=True, a16=True, model_version=mv, mmdit_config=cfg, local_ckpt=path,
                     vae_params=None if kind == "sd35" else {k: v.to(DEV) for k, v in v16.items()})
        b = Pipe(w16=True, a16=True, model_version=mv, mmdit_config=cfg, params={k: v.to(DEV) for k, v in dense.items()},
                 vae_params={k: v.to(DEV) for k, v in v16.items()})
        cond, pooled = a.synthetic_text_embeddings(text_len=16)
        cfgw = 0.0 if kind == "flux" else 4.0
        la, _ = a.denoise_latents(cond, pooled, num_steps=2, cfg_weight=cfgw, latent_size=(8, 8), seed=3)
        lb, _ = b.denoise_latents(cond, pooled, num_steps=2, cfg_weight=cfgw, latent_size=(8, 8), seed=3)
        assert torch.equal(la, lb), kind
        assert torch.equal(a.decode_latents_to_image(la), b.decode_latents_to_image(lb)), kind
        out[kind + "_quantised_linears"] = nq
    return out


def _clip_case(cfg, dtype, B, N, tol):
    from diffusionkit_b200.text_encoders import CLIPTextModel, clip_param_specs
    from oracle.text_ref import CLIPTextModelRef

    p16 = {k: v.to(dtype) for k, v in init_params(clip_param_specs(cfg), seed=21, dtype=torch.float32).items()}
    gen = torch.Generator().manual_seed(2)
    tokens = torch.randint(1, cfg.vocab_size - 1, (B, N), generator=gen)
    for b in range(B):
        tokens[b, N - 1 - 3 * b] = cfg.vocab_size - 1                  # EOS (largest id) at different positions
    pooled, last, hidden = CLIPTextModelRef({k: v.float() for k, v in p16.items()}, cfg.num_layers, cfg.num_heads,
                                            cfg.hidden_act)(tokens)
    out = CLIPTextModel({k: v.to(DEV) for k, v in p16.items()}, cfg)(tokens)
    torch.cuda.synchronize()
    res = {"last": rel_l2(out.last_hidden_state, last), "pooled": rel_l2(out.pooled_output, pooled),
           "hidden_m2": rel_l2(out.hidden_states[-2], hidden[-2])}
    assert len(out.hidden_states) == cfg.num_layers
    for k, v in res.items():
        assert v <= tol, f"clip {k} rel_l2 {v:.3e}"
    return res


def check_clip_tiny():
    from diffusionkit_b200.config import tiny_clip_config

    a = _clip_case(tiny_clip_config(True, "quick_gelu"), torch.bfloat16, 2, 77, 2e-2)
    b = _clip_case(tiny_clip_config(False, "gelu"), torch.float16, 3, 20, 3e-3)
    return {"bf16_quick_gelu": a, "fp16_gelu_noproj": b}


def check_t5_tiny():
    from diffusionkit_b200.config import tiny_t5_config
    from diffusionkit_b200.text_encoders import SD3T5Encoder, t5_param_specs
    from oracle.text_ref import T5EncoderRef

    cfg = tiny_t5_config()
    p32 = init_params(t5_param_specs(cfg), seed=22, dtype=torch.float32)
    p32["encoder.relative_attention_bias.embeddings.weight"] *= 50.0        # make the position bias matter
    p32["wte.weight"] *= 50.0                                               # O(1) embeddings
    p16 = {k: v.to(torch.bfloat16) for k, v in p32.items()}
    gen = torch.Generator().manual_seed(3)
    out = {}
    enc = SD3T5Encoder({k: v.to(DEV) for k, v in p16.items()}, cfg)
    ref = T5EncoderRef({k: v.float() for k, v in p16.items()}, cfg.num_layers, cfg.num_heads)
    ref16 = T5EncoderRef({k: v.float() for k, v in p16.items()}, cfg.num_layers, cfg.num_heads, dt=torch.bfloat16)
    for (B, L) in [(2, 64), (1, 200)]:
        tokens = torch.randint(0, cfg.vocab_size, (B, L), generator=gen)
        got = enc(tokens)
        torch.cuda.synchronize()
        assert got.shape == (B, L, cfg.d_model)
        want = ref(tokens)
        r = rel_l2(got, want)
        # yardstick: the oracle run with the reference's own 16-bit rounding points (attention in bf16, t5.py:216-218)
        # against the same oracle in fp32.  The engine has to be at least as close to fp32 as that.
        r16 = rel_l2(ref16(tokens), want)
        assert r <= max(2e-2, r16), f"t5 rel_l2 {r:.3e} (reference-dtype oracle: {r16:.3e})"
        out[f"L{L}"] = r
        out[f"L{L}_reference_dtype_oracle"] = r16
    return out


def check_pipeline_encode_text():
    """encode_text of both pipelines on tiny encoders + a synthetic CLIP vocabulary and a sentencepiece model trained
    on the spot, vs the oracle encoders on the same tokens; then generate_image from a prompt string."""
    import tempfile

    import sentencepiece as spm

    from diffusionkit_b200.config import CLIPTextModelConfig, T5EncoderConfig
    from diffusionkit_b200.text_encoders import clip_param_specs, t5_param_specs
    from diffusionkit_b200.tokenizer import load_t5_tokenizer, load_tokenizer
    from oracle.text_ref import CLIPTextModelRef, T5EncoderRef, tokenize_pair
    from tests.test_text_cpu import _WORDS, _synthetic_clip_vocab

    res = {}
    with tempfile.TemporaryDirectory() as d:
        import pathlib

        vf, mf, vocab = _synthetic_clip_vocab(pathlib.Path(d))
        corpus = os.path.join(d, "corpus.txt")
        with open(corpus, "w") as f:
            for i in range(200):
                f.write(" ".join(_WORDS[(i + j) % len(_WORDS)] for j in range(6)) + "\n")
        spm.SentencePieceTrainer.train(input=corpus, model_prefix=os.path.join(d, "spiece"), vocab_size=64,
                                       model_type="unigram", pad_id=0, eos_id=1, unk_id=2, bos_id=-1,
                                       character_coverage=1.0, hard_vocab_limit=False, minloglevel=2)
        tok_l = load_tokenizer(vf, mf, pad_with_eos=True)
        tok_g = load_tokenizer(vf, mf, pad_with_eos=False)
        V = len(vocab)
        cl = CLIPTextModelConfig(num_layers=2, model_dims=128, num_heads=2, vocab_size=V, projection_dim=None)
        cg = CLIPTextModelConfig(num_layers=3, model_dims=192, num_heads=3, vocab_size=V, projection_dim=192,
                                 hidden_act="gelu")
        t5c = T5EncoderConfig(vocab_size=256, d_model=4096, d_kv=64, d_ff=256, num_layers=2, num_heads=2)
        pl = init_params(clip_param_specs(cl), seed=31, dtype=torch.float32)
        pg = init_params(clip_param_specs(cg), seed=32, dtype=torch.float32)
        pt = init_params(t5_param_specs(t5c), seed=33, dtype=torch.float32)
        pt["wte.weight"] *= 50.0
        prompt, negative = "a photo of the astronaut riding a horse on mars!", "cats"
        for kind in ("sd3", "flux"):
            if kind == "sd3":
                cfg = replace(tiny_sd3_config(), pooled_text_embed_dim=128 + 192, token_level_text_embed_dim=4096)
                pipe = dk.DiffusionPipeline(w16=True, a16=True, shift=3.0, mmdit_config=cfg)
                t5_len = 512
            else:
                cfg = replace(tiny_flux_config(), pooled_text_embed_dim=128, token_level_text_embed_dim=4096)
                pipe = dk.FluxPipeline(w16=True, a16=True, mmdit_config=cfg)
                t5_len = 256
            dt = pipe.dtype
            tok_t5 = load_t5_tokenizer(os.path.join(d, "spiece.model"), t5_len)
            try:
                pipe.encode_text(prompt)
                raise RuntimeError("encode_text without encoders should refuse")
            except dk.DkError:
                pass
            pipe.load_text_encoders(clip_l={k: v.to(dt) for k, v in pl.items()}, clip_g={k: v.to(dt) for k, v in pg.items()},
                                    t5={k: v.to(torch.bfloat16) for k, v in pt.items()}, tokenizer_l=tok_l,
                                    tokenizer_g=tok_g, t5_tokenizer=tok_t5, clip_l_config=cl, clip_g_config=cg,
                                    t5_config=t5c)
            cond, pooled = pipe.encode_text(prompt, cfg_weight=5.0, negative_text=negative)
            # oracle on the same tokens, weights rounded like the device copies
            ref_l = CLIPTextModelRef({k: v.to(dt).float() for k, v in pl.items()}, cl.num_layers, cl.num_heads, cl.hidden_act)
            ref_g = CLIPTextModelRef({k: v.to(dt).float() for k, v in pg.items()}, cg.num_layers, cg.num_heads, cg.hidden_act)
            ref_t = T5EncoderRef({k: v.to(torch.bfloat16).float() for k, v in pt.items()}, t5c.num_layers, t5c.num_heads)
            tl, tg, tt = [tokenize_pair(t, prompt, negative) for t in (tok_l, tok_g, tok_t5)]
            if kind == "sd3":
                pl_o, _, hl = ref_l(tl)
                pg_o, _, hg = ref_g(tg)
                c = torch.cat([hl[-2], hg[-2]], dim=-1)
                c = torch.cat([c, torch.zeros(2, 77, 4096 - c.shape[-1])], dim=-1)
                assert tt.shape == (2, 512) and cond.shape == (2, 77 + 512, 4096) and pooled.shape == (2, 320)
                want_c, want_p = torch.cat([c, ref_t(tt)], dim=1), torch.cat([pl_o, pg_o], dim=-1)
            else:
                pl_o, _, _ = ref_l(tl[[0]])
                padded = torch.zeros((1, 256), dtype=torch.int64)
                padded[:, : tt.shape[1]] = tt[[0]]
                want_c, want_p = ref_t(padded), pl_o
                assert cond.shape == (1, 256, 4096) and pooled.shape == (1, 128)
            assert cond.dtype == pooled.dtype == pipe.activation_dtype
            res[kind + "_cond"], res[kind + "_pooled"] = rel_l2(cond, want_c), rel_l2(pooled, want_p)
            assert res[kind + "_cond"] <= 2e-2 and res[kind + "_pooled"] <= 2e-2, res
            image, log = pipe.generate_image(prompt, num_steps=2, cfg_weight=5.0 if kind == "sd3" else 0.0,
                                             negative_text=negative, latent_size=(8, 8), seed=1, verbose=False)
            assert image.size == (64, 64) and log["text_encoding"]["time"] >= 0
            # batch-N extension with a TEXT prompt: one prompt, several seeds -> a list of images; image i equals the
            # single-seed run with that seed (the prompt's conditioning is shared, [positive x B | negative x B])
            many, _ = pipe.generate_image(prompt, num_steps=2, cfg_weight=5.0 if kind == "sd3" else 0.0,
                                          negative_text=negative, latent_size=(8, 8), seed=[1, 9], verbose=False)
            assert isinstance(many, list) and len(many) == 2
            solo9, _ = pipe.generate_image(prompt, num_steps=2, cfg_weight=5.0 if kind == "sd3" else 0.0,
                                           negative_text=negative, latent_size=(8, 8), seed=9, verbose=False)
            d0 = np.abs(np.asarray(many[0]).astype(np.int32) - np.asarray(image).astype(np.int32)).max()
            d1 = np.abs(np.asarray(many[1]).astype(np.int32) - np.asarray(solo9).astype(np.int32)).max()
            assert d0 <= 1 and d1 <= 1, (kind, d0, d1)
            res[kind + "_multiseed_u8_diff"] = int(max(d0, d1))
    return res


def check_full_size_text_encoders():
    """CLIP-L/14, OpenCLIP bigG and T5-XXL (4.7 B parameters) at their real sizes with synthetic weights: shapes,
    determinism, finiteness, batch independence; CUDA-event times for DESIGN.md."""
    from diffusionkit_b200.config import CLIP_G, CLIP_L, T5EncoderConfig
    from diffusionkit_b200.text_encoders import CLIPTextModel, SD3T5Encoder, clip_param_specs, t5_param_specs

    out = {}
    gen = torch.Generator().manual_seed(9)

    def timed(fn):
        fn()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        r = fn()
        e.record()
        torch.cuda.synchronize()
        return r, s.elapsed_time(e)

    for name, cfg in (("clip_l", CLIP_L), ("clip_g", CLIP_G)):
        m = CLIPTextModel(init_params(clip_param_specs(cfg), seed=41, dtype=torch.float16, device=DEV), cfg)
        tokens = torch.randint(1, 49406, (2, 77), generator=gen)
        tokens[:, 30] = 49407
        o, ms = timed(lambda: m(tokens))
        o2 = m(tokens[1:2])
        assert o.last_hidden_state.shape == (2, 77, cfg.model_dims) and bool(torch.isfinite(o.last_hidden_state.float()).all())
        assert o.pooled_output.shape == (2, cfg.projection_dim or cfg.model_dims)
        assert rel_l2(o2.last_hidden_state, o.last_hidden_state[1:2]) <= 1e-5
        out[name + "_ms"] = round(ms, 3)
        del m
    t5 = SD3T5Encoder(init_params(t5_param_specs(T5EncoderConfig()), seed=42, dtype=torch.bfloat16, device=DEV))
    for L in (256, 512):
        tokens = torch.randint(0, 32128, (2, L), generator=gen)
        o, ms = timed(lambda: t5(tokens))
        assert o.shape == (2, L, 4096) and bool(torch.isfinite(o.float()).all())
        assert torch.equal(o, t5(tokens)), "T5 encoder is not deterministic"
        assert rel_l2(t5(tokens[1:2]), o[1:2]) <= 1e-5
        out[f"t5_xxl_L{L}_B2_ms"] = round(ms, 3)
    return out


def check_product_vs_reference_source():
    """The CUDA product directly against outputs of the REFERENCE'S OWN SOURCE — its MLX files executed (fp32) on the
    torch-backed stand-in for the MLX primitives, tests/golden/make_reference_mlx_golden.py — with no oracle in between:
    FLUX and SD3 MMDiT forward through the modulation cache, VAE decoder (raw output and clipped image) and VAE encoder
    (uint8 image in, read_image scaling fused) at their real widths.  16-bit product vs fp32 reference source; bounds =
    the 16-bit-vs-fp32 tolerances of this file."""
    from tests.golden import make_reference_mlx_golden as mk

    out = {}
    flux, sd3 = mk.pin_configs()
    for kind, cfg, dtype in (("flux", flux, torch.bfloat16), ("sd3", sd3, torch.float16)):
        g = np.load(os.path.join(GOLD, f"reference_mlxsrc_{kind}_mmdit.npz"))
        latent, text, pooled, timesteps = [torch.from_numpy(g[k]) for k in ("latent", "text", "pooled", "timesteps")]
        ti = int(g["t_index"])
        p16 = {k: v.to(dtype) for k, v in init_params(mmdit_param_specs(cfg), seed=mk.SEEDS[kind],
                                                       dtype=torch.float32).items()}
        m = dk.MMDiT(cfg, {k: v.to(DEV) for k, v in p16.items()})
        m.cache_modulation_params(pooled.to(dtype).to(DEV), [float(t) for t in timesteps])
        got = m(latent_image_embeddings=latent.to(dtype).to(DEV),
                token_level_text_embeddings=text.to(dtype).to(DEV).unsqueeze(2),
                timestep=torch.full((latent.shape[0],), float(timesteps[ti])))
        torch.cuda.synchronize()
        want = torch.from_numpy(g["out"])
        r, ps = rel_l2(got, want), psnr(want, got)
        assert r <= 2e-2 and ps >= 35.0, f"{kind} vs reference source: rel_l2={r:.3e} psnr={ps:.1f}"
        out[kind + "_rel_l2"], out[kind + "_psnr"] = r, ps
    g = np.load(os.path.join(GOLD, "reference_mlxsrc_vae_fullwidth.npz"))
    dt = torch.bfloat16
    # same CPU-generated fp32 weights as the fixture, rounded to 16 bits, then moved (a CUDA generator would differ)
    dec = dk.VAEDecoder({k: v.to(dt).to(DEV) for k, v in init_params(
        vae_decoder_param_specs(VAEDecoderConfig()), seed=mk.SEEDS["vae_dec"], dtype=torch.float32).items()})
    raw = dec(torch.from_numpy(g["latent"]).to(dt).to(DEV))
    want_raw = torch.from_numpy(g["decoded"].astype(np.float32))
    out["vae_decoder_rel_l2"] = rel_l2(raw, want_raw)
    assert out["vae_decoder_rel_l2"] <= 3e-2, out
    Bo, Ho, Wo, _ = raw.shape
    padded = raw.as_strided((Bo, Ho, Wo, raw.stride(2)), (raw.stride(0), raw.stride(1), raw.stride(2), 1))
    f, _ = ops.image_post(padded)
    out["vae_image_psnr"] = psnr(torch.from_numpy(g["decoded_image"].astype(np.float32)), f)
    assert out["vae_image_psnr"] >= 35.0, out
    enc = dk.VAEEncoder({k: v.to(dt).to(DEV) for k, v in init_params(
        vae_encoder_param_specs(VAEEncoderConfig()), seed=mk.SEEDS["vae_enc"], dtype=torch.float32).items()})
    hid = enc(torch.from_numpy(g["image_u8"]).unsqueeze(0).to(DEV))
    torch.cuda.synchronize()
    out["vae_encoder_rel_l2"] = rel_l2(hid, torch.from_numpy(g["encoded"]))
    assert out["vae_encoder_rel_l2"] <= 3e-2, out
    return out


def check_full_size_sd35_properties():
    """SD3.5-large at its real width/depth (SD3_8b: 38 blocks, 38 heads x 64, hidden 2432, QK-norm; 8 B synthetic
    parameters), 512x512, CFG: determinism, batch independence, finiteness."""
    pipe = dk.DiffusionPipeline(w16=True, a16=True, shift=3.0, model_version="argmaxinc/mlx-stable-diffusion-3.5-large",
                                load_decoder=False)
    assert pipe.config.hidden_size == 2432 and pipe.config.head_dim == 64 and pipe.config.use_qk_norm
    cond, pooled = pipe.synthetic_text_embeddings(n_images=2, text_len=154)
    kw = dict(num_steps=3, cfg_weight=4.5, latent_size=(64, 64))
    a, _ = pipe.denoise_latents(cond, pooled, seed=[5, 6], **kw)
    b, _ = pipe.denoise_latents(cond, pooled, seed=[5, 6], **kw)
    assert torch.equal(a, b), "denoise loop is not deterministic"
    assert bool(torch.isfinite(a).all())
    solo, _ = pipe.denoise_latents(cond[[1, 3]], pooled[[1, 3]], seed=6, **kw)
    r = rel_l2(a[1:2], solo)
    assert r <= 1e-5, f"batch composition changed image 1: rel_l2 {r:.3e}"
    return {"batch_vs_solo_rel_l2": r, "latent_abs_mean": float(a.abs().mean()), "latent_abs_max": float(a.abs().max())}


def check_full_size_flux_properties():
    """FLUX.1-schnell at its real width/depth (11.9 B synthetic parameters), 512x512, 4 steps: size-independent
    properties the oracle cannot check in seconds — determinism (no atomics on the path), batch independence
    (image i of a batch == the same seed/prompt alone; the property batch sharding across GPUs relies on), finiteness."""
    pipe = dk.FluxPipeline(w16=True, a16=True, shift=1.0, model_version="argmaxinc/mlx-FLUX.1-schnell",
                           load_decoder=False)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=2)
    kw = dict(num_steps=4, cfg_weight=0.0, latent_size=(64, 64))
    a, _ = pipe.denoise_latents(cond, pooled, seed=[5, 6], **kw)
    b, _ = pipe.denoise_latents(cond, pooled, seed=[5, 6], **kw)
    assert torch.equal(a, b), "denoise loop is not deterministic"
    solo, _ = pipe.denoise_latents(cond[1:2], pooled[1:2], seed=6, **kw)
    assert bool(torch.isfinite(a).all())
    r = rel_l2(a[1:2], solo)
    assert r <= 1e-5, f"batch composition changed image 1: rel_l2 {r:.3e}"
    # statistics of a 4-step latent stay in a sane range for unit-variance synthetic inputs
    return {"batch_vs_solo_rel_l2": r, "latent_abs_mean": float(a.abs().mean()), "latent_abs_max": float(a.abs().max())}


def check_full_size_vae_properties():
    """VAE decode at 1024x1024: batch independence, determinism, range."""
    vp = init_params(vae_decoder_param_specs(VAEDecoderConfig()), seed=8, dtype=torch.bfloat16, device=DEV)
    dec = dk.VAEDecoder(vp)
    g = torch.Generator().manual_seed(2)
    z = torch.randn((2, 128, 128, 16), generator=g).to(torch.bfloat16).to(DEV)

    def run(zz):
        raw = dec(zz)
        Bo, Ho, Wo, _ = raw.shape
        padded = raw.as_strided((Bo, Ho, Wo, raw.stride(2)), (raw.stride(0), raw.stride(1), raw.stride(2), 1))
        return ops.image_post(padded)

    f2, u2 = run(z)
    f2b, _ = run(z)
    assert torch.equal(f2, f2b), "VAE decode is not deterministic"
    f1, u1 = run(z[1:2].contiguous())
    assert f2.shape == (2, 1024, 1024, 3) and float(f2.min()) >= 0.0 and float(f2.max()) <= 1.0
    d = (u2[1:2].int() - u1.int()).abs()
    assert int(d.max()) == 0, f"batch composition changed image 1 by {int(d.max())} uint8 levels"
    return {"u8_max_diff_batch_vs_solo": int(d.max()), "mean": float(f2.mean())}


# ------------------------------------------------------------------------------------------------ BASELINE widths
def _fullwidth_cfg(model_version, depth_mm, depth_uni):
    from diffusionkit_b200.config import MODEL_CONFIGS

    full = MODEL_CONFIGS[model_version]
    return full, replace(full, depth_multimodal=depth_mm, depth_unified=depth_uni, hidden_size_override=full.hidden_size)


def check_fullwidth_flux_vs_oracle():
    """FLUX.1-schnell at its REAL width and the C4 sequence length (h = 3072, 24 heads x 128, S = 4096 + 256, 1024^2
    image) through a truncated depth (1 double + 1 single block) against the fp32 oracle — the shapes bench.py times
    (reference mlx/mmdit.py:188-266, 568-751)."""
    full, cfg = _fullwidth_cfg("argmaxinc/mlx-FLUX.1-schnell", 1, 1)
    assert cfg.hidden_size == 3072 and cfg.head_dim == 128
    return _mmdit_case(cfg, torch.bfloat16, 1, (128, 128), 256)


def check_fullwidth_flux_dev_len_vs_oracle():
    """same at the C5 text length (S = 4096 + 512), batch 2: 4608 is not a multiple of the 256-row attention work item"""
    full, cfg = _fullwidth_cfg("argmaxinc/mlx-FLUX.1-schnell", 1, 1)
    return _mmdit_case(cfg, torch.bfloat16, 2, (128, 64), 512)


def check_fullwidth_sd3_vs_oracle():
    """SD3-medium at its real width and the C3 sequence length (h = 1536, 24 heads x 64, S = 4096 + 589 (77 + 512 T5),
    fp16) through 2 blocks (the last one skips the text post-attention path, mlx/mmdit.py:62-66)"""
    full, cfg = _fullwidth_cfg("argmaxinc/mlx-stable-diffusion-3-medium", 2, 0)
    assert cfg.hidden_size == 1536 and cfg.head_dim == 64
    return _mmdit_case(cfg, torch.float16, 1, (128, 128), 589)


def check_vae_decode_512_vs_oracle():
    """a complete 512 x 512 decode (latent 64^2, every layer at its real width) against the fp32 oracle
    (reference mlx/vae.py:386-401)"""
    return _vae_case(torch.bfloat16, 1, (64, 64), 35.0)


def check_vae_decode_1024_vs_oracle():
    """the BASELINE decode: 1024 x 1024 (latent 128^2, mid attention over S = 16384) against the fp32 oracle"""
    return _vae_case(torch.bfloat16, 1, (128, 128), 35.0)


def check_mmdit_shape_switch_graphs():
    """one model serving shapes A, B, A, C... with CUDA-graph replay == the same model launching kernel by kernel:
    each captured graph owns its workspace / RoPE table / cropped positional embedding, including after an LRU
    eviction (max_cached_shapes = 2 here) — the replay of A after B must not read freed buffers"""
    out = {}
    for name, cfg, dt in (("flux", tiny_flux_config(), torch.bfloat16), ("sd3", tiny_sd3_config(), torch.float16)):
        p16 = init_params(mmdit_param_specs(cfg), seed=11, dtype=dt, device=DEV)
        mg, me = dk.MMDiT(cfg, p16), dk.MMDiT(cfg, p16)
        mg.use_cuda_graphs, me.use_cuda_graphs = True, False
        mg.max_cached_shapes = 2
        gen = torch.Generator().manual_seed(3)
        pooled = torch.randn((2, cfg.pooled_text_embed_dim), generator=gen).to(dt).to(DEV)
        for m in (mg, me):
            m.cache_modulation_params(pooled, [752.0, 500.0])
        shapes = {"A": ((8, 12), 16), "B": ((16, 8), 24), "C": ((12, 12), 8)}
        worst = 0.0
        for step, sk in enumerate("ABACABCA"):
            (H, W), T = shapes[sk]
            lat = torch.randn((2, H, W, 16), generator=gen).to(dt).to(DEV)
            txt = torch.randn((2, T, cfg.token_level_text_embed_dim), generator=gen).to(dt).to(DEV)
            tval = 752.0 if step % 2 == 0 else 500.0
            a = mg(lat, txt, timestep=tval).clone()
            # garbage allocations between calls: whatever a stale graph pointed at would now hold other data
            junk = [torch.full((1 << 18,), float("nan"), dtype=dt, device=DEV) for _ in range(8)]
            b = me(lat, txt, timestep=tval)
            torch.cuda.synchronize()
            del junk
            assert bool(torch.isfinite(a.float()).all()), f"{name} step {step} ({sk}): non-finite output"
            assert torch.equal(a, b), f"{name} step {step} (shape {sk}): graph replay != eager, rel_l2 {rel_l2(a, b):.3e}"
            worst = max(worst, rel_l2(a, b))
        assert len(mg._shapes) <= 2
        out[name] = worst
    return out


ALL_CHECKS = [check_mmdit_flux_tiny, check_mmdit_sd3_tiny, check_product_vs_reference_source, check_mmdit_sd35_tiny, check_pipeline_q4_ckpt,
              check_full_size_sd35_properties, check_clip_tiny, check_t5_tiny, check_pipeline_encode_text,
              check_full_size_text_encoders, check_mmdit_flux_ragged, check_mmdit_sd3_d64_long, check_mmdit_shape_switch_graphs,
              check_vae_decode_tiny, check_vae_decode_batch_fp16, check_vae_encode_tiny, check_vae_encode_batch_fp16,
              check_pipeline_img2img, check_pipeline_flux_tiny, check_pipeline_sd3_cfg_tiny,
              check_pipeline_errors, check_pipeline_local_ckpt, check_full_size_flux_properties, check_full_size_vae_properties,
              check_fullwidth_flux_vs_oracle, check_fullwidth_flux_dev_len_vs_oracle, check_fullwidth_sd3_vs_oracle,
              check_vae_decode_512_vs_oracle, check_vae_decode_1024_vs_oracle]
