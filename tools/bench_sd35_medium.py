#!/usr/bin/env python
"""SD3.5 Medium (MMDiT-X) and skip-layer guidance at 1024^2 (latent 128^2, text length 77 + 512 = 589), synthetic
weights, arms alternated --rounds times in one process:

  python tools/bench_sd35_medium.py [--rounds 3] [--forwards 10] [--steps 40]

(a) one MMDiT forward, SD3.5 Medium against SD3-medium (SD3_2b) at the same shape, at B = 2 and B = 8 (1 and 4 images
    under CFG), beside the matmul FLOPs both need, computed from the shapes;
(b) the 3B skip-layer-guidance forward (layers 7, 8, 9 skipped for the last B) against the 2B forward, one image;
(c) a --steps DPM-Solver++(2M) CFG 4.5 denoise of one image (denoise_latents, no decode) with SLG off and with
    SkipLayerGuidance(), then one generate_image with SLG through the VAE, under CUDA graphs.
Host clock around work that ends in a device synchronise; prints the card, its power limit and SM clock read in the
same run, and fails when there is no GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_gemm import card_info  # noqa: E402

LAT, T, CFGW = 128, 589, 4.5
MEDIUM = "stabilityai/stable-diffusion-3.5-medium"
SD3 = "argmaxinc/mlx-stable-diffusion-3-medium"


def forward_tflop(cfg, B: int) -> float:
    """matmul FLOPs of one MMDiT forward of B sequences at the bench shape (block linears and attention; the
    embedders, modulation and final layer are < 0.1 %)"""
    h, N = cfg.hidden_size, (LAT // 2) ** 2
    S = N + T
    f = 0.0
    for i in range(cfg.depth_multimodal):
        last = i == cfg.depth_multimodal - 1
        f += 2 * N * 12 * h * h + 2 * T * (3 if last else 12) * h * h + 4 * S * S * h
        if i in cfg.x_block_self_attn_layers:
            f += 2 * N * 4 * h * h + 4 * N * N * h                   # attn2 q/k/v/o and its attention
    return B * f / 1e12


def wall(fn, n):
    import torch

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--forwards", type=int, default=10)
    ap.add_argument("--steps", type=int, default=40)
    args = ap.parse_args()
    import torch

    import diffusionkit_b200 as dk
    from diffusionkit_b200.sampler import SkipLayerGuidance, skip_layer_guidance_steps

    if not torch.cuda.is_available():
        raise SystemExit("bench_sd35_medium.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    pipes = {mv: dk.DiffusionPipeline(w16=True, a16=True, shift=3.0, model_version=mv, device=dev,
                                      load_decoder=mv == MEDIUM) for mv in (SD3, MEDIUM)}
    out = {"tflop_per_forward": {f"B{B}": {mv: round(forward_tflop(p.config, B), 2) for mv, p in pipes.items()}
                                 for B in (2, 8)}}

    # (a) forward, Medium against SD3-medium, alternated
    fw = {f"B{B}": {mv: [] for mv in pipes} for B in (2, 8)}
    for B in (2, 8):
        inputs = {}
        for mv, p in pipes.items():
            cond, pooled = [t.to(dev) for t in p.synthetic_text_embeddings(n_images=B // 2, text_len=T)]
            inputs[mv] = (torch.randn((B, LAT, LAT, 16), device=dev).to(torch.float16), cond, pooled)
        for _ in range(args.rounds):
            for mv, p in pipes.items():
                x, cond, pooled = inputs[mv]
                p.mmdit.cache_modulation_params(pooled, [500.0])
                wall(lambda: p.mmdit(x, cond, 500.0), 2)
                fw[f"B{B}"][mv].append(round(wall(lambda: p.mmdit(x, cond, 500.0), args.forwards) * 1e3, 2))
        del inputs
    out["forward_ms"] = fw
    out["medium_over_sd3"] = {k: round(min(v[MEDIUM]) / min(v[SD3]), 4) for k, v in fw.items()}
    del pipes[SD3]
    torch.cuda.empty_cache()

    # (b) the 3B SLG forward against the 2B forward, one image
    pipe = pipes[MEDIUM]
    m = pipe.mmdit
    cond, pooled = [t.to(dev) for t in pipe.synthetic_text_embeddings(n_images=1, text_len=T)]
    cond3, pooled3 = torch.cat([cond, cond[:1]]), torch.cat([pooled, pooled[:1]])
    x3 = torch.randn((3, LAT, LAT, 16), device=dev).to(torch.float16)
    m.cache_modulation_params(pooled3, [500.0], skip_batch=1)
    arms = {"2B": lambda: m(x3[:2], cond, 500.0),
            "3B_skip_7_8_9": lambda: m(x3, cond3, 500.0, skip_layers=(7, 8, 9), skip_batch=1)}
    sf = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, fn in arms.items():
            wall(fn, 2)
            sf[k].append(round(wall(fn, args.forwards) * 1e3, 2))
    out["slg_forward_ms"] = sf
    out["slg_forward_over_2B"] = round(min(sf["3B_skip_7_8_9"]) / min(sf["2B"]), 4)

    # (c) a --steps DPM-Solver++(2M) CFG denoise of one image, SLG off and on
    slg = SkipLayerGuidance()
    den = {"slg_off": [], "slg_default": []}

    def denoise(s):
        lat, _ = pipe.denoise_latents(cond, pooled, num_steps=args.steps, cfg_weight=CFGW, latent_size=(LAT, LAT),
                                      seed=0, solver="dpmpp_2m", slg=s)
        torch.cuda.synchronize()
        return lat

    for s in (None, slg):
        denoise(s)                                                   # captures each shape's graph
    for _ in range(args.rounds):
        for arm, s in (("slg_off", None), ("slg_default", slg)):
            t0 = time.perf_counter()
            lat = denoise(s)
            den[arm].append(round(time.perf_counter() - t0, 3))
            assert bool(torch.isfinite(lat).all())
    n_slg = len(skip_layer_guidance_steps(slg, args.steps))
    out["denoise_s"] = den
    out["denoise_slg_over_off"] = round(min(den["slg_default"]) / min(den["slg_off"]), 4)
    out["denoise_steps"], out["slg_steps"] = args.steps, n_slg
    image, log = pipe.generate_image("", num_steps=args.steps, cfg_weight=CFGW, latent_size=(LAT, LAT), seed=0,
                                     verbose=False, conditioning=cond, pooled_conditioning=pooled, solver="dpmpp_2m",
                                     slg=slg)
    out["generate_image"] = {"size": list(image.size), "cuda_graphs": m.use_cuda_graphs,
                             "skip_layer_guidance": log["denoising"]["skip_layer_guidance"],
                             "denoise_time_s": log["denoising"]["time"]}
    print(json.dumps({**out, "rounds": args.rounds, "forwards": args.forwards, **card_info()}), flush=True)


if __name__ == "__main__":
    main()
