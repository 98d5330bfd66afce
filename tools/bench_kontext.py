#!/usr/bin/env python
"""FLUX.1 Kontext [dev] at the C5 shape (FLUX.1-dev config, 1024^2 target = latent 128^2, T = 512, one image, synthetic
weights, CUDA graphs), arms alternated --rounds times in one process:

  python tools/bench_kontext.py [--rounds 3] [--forwards 10] [--steps 28]

(a) one MMDiT forward with no reference, with a 512^2 reference (latent 64^2) and with a 1024^2 reference (latent
    128^2), beside the FLOPs each needs, computed from the shapes;
(b) a --steps Euler denoise (denoise_latents, no decode) with no reference and with the 1024^2 reference.
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

LAT, T, GUIDANCE = 128, 512, 3.5
KONTEXT = "black-forest-labs/FLUX.1-Kontext-dev"
REFS = {"none": None, "ref512": 64, "ref1024": 128}              # arm -> reference latent side


def forward_tflop(cfg, ref_side) -> dict:
    """FLOPs of one forward of one sequence: the block linears (12 h^2 MACs per token per block) and attention
    (4 S^2 h per block); the embedders, modulation and final layer are < 0.1 %"""
    h, blocks = cfg.hidden_size, cfg.depth_multimodal + cfg.depth_unified
    S = T + (LAT // 2) ** 2 + (0 if ref_side is None else (ref_side // 2) ** 2)
    lin, att = 24 * blocks * h * h * S / 1e12, 4 * blocks * S * S * h / 1e12
    return {"S": S, "tflop": round(lin + att, 1), "attention_tflop": round(att, 1)}


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
    ap.add_argument("--steps", type=int, default=28)
    args = ap.parse_args()
    import torch

    import diffusionkit_b200 as dk
    from diffusionkit_b200.sampler import flux_resolution_shift

    if not torch.cuda.is_available():
        raise SystemExit("bench_kontext.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    pipe = dk.FluxPipeline(w16=True, a16=True, shift=flux_resolution_shift((LAT, LAT)), model_version=KONTEXT,
                           device=dev, load_decoder=False)
    m = pipe.mmdit
    assert m.use_cuda_graphs
    cond, pooled = [t.to(dev) for t in pipe.synthetic_text_embeddings(n_images=1, text_len=T)]
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn((1, LAT, LAT, 16), generator=g, device=dev).to(torch.bfloat16)
    refs32 = {k: None if s is None else torch.randn((1, s, s, 16), generator=g, device=dev) for k, s in REFS.items()}
    refs16 = {k: None if r is None else r.to(torch.bfloat16) for k, r in refs32.items()}
    flops = {k: forward_tflop(pipe.config, s) for k, s in REFS.items()}
    out = {"flops": flops, "tflop_ratio": {k: round(f["tflop"] / flops["none"]["tflop"], 2) for k, f in flops.items()}}

    # (a) forward, alternated
    m.cache_modulation_params(pooled, [500.0], [GUIDANCE])
    fw = {k: [] for k in REFS}
    for _ in range(args.rounds):
        for k in REFS:
            fn = (lambda r=refs16[k]: m(x, cond, 500.0, reference=r))
            wall(fn, 2)
            fw[k].append(round(wall(fn, args.forwards) * 1e3, 2))
    out["forward_ms"] = fw
    out["forward_over_none"] = {k: round(min(v) / min(fw["none"]), 3) for k, v in fw.items()}
    out["achieved_tflops"] = {k: round(flops[k]["tflop"] / (min(v) / 1e3), 1) for k, v in fw.items()}

    # (b) a --steps Euler denoise, no reference and the 1024^2 reference
    den = {"none": [], "ref1024": []}

    def denoise(k):
        lat, _ = pipe.denoise_latents(cond, pooled, num_steps=args.steps, latent_size=(LAT, LAT), seed=0,
                                      guidance=GUIDANCE, reference_latents=refs32[k])
        torch.cuda.synchronize()
        return lat

    for k in den:
        denoise(k)                                                   # captures each shape's graph
    for _ in range(args.rounds):
        for k in den:
            t0 = time.perf_counter()
            lat = denoise(k)
            den[k].append(round(time.perf_counter() - t0, 3))
            assert bool(torch.isfinite(lat).all())
    out["denoise_s"] = den
    out["denoise_ref1024_over_none"] = round(min(den["ref1024"]) / min(den["none"]), 3)
    out["denoise_steps"] = args.steps
    print(json.dumps({**out, "rounds": args.rounds, "forwards": args.forwards, **card_info()}), flush=True)


if __name__ == "__main__":
    main()
