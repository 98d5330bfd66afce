#!/usr/bin/env python
"""FLUX.1 Redux image prompts (DESIGN.md §15) on FLUX.1-dev (FLUX_DEV config, synthetic weights, CUDA graphs for the
MMDiT), arms alternated --rounds times in one process:

  python tools/bench_redux.py [--rounds 3] [--forwards 10] [--encodes 10] [--steps 28]

(a) the SigLIP so400m + Redux encode of 1 and 4 images at real width and depth (27 layers, 384^2, 729 tokens), eager,
    device time from 384^2 images already in HBM, with the achieved TFLOP/s of the FLOPs it needs computed from the
    (padded) shapes; and encode_redux end to end, host resize included;
(b) one MMDiT forward at the C5 shape (1024^2 = latent 128^2, one image) with T = 512 text rows and with T = 512 + 729;
(c) a --steps Euler denoise (denoise_latents, no decode) without and with an image prompt.
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
from tools.bench_kontext import wall  # noqa: E402

LAT, T, GUIDANCE = 128, 512, 3.5


def encoder_tflop(scfg, txt_dim: int = 4096) -> dict:
    """FLOPs of one image's encode as the kernels run it: the padded linears (head dim 72 -> 128 in qkv / out_proj,
    patch K 588 -> 592), the padded attention (QK^T and PV at d = 128), and the Redux projector"""
    from diffusionkit_b200.image_encoders import padded_head_dim, patch_weight_kp

    P, D, F, L = scfg.num_patches, scfg.hidden_size, scfg.intermediate_size, scfg.num_hidden_layers
    hd = scfg.num_attention_heads * padded_head_dim(scfg)
    lin = 2 * P * (patch_weight_kp(scfg) * D + L * (D * 3 * hd + hd * D + 2 * D * F))
    att = L * 4 * P * P * hd
    proj = 2 * P * (D * 3 * txt_dim + 3 * txt_dim * txt_dim)
    return {"linear": round(lin / 1e12, 3), "attention": round(att / 1e12, 3), "projector": round(proj / 1e12, 3),
            "total": round((lin + att + proj) / 1e12, 3)}


def forward_tflop(cfg, text_rows: int) -> dict:
    """FLOPs of one FLUX forward of one sequence (tools/bench_kontext.forward_tflop's terms)"""
    h, blocks = cfg.hidden_size, cfg.depth_multimodal + cfg.depth_unified
    S = text_rows + (LAT // 2) ** 2
    lin, att = 24 * blocks * h * h * S / 1e12, 4 * blocks * S * S * h / 1e12
    return {"S": S, "tflop": round(lin + att, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--forwards", type=int, default=10)
    ap.add_argument("--encodes", type=int, default=10)
    ap.add_argument("--steps", type=int, default=28)
    args = ap.parse_args()
    import numpy as np
    import torch

    import diffusionkit_b200 as dk
    from diffusionkit_b200.config import FLUX_DEV
    from diffusionkit_b200.sampler import flux_resolution_shift

    if not torch.cuda.is_available():
        raise SystemExit("bench_redux.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    pipe = dk.FluxPipeline(w16=True, a16=True, shift=flux_resolution_shift((LAT, LAT)),
                           model_version="argmaxinc/mlx-FLUX.1-dev", mmdit_config=FLUX_DEV, device=dev,
                           load_decoder=False)
    pipe.load_redux()
    scfg = pipe.siglip.config
    P = scfg.num_patches
    rng = np.random.RandomState(0)
    imgs = [rng.randint(0, 256, (512, 640, 3)).astype(np.uint8) for _ in range(4)]
    out = {"encoder_tflop_per_image": encoder_tflop(scfg)}

    # (a) the encode, 1 and 4 images
    enc = {}
    for n in (1, 4):
        x = torch.from_numpy(np.stack([pipe._redux_image_u8(im) for im in imgs[:n]])).to(dev)

        def device_encode(x=x):
            h = pipe.siglip(x)
            return pipe.redux(h.reshape(-1, h.shape[2]), P)

        wall(device_encode, 2)
        wall(lambda n=n: pipe.encode_redux(imgs[:n]), 2)
        dt = min(wall(device_encode, args.encodes) for _ in range(args.rounds))
        e2e = min(wall(lambda n=n: pipe.encode_redux(imgs[:n]), args.encodes) for _ in range(args.rounds))
        enc[n] = {"device_ms": round(dt * 1e3, 2), "encode_redux_ms": round(e2e * 1e3, 2),
                  "achieved_tflops": round(n * out["encoder_tflop_per_image"]["total"] / dt, 1)}
    out["encode"] = enc

    # (b) the forward at T = 512 and T = 512 + 729, alternated
    cond, pooled = [t.to(dev) for t in pipe.synthetic_text_embeddings(n_images=1, text_len=T)]
    tok = pipe.encode_redux(imgs[0])
    arms = {"T512": cond, "T1241": torch.cat([cond, tok], dim=1).contiguous()}
    out["flops"] = {k: forward_tflop(pipe.config, v.shape[1]) for k, v in arms.items()}
    out["tflop_ratio"] = round(out["flops"]["T1241"]["tflop"] / out["flops"]["T512"]["tflop"], 3)
    m = pipe.mmdit
    assert m.use_cuda_graphs
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn((1, LAT, LAT, 16), generator=g, device=dev).to(torch.bfloat16)
    m.cache_modulation_params(pooled, [500.0], [GUIDANCE])
    fw = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, c in arms.items():
            fn = (lambda c=c: m(x, c, 500.0))
            wall(fn, 2)
            fw[k].append(round(wall(fn, args.forwards) * 1e3, 2))
    out["forward_ms"] = fw
    out["forward_ratio"] = round(min(fw["T1241"]) / min(fw["T512"]), 3)

    # (c) a --steps Euler denoise without and with an image prompt
    den = {"none": [], "redux": []}

    def denoise(k):
        lat, _ = pipe.denoise_latents(cond, pooled, num_steps=args.steps, latent_size=(LAT, LAT), seed=0,
                                      guidance=GUIDANCE, redux_image=imgs[0] if k == "redux" else None)
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
    out["denoise_redux_over_none"] = round(min(den["redux"]) / min(den["none"]), 3)
    out["denoise_steps"] = args.steps
    print(json.dumps({**out, "rounds": args.rounds, "forwards": args.forwards, **card_info()}), flush=True)


if __name__ == "__main__":
    main()
