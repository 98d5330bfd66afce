#!/usr/bin/env python
"""FLUX.1 Fill [dev] (DESIGN.md §18), synthetic weights, one H100:

  python tools/bench_fill.py [--rounds 3] [--steps 28]

(a) the conditioning build of one 1024^2 source with a half-image mask: the masked encode (dk_image_pre_masked and the
    VAE encoder), the posterior mean, the packing, dk_fill_cond_rows and the K = 320 GEMM (cache_fill_conditioning);
(b) one MMDiT forward at the C5 shape (1024^2, T = 512, one image) on FLUX.1-dev and on FLUX.1 Fill, CUDA graphs on;
(c) a 28-step Euler denoise at that shape: FLUX.1-dev text-to-image and FLUX.1 Fill at denoise 1.0 (which adds the
    img2img encode of the source and (a)).
Arms alternate --rounds times in one process; host clock around calls that end in a device synchronise; best of the
rounds.  Prints the card, its power limit and SM clock read in the same run, and fails when there is no GPU.
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

LAT, T = 128, 512


def _timed(fn, sync):
    sync()
    t0 = time.perf_counter()
    fn()
    sync()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=28)
    ap.add_argument("--forwards", type=int, default=10)
    args = ap.parse_args()
    import numpy as np
    import torch

    import diffusionkit_b200 as dk
    from diffusionkit_b200 import fill

    if not torch.cuda.is_available():
        raise SystemExit("bench_fill.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    sync = torch.cuda.synchronize
    pipes = {"dev": dk.FluxPipeline(w16=True, a16=True, model_version="argmaxinc/mlx-FLUX.1-dev",
                                    mmdit_config=dk.FLUX_DEV, device=dev, load_decoder=False),
             "fill": dk.FluxPipeline(w16=True, a16=True, model_version="black-forest-labs/FLUX.1-Fill-dev",
                                     device=dev, load_decoder=False, load_encoder=True)}
    cond, pooled = [t.to(dev) for t in pipes["dev"].synthetic_text_embeddings(n_images=1, text_len=T)]
    side = 8 * LAT
    rng = np.random.RandomState(0)
    img = rng.randint(0, 256, (side, side, 3)).astype(np.uint8)
    mask = np.zeros((side, side), dtype=np.uint8)
    mask[:, side // 2:] = 1
    fp, lf = pipes["fill"], pipes["fill"].latent_format
    src, m = torch.from_numpy(img)[None].to(dev), torch.from_numpy(mask).to(dev)

    def build():
        rows = fill.conditioning_rows(fp.encoder, src, m, lf.shift_factor, lf.scale_factor, fp.activation_dtype)
        fp.mmdit.cache_fill_conditioning(rows)

    latent = torch.randn((1, LAT, LAT, 16), device=dev).to(torch.bfloat16)
    for p in pipes.values():
        p.mmdit.cache_modulation_params(pooled, [500.0], [3.5])
    build()

    def forwards(p):
        for _ in range(args.forwards):
            p.mmdit(latent, cond, timestep=500.0)

    kw = dict(num_steps=args.steps, seed=0, solver="euler")
    arms = {"dev": lambda: pipes["dev"].denoise_latents(cond, pooled, latent_size=(LAT, LAT), **kw),
            "fill": lambda: fp.denoise_latents(cond, pooled, image_path=img, mask_image=mask * 255, **kw)}
    for p in pipes.values():
        forwards(p)                                                            # capture the forward graphs
    for a in arms.values():
        a()
    res = {"build_s": [], "forward_ms": {"dev": [], "fill": []}, "denoise_s": {"dev": [], "fill": []}}
    for _ in range(args.rounds):
        res["build_s"].append(_timed(build, sync))
        for name, p in pipes.items():
            p.mmdit.cache_modulation_params(pooled, [500.0], [3.5])
            res["forward_ms"][name].append(_timed(lambda: forwards(p), sync) * 1e3 / args.forwards)
        for name, a in arms.items():
            res["denoise_s"][name].append(_timed(a, sync))
    best = {"build_s": round(min(res["build_s"]), 4),
            "forward_ms": {k: round(min(v), 2) for k, v in res["forward_ms"].items()},
            "denoise_s": {k: round(min(v), 3) for k, v in res["denoise_s"].items()}}
    print(json.dumps({"best": best, "all": res, "rounds": args.rounds, "steps": args.steps, **card_info()}), flush=True)


if __name__ == "__main__":
    main()
