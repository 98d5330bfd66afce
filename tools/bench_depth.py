#!/usr/bin/env python
"""FLUX.1 Depth [dev] with its depth estimator (DESIGN.md §20), synthetic weights, one H100:

  python tools/bench_depth.py [--rounds 3] [--steps 28]

(a) the estimator (Depth Anything large, bf16) at a 1024^2 and a 1024 wide x 768 high control image: the host round
    trip and resize, the 518^2 / 518 x 686 network, the antialiased bicubic back to the image size;
(b) the conditioning build of one 1024^2 control image: the depth map as given (VAE encoder, posterior mean, packing,
    K = 64 GEMM), and with the estimator in front (estimate_depth);
(c) a 28-step Euler FLUX.1 Depth denoise at 1024^2 (T = 512, one image) with a depth map, and with a photo through
    the estimator.
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


def _photo(h, w, rng):
    """a smooth picture with a few objects: low-frequency colour fields and blurred blocks"""
    import numpy as np
    from scipy import ndimage

    blocks = np.kron(rng.randint(0, 256, (h // 64, w // 64, 3)), np.ones((64, 64, 1))).astype(np.float32)
    return ndimage.gaussian_filter(blocks + rng.randn(h, w, 3) * 6, (4, 4, 0)).clip(0, 255).astype(np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=28)
    args = ap.parse_args()
    import numpy as np
    import torch

    import diffusionkit_b200 as dk
    from diffusionkit_b200 import control

    if not torch.cuda.is_available():
        raise SystemExit("bench_depth.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    sync = torch.cuda.synchronize
    rng = np.random.RandomState(0)
    photos = {"1024x1024": _photo(1024, 1024, rng), "1024x768": _photo(768, 1024, rng)}
    pipe = dk.FluxPipeline(w16=True, a16=True, model_version="black-forest-labs/FLUX.1-Depth-dev", device=dev,
                           load_decoder=False, load_encoder=True)
    pipe.load_depth_estimator()
    cond, pooled = [t.to(dev) for t in pipe.synthetic_text_embeddings(n_images=1, text_len=T)]
    lf = pipe.latent_format
    photo = photos["1024x1024"]
    depth_map = pipe.estimate_depth(photo)
    depth_u8 = depth_map.clamp(0, 255).to(torch.uint8)[..., None].expand(-1, -1, 3).contiguous()

    def build(estimate):
        img = pipe._depth_image(photo, rgb=True) if estimate else depth_u8
        rows = control.control_rows(pipe.encoder, img, "depth", lf.shift_factor, lf.scale_factor,
                                    pipe.activation_dtype)
        pipe.mmdit.cache_fill_conditioning(rows)

    kw = dict(num_steps=args.steps, seed=0, solver="euler", latent_size=(LAT, LAT))
    arms = {"depth_map": lambda: pipe.denoise_latents(cond, pooled, control_image=depth_u8.cpu().numpy(), **kw),
            "estimate_depth": lambda: pipe.denoise_latents(cond, pooled, control_image=photo, estimate_depth=True,
                                                           **kw)}
    for p in photos.values():
        pipe.estimate_depth(p)
    for e in (False, True):
        build(e)
    for a in arms.values():
        a()
    res = {"estimator_ms": {k: [] for k in photos}, "build_ms": {"depth_map": [], "estimate_depth": []},
           "denoise_s": {k: [] for k in arms}}
    for _ in range(args.rounds):
        for k, p in photos.items():
            res["estimator_ms"][k].append(_timed(lambda: pipe.estimate_depth(p), sync) * 1e3)
        for name, e in (("depth_map", False), ("estimate_depth", True)):
            res["build_ms"][name].append(_timed(lambda: build(e), sync) * 1e3)
        for name, a in arms.items():
            res["denoise_s"][name].append(_timed(a, sync))
    best = {g: {k: round(min(v), 3) for k, v in d.items()} for g, d in res.items()}
    print(json.dumps({"best": best, "all": res, "rounds": args.rounds, "steps": args.steps,
                      "network_input": {k: dk.depth.network_size(*p.shape[:2]) for k, p in photos.items()},
                      **card_info()}), flush=True)


if __name__ == "__main__":
    main()
