#!/usr/bin/env python
"""The first-block step cache at the C5 shape (FLUX.1-dev config, 1024^2, text length 512, 1 image) and the C3 shape
(SD3-medium, CFG 5, 4 images, text length 589), synthetic weights, arms alternated --rounds times in one process:

  python tools/bench_step_cache.py [--rounds 3] [--forwards 10] [--steps 50] [--only C5|C3]

(a) full-step time, cache off against cache on at threshold 0 (never skips): what the split, the reduction and the
    stream synchronise per step cost;
(b) skipped-step time (threshold inf after one full step);
(c) a --steps denoise (sample_euler, no decode) with threshold inf and max_consecutive_skips 1 and 2 (fixed skip
    patterns) against the cache off.
Host clock around work that ends in a device synchronise; prints the card, its power limit and SM clock read in the
same run, and fails when there is no GPU.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_gemm import card_info  # noqa: E402

SHAPES = {  # name: (pipeline, model version, latent, cfg weight, shift, images, text length)
    "C5": ("FluxPipeline", "argmaxinc/mlx-FLUX.1-dev", 128, 0.0, 1.0, 1, 512),
    "C3": ("DiffusionPipeline", "argmaxinc/mlx-stable-diffusion-3-medium", 128, 5.0, 3.0, 4, 589),
}


def wall(fn, n):
    import torch

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n


def bench_shape(name, args, dev):
    import torch

    import diffusionkit_b200 as dk

    cls, mv, lat, cfgw, shift, n_img, T = SHAPES[name]
    pipe = getattr(dk, cls)(w16=True, a16=True, shift=shift, model_version=mv, device=dev, load_decoder=False)
    m = pipe.mmdit
    cond, pooled = [t.to(dev) for t in pipe.synthetic_text_embeddings(n_images=n_img, text_len=T)]
    reps = 2 if cfgw > 0 else 1
    latent = torch.randn((reps * n_img, lat, lat, 16), device=dev).to(pipe.activation_dtype)

    def forward():
        m(latent, cond, timestep=500.0)

    def modes(threshold, cap=None):
        pipe.set_step_cache(threshold, cap)
        m.cache_modulation_params(pooled, [500.0])

    res = {"full_ms_cache_off": [], "full_ms_threshold0": [], "skipped_ms": []}
    for _ in range(args.rounds):
        modes(None)
        wall(forward, 2)
        res["full_ms_cache_off"].append(wall(forward, args.forwards) * 1e3)
        modes(0.0)
        wall(forward, 2)
        res["full_ms_threshold0"].append(wall(forward, args.forwards) * 1e3)
        modes(math.inf)
        forward()                                           # the full first step
        wall(forward, 2)
        res["skipped_ms"].append(wall(forward, args.forwards) * 1e3)
        assert all(s for _, s in m.step_cache_log[1:])
    den = {"off": [], "cap1": [], "cap2": []}
    patterns = {}
    for _ in range(args.rounds):
        for arm, (thr, cap) in {"off": (None, None), "cap1": (math.inf, 1), "cap2": (math.inf, 2)}.items():
            pipe.set_step_cache(thr, cap)
            t0 = time.perf_counter()
            pipe.denoise_latents(cond, pooled, num_steps=args.steps, cfg_weight=cfgw, latent_size=(lat, lat),
                                 seed=list(range(n_img)))
            torch.cuda.synchronize()
            den[arm].append(time.perf_counter() - t0)
            if thr is not None:
                patterns[arm] = sum(s for _, s in m.step_cache_log)
    pipe.set_step_cache(None)
    out = {k: [round(v, 2) for v in vs] for k, vs in res.items()}
    off, t0 = min(res["full_ms_cache_off"]), min(res["full_ms_threshold0"])
    out.update({"threshold0_overhead_pct": round(100.0 * (t0 - off) / off, 2),
                "skipped_over_full": round(min(res["skipped_ms"]) / off, 4),
                "denoise_s": {k: [round(v, 3) for v in vs] for k, vs in den.items()},
                "skipped_steps": patterns, "steps": args.steps,
                "denoise_speedup": {k: round(min(den["off"]) / min(den[k]), 3) for k in ("cap1", "cap2")}})
    print(name, json.dumps(out), flush=True)
    del pipe, m
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--forwards", type=int, default=10)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--only", choices=sorted(SHAPES))
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_step_cache.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    out = {name: bench_shape(name, args, dev) for name in SHAPES if args.only in (None, name)}
    print(json.dumps({**out, "rounds": args.rounds, "forwards": args.forwards, **card_info()}), flush=True)


if __name__ == "__main__":
    main()
