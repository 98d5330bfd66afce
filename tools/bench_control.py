#!/usr/bin/env python
"""FLUX.1 Canny / Depth [dev] (DESIGN.md §19), synthetic weights, one H100:

  python tools/bench_control.py [--rounds 3] [--steps 28]

(a) dk_canny (five launches) on a 3-channel image at 1024^2 and 2048^2, CUDA events over --reps calls;
(b) the conditioning build of one 1024^2 control image on Canny: dk_canny, the VAE encoder, the posterior mean, the
    packing and the K = 64 GEMM (cache_fill_conditioning);
(c) one MMDiT forward at the C5 shape (1024^2, T = 512, one image) on FLUX.1-dev and on FLUX.1 Canny, CUDA graphs on,
    the two models alternated;
(d) a 28-step Euler denoise at that shape: FLUX.1-dev text-to-image and FLUX.1 Canny text-to-image with a control
    image (which adds (b)).
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


def _image(side, rng):
    """a 3-channel test image with edges at every scale: blurred random blocks"""
    import numpy as np
    from scipy import ndimage

    blocks = np.kron(rng.randint(0, 256, (side // 32, side // 32, 3)), np.ones((32, 32, 1))).astype(np.float32)
    return ndimage.gaussian_filter(blocks + rng.randn(side, side, 3) * 8, (1.5, 1.5, 0)).clip(0, 255).astype(np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=28)
    ap.add_argument("--forwards", type=int, default=10)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import numpy as np
    import torch

    import diffusionkit_b200 as dk
    from diffusionkit_b200 import control

    if not torch.cuda.is_available():
        raise SystemExit("bench_control.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    sync = torch.cuda.synchronize
    rng = np.random.RandomState(0)
    imgs = {s: torch.from_numpy(_image(s, rng)).to(dev) for s in (1024, 2048)}

    def canny_us(img):
        control.canny(img)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            control.canny(img)
        e1.record()
        sync()
        return e0.elapsed_time(e1) * 1e3 / args.reps

    pipes = {"dev": dk.FluxPipeline(w16=True, a16=True, model_version="argmaxinc/mlx-FLUX.1-dev",
                                    mmdit_config=dk.FLUX_DEV, device=dev, load_decoder=False),
             "canny": dk.FluxPipeline(w16=True, a16=True, model_version="black-forest-labs/FLUX.1-Canny-dev",
                                      device=dev, load_decoder=False, load_encoder=True)}
    cond, pooled = [t.to(dev) for t in pipes["dev"].synthetic_text_embeddings(n_images=1, text_len=T)]
    cp, lf = pipes["canny"], pipes["canny"].latent_format
    ctl = imgs[8 * LAT]

    def build():
        rows = control.control_rows(cp.encoder, ctl, "canny", lf.shift_factor, lf.scale_factor, cp.activation_dtype)
        cp.mmdit.cache_fill_conditioning(rows)

    latent = torch.randn((1, LAT, LAT, 16), device=dev).to(torch.bfloat16)
    for p in pipes.values():
        p.mmdit.cache_modulation_params(pooled, [500.0], [3.5])
    build()

    def forwards(p):
        for _ in range(args.forwards):
            p.mmdit(latent, cond, timestep=500.0)

    ctl_host = ctl.cpu().numpy()
    kw = dict(num_steps=args.steps, seed=0, solver="euler", latent_size=(LAT, LAT))
    arms = {"dev": lambda: pipes["dev"].denoise_latents(cond, pooled, **kw),
            "canny": lambda: cp.denoise_latents(cond, pooled, control_image=ctl_host, **kw)}
    for p in pipes.values():
        forwards(p)                                                            # capture the forward graphs
    for a in arms.values():
        a()
    res = {"canny_us": {str(s): [] for s in imgs}, "build_s": [], "forward_ms": {"dev": [], "canny": []},
           "denoise_s": {"dev": [], "canny": []}}
    for _ in range(args.rounds):
        for s, img in imgs.items():
            res["canny_us"][str(s)].append(canny_us(img))
        res["build_s"].append(_timed(build, sync))
        for name, p in pipes.items():
            p.mmdit.cache_modulation_params(pooled, [500.0], [3.5])
            res["forward_ms"][name].append(_timed(lambda: forwards(p), sync) * 1e3 / args.forwards)
        for name, a in arms.items():
            res["denoise_s"][name].append(_timed(a, sync))
    best = {"canny_us": {k: round(min(v), 1) for k, v in res["canny_us"].items()},
            "build_s": round(min(res["build_s"]), 4),
            "forward_ms": {k: round(min(v), 2) for k, v in res["forward_ms"].items()},
            "denoise_s": {k: round(min(v), 3) for k, v in res["denoise_s"].items()}}
    print(json.dumps({"best": best, "all": res, "rounds": args.rounds, "steps": args.steps, **card_info()}), flush=True)


if __name__ == "__main__":
    main()
