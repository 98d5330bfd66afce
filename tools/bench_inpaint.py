#!/usr/bin/env python
"""Masked inpainting (DESIGN.md §17), synthetic weights:

  python tools/bench_inpaint.py [--launches 200] [--rounds 3] [--only C5|C3]

(a) dk_inpaint_blend at the C3/C4 latent shape (4, 128, 128, 16) with nothing repainted (the most bytes) and with
    half of it repainted, and dk_inpaint_paste at 4 x 1024^2 with half of it kept: --launches launches captured in a
    CUDA graph, its replay timed with CUDA events, over enough buffer sets to cover 256 MB (so the data comes from HBM,
    not the 50 MB L2).  Reported with the bytes each must move (from the shape), its GB/s and that rate over the
    3.35 TB/s of the H100 SXM data sheet.
(b) an img2img denoise from a 1024^2 image at denoise 1.0 (no decode) without and with a half-image mask, alternated
    --rounds times in one process: 28 FLUX.1-dev Euler steps at the C5 shape and 20 SD3 DPM-Solver++(2M) steps at the
    C3 shape (CFG 5, 4 images); host clock around calls that end in a device synchronise.
Prints the card, its power limit and SM clock read in the same run, and fails when there is no GPU.
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
from tools.bench_solvers import HBM_BYTES_PER_S, ROTATE_BYTES, SHAPES  # noqa: E402

DENOISE = {"C5": ("euler", 28), "C3": ("dpmpp_2m", 20)}


def blend_bytes(B, HW, C, kept):
    """eps and x0 read and x written at the kept positions (fp32), and the mask read once (the B images share it, and
    its HW bytes stay in L2)"""
    return 3 * 4 * B * kept * C + HW


def paste_bytes(B, P, kept):
    """the image written at the kept pixels (3 bytes each), and the source at those pixels and the mask read once (the
    B images share both, and they stay in L2)"""
    return 3 * B * kept + 3 * kept + P


def _timed(graphs, rounds, launches):
    import torch

    times = {k: [] for k in graphs}
    for _ in range(rounds):
        for k, g in graphs.items():
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            start.record()
            g.replay()
            end.record()
            torch.cuda.synchronize()
            times[k].append(start.elapsed_time(end) * 1e3 / launches)
    return times


def _capture(fn, sets, launches):
    import torch

    for i, s in enumerate(sets):
        fn(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(launches):
            fn(sets[i % len(sets)])
    g.replay()
    return g


def bench_kernels(args, dev):
    import torch

    from diffusionkit_b200.inpaint import inpaint_blend, inpaint_paste

    B, H, W, C = 4, 128, 128, 16
    none = torch.zeros((H, W), dtype=torch.uint8, device=dev)
    half = torch.zeros((H, W), dtype=torch.uint8, device=dev)
    half[:, W // 2:] = 1
    per = blend_bytes(B, H * W, C, H * W)
    sets = [{k: torch.randn((B, H, W, C), device=dev) for k in ("x", "eps", "x0")}
            for _ in range(max(2, -(-ROTATE_BYTES // per)))]
    graphs = {"blend_none_repainted": _capture(lambda s: inpaint_blend(s["x"], s["eps"], s["x0"], none, 0.4, 0.6),
                                               sets, args.launches),
              "blend_half_repainted": _capture(lambda s: inpaint_blend(s["x"], s["eps"], s["x0"], half, 0.4, 0.6),
                                               sets, args.launches)}
    nbytes = {"blend_none_repainted": per, "blend_half_repainted": blend_bytes(B, H * W, C, H * W // 2)}
    Bp, Hp, Wp = 4, 1024, 1024
    pm = torch.zeros((Hp, Wp), dtype=torch.uint8, device=dev)
    pm[:, Wp // 2:] = 1
    per_p = 3 * Bp * Hp * Wp + 3 * Hp * Wp                     # the buffers of one set
    psets = [{"img": torch.randint(0, 256, (Bp, Hp, Wp, 3), dtype=torch.uint8, device=dev),
              "src": torch.randint(0, 256, (Hp, Wp, 3), dtype=torch.uint8, device=dev)}
             for _ in range(max(2, -(-ROTATE_BYTES // per_p)))]
    graphs["paste_half_kept"] = _capture(lambda s: inpaint_paste(s["img"], s["src"], pm), psets, args.launches)
    nbytes["paste_half_kept"] = paste_bytes(Bp, Hp * Wp, Hp * Wp // 2)
    res = {"blend_shape": [B, H, W, C], "paste_shape": [Bp, Hp, Wp, 3], "rotating_sets": [len(sets), len(psets)]}
    for k, ts in _timed(graphs, args.rounds, args.launches).items():
        us = min(ts)
        gbs = nbytes[k] / (us * 1e-6) / 1e9
        res[k] = {"us": [round(t, 2) for t in ts], "best_us": round(us, 2), "bytes": nbytes[k],
                  "GB_s": round(gbs, 1), "of_3350_GB_s": round(gbs * 1e9 / HBM_BYTES_PER_S, 3),
                  "us_at_3350_GB_s": round(nbytes[k] / HBM_BYTES_PER_S * 1e6, 2)}
    print("kernels", json.dumps(res), flush=True)
    del graphs, sets, psets
    torch.cuda.empty_cache()
    return res


def bench_denoise(name, args, dev):
    import numpy as np
    import torch

    import diffusionkit_b200 as dk

    cls, mv, lat, cfgw, shift, n_img, T = SHAPES[name]
    solver, steps = DENOISE[name]
    pipe = getattr(dk, cls)(w16=True, a16=True, shift=shift, model_version=mv, device=dev, load_decoder=False,
                            load_encoder=True)
    cond, pooled = [t.to(dev) for t in pipe.synthetic_text_embeddings(n_images=n_img, text_len=T)]
    side = 8 * lat
    rng = np.random.RandomState(0)
    img = rng.randint(0, 256, (side, side, 3)).astype(np.uint8)
    mask = np.zeros((side, side), dtype=np.uint8)
    mask[:, side // 2:] = 255
    kw = dict(cfg_weight=cfgw, seed=list(range(n_img)), image_path=img, denoise=1.0, solver=solver)
    pipe.denoise_latents(cond, pooled, num_steps=2, **kw)                      # capture the forward's graph
    arms = {"img2img": {}, "half_mask": {"mask_image": mask}}
    den = {a: [] for a in arms}
    for _ in range(args.rounds):
        for a, extra in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            lat_out, _ = pipe.denoise_latents(cond, pooled, num_steps=steps, **kw, **extra)
            torch.cuda.synchronize()
            den[a].append(time.perf_counter() - t0)
            assert bool(torch.isfinite(lat_out).all())
    out = {"solver": solver, "steps": steps, "images": n_img, "denoise_s": {a: [round(v, 3) for v in vs]
                                                                            for a, vs in den.items()},
           "best_s": {a: round(min(vs), 3) for a, vs in den.items()}}
    print(name, "denoise", json.dumps(out), flush=True)
    del pipe
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--only", choices=sorted(SHAPES))
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_inpaint.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    out = {"kernels": bench_kernels(args, dev)}
    for name in SHAPES:
        if args.only in (None, name):
            out[name] = bench_denoise(name, args, dev)
    print(json.dumps({**out, "launches": args.launches, "rounds": args.rounds, **card_info()}), flush=True)


if __name__ == "__main__":
    main()
