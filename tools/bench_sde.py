#!/usr/bin/env python
"""The stochastic samplers (DESIGN.md §16) at the C3 shape (SD3-medium, CFG 5, 4 x 1024^2) and the C5 shape
(FLUX.1-dev config, 1 x 1024^2, text length 512), synthetic weights:

  python tools/bench_sde.py [--launches 200] [--steps 20] [--rounds 3] [--only C5|C3]

(a) dk_sampler_sde_step against dk_sampler_dpmpp_2m, alternated --rounds times in one process: --launches launches
    captured in a CUDA graph, its replay timed with CUDA events, over enough buffer sets to cover 256 MB (so the data
    comes from HBM, not the 50 MB L2).  Arms: the 2M kernel (second-order step), the SDE kernel with that step plus
    noise (dpmpp_2m_sde), the SDE kernel with the same arithmetic and no noise, and Euler ancestral (no d_prev).
    Reported with the bytes each must move, its GB/s and that rate over the 3.35 TB/s of the H100 SXM data sheet.
(b) a --steps denoise (no decode) with dpmpp_2m, euler_ancestral and dpmpp_2m_sde, alternated --rounds times; host
    clock around calls that end in a device synchronise.
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


def kernel_bytes(arm: str, n: int, reps: int) -> int:
    """bytes an update must move for n fp32 state elements: x read and written, d_prev read (c != 0) and written
    where the solver keeps it, and the 16-bit model input and output of reps * n elements each"""
    fp32_vectors = 2 if arm == "euler_ancestral" else 4
    return fp32_vectors * 4 * n + 2 * 2 * reps * n


def bench_kernels(name, args, dev):
    import torch

    from diffusionkit_b200 import ops
    from diffusionkit_b200.pipeline import sampler_sde_step, seeds_tensor

    _, _, lat, cfgw, _, n_img, _ = SHAPES[name]
    dt = torch.float16 if name == "C3" else torch.bfloat16
    reps = 2 if cfgw > 0 else 1
    n = n_img * lat * lat * 16
    per_set = kernel_bytes("dpmpp_2m", n, reps)
    sets = []
    for _ in range(max(2, -(-ROTATE_BYTES // per_set))):
        sets.append({"x": torch.randn((n_img, n // n_img), device=dev), "d": torch.randn((n_img, n // n_img), device=dev),
                     "xin": torch.randn((reps * n,), device=dev).to(dt),
                     "out": torch.randn((reps * n,), device=dev).to(dt)})
    seeds = seeds_tensor(range(n_img), dev)
    sigma, a, b, c = 0.5, 0.9, 0.15, -0.05
    arms = {
        "dpmpp_2m": lambda s, i: ops.sampler_dpmpp_2m(s["x"], s["d"], s["xin"], s["out"], sigma, a, b, c, cfgw),
        "dpmpp_2m_sde": lambda s, i: sampler_sde_step(s["x"], s["d"], s["xin"], s["out"], sigma, a, b, c, 0.3, cfgw,
                                                      0.0, seeds, i),
        "sde_no_noise": lambda s, i: sampler_sde_step(s["x"], s["d"], s["xin"], s["out"], sigma, a, b, c, 0.0, cfgw,
                                                      0.0, seeds, i),
        "euler_ancestral": lambda s, i: sampler_sde_step(s["x"], None, s["xin"], s["out"], sigma, a, b, 0.0, 0.3,
                                                         cfgw, 0.0, seeds, i),
    }
    graphs = {}
    for arm, fn in arms.items():
        for i, s in enumerate(sets):                      # warm-up
            fn(s, i)
        # one launch through ctypes takes longer on the host than these kernels take on the device: the launches are
        # captured into a CUDA graph and the replay is timed
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for i in range(args.launches):
                fn(sets[i % len(sets)], i)
        g.replay()
        graphs[arm] = g
    times = {arm: [] for arm in arms}
    for _ in range(args.rounds):
        for arm, g in graphs.items():
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            start.record()
            g.replay()
            end.record()
            torch.cuda.synchronize()
            times[arm].append(start.elapsed_time(end) * 1e3 / args.launches)
    res = {"n_state": n, "reps": reps, "rotating_sets": len(sets), "dtype": str(dt).replace("torch.", "")}
    for arm, ts in times.items():
        us = min(ts)
        nbytes = kernel_bytes(arm, n, reps)
        gbs = nbytes / (us * 1e-6) / 1e9
        res[arm] = {"us": [round(t, 2) for t in ts], "best_us": round(us, 2), "bytes": nbytes, "GB_s": round(gbs, 1),
                    "of_3350_GB_s": round(gbs * 1e9 / HBM_BYTES_PER_S, 3)}
    print(name, "kernels", json.dumps(res), flush=True)
    del graphs, sets
    torch.cuda.empty_cache()
    return res


def bench_denoise(name, args, dev):
    import torch

    import diffusionkit_b200 as dk

    cls, mv, lat, cfgw, shift, n_img, T = SHAPES[name]
    pipe = getattr(dk, cls)(w16=True, a16=True, shift=shift, model_version=mv, device=dev, load_decoder=False)
    cond, pooled = [t.to(dev) for t in pipe.synthetic_text_embeddings(n_images=n_img, text_len=T)]
    kw = dict(num_steps=args.steps, cfg_weight=cfgw, latent_size=(lat, lat), seed=list(range(n_img)))
    solvers = ("dpmpp_2m", "euler_ancestral", "dpmpp_2m_sde")
    pipe.denoise_latents(cond, pooled, **{**kw, "num_steps": 2})                  # capture the forward's graph
    den = {s: [] for s in solvers}
    for _ in range(args.rounds):
        for s in solvers:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            lat_out, _ = pipe.denoise_latents(cond, pooled, solver=s, **kw)
            torch.cuda.synchronize()
            den[s].append(time.perf_counter() - t0)
            assert bool(torch.isfinite(lat_out).all())
    out = {"steps": args.steps, "denoise_s": {s: [round(v, 3) for v in vs] for s, vs in den.items()},
           "best_s": {s: round(min(vs), 3) for s, vs in den.items()}}
    print(name, "denoise", json.dumps(out), flush=True)
    del pipe
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--only", choices=sorted(SHAPES))
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_sde.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    out = {}
    for name in SHAPES:
        if args.only in (None, name):
            out[name] = {"kernels": bench_kernels(name, args, dev), "denoise": bench_denoise(name, args, dev)}
    print(json.dumps({**out, "launches": args.launches, "rounds": args.rounds, **card_info()}), flush=True)


if __name__ == "__main__":
    main()
