#!/usr/bin/env python
"""The Heun and DPM-Solver++(2M) samplers at the C3 shape (SD3-medium, CFG 5, 4 x 1024^2) and the C5 shape
(FLUX.1-dev config, 1 x 1024^2, text length 512), synthetic weights:

  python tools/bench_solvers.py [--launches 200] [--steps 20] [--rounds 2] [--only C5|C3]

(a) each sampler step kernel, dk_sampler_step beside the new ones: --launches launches captured in a CUDA graph, its
    replay timed with CUDA events.  The launches rotate over enough buffer sets to cover 256 MB, so the data comes
    from HBM and not from the 50 MB L2.
    Reported with the bytes the kernel must move, its GB/s and that rate over the 3.35 TB/s of the H100 SXM data sheet.
(b) C5 only: a --steps denoise (no decode) with each solver, alternated --rounds times; host clock around calls that
    end in a device synchronise.  Heun spends 2 * steps - 1 forwards, the others `steps`.
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

HBM_BYTES_PER_S = 3.35e12
ROTATE_BYTES = 256 << 20
SHAPES = {  # name: (pipeline, model version, latent, cfg weight, shift, images, text length)
    "C5": ("FluxPipeline", "argmaxinc/mlx-FLUX.1-dev", 128, 0.0, 1.0, 1, 512),
    "C3": ("DiffusionPipeline", "argmaxinc/mlx-stable-diffusion-3-medium", 128, 5.0, 3.0, 4, 589),
}


def kernel_bytes(kernel: str, n: int, reps: int) -> int:
    """bytes a step kernel must move for n fp32 state elements: fp32 vectors read or written, plus the 16-bit model
    input and output of reps * n elements each (read)"""
    fp32_vectors = {"step": 2,                  # x read, x written
                    "heun_predict": 3,          # x read, d and x2 written
                    "heun_correct": 4,          # x, d, x2 read, x written
                    "dpmpp_2m": 4}[kernel]      # x, d_prev read (c != 0), both written
    return fp32_vectors * 4 * n + 2 * 2 * reps * n


def bench_kernels(name, args, dev):
    import torch

    from diffusionkit_b200 import ops

    _, _, lat, cfgw, _, n_img, _ = SHAPES[name]
    dt = torch.float16 if name == "C3" else torch.bfloat16
    reps = 2 if cfgw > 0 else 1
    n = n_img * lat * lat * 16
    per_set = kernel_bytes("dpmpp_2m", n, reps) + 8 * n      # every buffer a set holds
    sets = []
    for _ in range(max(2, -(-ROTATE_BYTES // per_set))):
        sets.append({"x": torch.randn((n,), device=dev), "d": torch.randn((n,), device=dev),
                     "x2": torch.randn((n,), device=dev), "xin": torch.randn((reps * n,), device=dev).to(dt),
                     "out": torch.randn((reps * n,), device=dev).to(dt)})
    sigma, sigma_next = 0.5, 0.45
    launch = {
        "step": lambda s: ops.sampler_step(s["x"], s["xin"], s["out"], sigma, sigma_next, cfgw),
        "heun_predict": lambda s: ops.sampler_heun_predict(s["x"], s["xin"], s["out"], sigma, sigma_next, cfgw,
                                                           s["d"], s["x2"]),
        "heun_correct": lambda s: ops.sampler_heun_correct(s["x"], s["d"], s["x2"], s["xin"], s["out"], sigma,
                                                           sigma_next, cfgw),
        "dpmpp_2m": lambda s: ops.sampler_dpmpp_2m(s["x"], s["d"], s["xin"], s["out"], sigma, 0.9, 0.15, -0.05, cfgw),
    }
    res = {"n_state": n, "rotating_sets": len(sets), "dtype": str(dt).replace("torch.", "")}
    for kernel, fn in launch.items():
        for s in sets:                                    # warm-up
            fn(s)
        # one launch through ctypes takes longer on the host than these kernels take on the device, so the launches
        # are captured into a CUDA graph and the replay is timed
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for i in range(args.launches):
                fn(sets[i % len(sets)])
        graph.replay()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        graph.replay()
        end.record()
        torch.cuda.synchronize()
        del graph
        us = start.elapsed_time(end) * 1e3 / args.launches
        nbytes = kernel_bytes(kernel, n, reps)
        gbs = nbytes / (us * 1e-6) / 1e9
        res[kernel] = {"us": round(us, 2), "bytes": nbytes, "GB_s": round(gbs, 1),
                       "of_3350_GB_s": round(gbs * 1e9 / HBM_BYTES_PER_S, 3)}
    print(name, "kernels", json.dumps(res), flush=True)
    del sets
    torch.cuda.empty_cache()
    return res


def bench_denoise(name, args, dev):
    import torch

    import diffusionkit_b200 as dk

    cls, mv, lat, cfgw, shift, n_img, T = SHAPES[name]
    pipe = getattr(dk, cls)(w16=True, a16=True, shift=shift, model_version=mv, device=dev, load_decoder=False)
    cond, pooled = [t.to(dev) for t in pipe.synthetic_text_embeddings(n_images=n_img, text_len=T)]
    kw = dict(num_steps=args.steps, cfg_weight=cfgw, latent_size=(lat, lat), seed=list(range(n_img)))
    solvers = ("euler", "heun", "dpmpp_2m")
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
    nfe = {"euler": args.steps, "heun": 2 * args.steps - 1, "dpmpp_2m": args.steps}
    out = {"steps": args.steps, "denoise_s": {s: [round(v, 3) for v in vs] for s, vs in den.items()}, "nfe": nfe,
           "s_per_forward": {s: round(min(den[s]) / nfe[s], 4) for s in solvers}}
    print(name, "denoise", json.dumps(out), flush=True)
    del pipe
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--only", choices=sorted(SHAPES))
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_solvers.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    out = {}
    for name in SHAPES:
        if args.only in (None, name):
            out[name] = {"kernels": bench_kernels(name, args, dev)}
            if name == "C5":
                out[name]["denoise"] = bench_denoise(name, args, dev)
    print(json.dumps({**out, "launches": args.launches, "rounds": args.rounds, **card_info()}), flush=True)


if __name__ == "__main__":
    main()
