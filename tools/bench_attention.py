#!/usr/bin/env python
"""Times the joint attention forward (dk_attention_fwd) at the shapes of the benchmark workloads.

  python tools/bench_attention.py [--iters 30] [--warmup 5] [--dump DIR] [--only NAME ...]
  python tools/bench_attention.py --compare DIR_A DIR_B

Inputs are seeded, so with --dump DIR the output of one launch is written per shape as DIR/<name>.npy (raw 16-bit
words, text rows then image rows), and --compare reports, per shape, how many 16-bit words differ between two such
directories and by how many ulp at most.  Timing: CUDA events around --iters back-to-back launches after --warmup
launches; TFLOP/s counts the two matrix products, 4 * B * S^2 * heads * d.  The JSON line names the card, its power
limit and the SM clock read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from bench_gemm import card_info  # noqa: E402

# name: (B, S, heads, d, dtype, split = rows that go to the first output), the attention of bench.py's workloads:
# C4: FLUX.1-schnell 1024^2, 4 images (256 text + 4096 image tokens); C5: FLUX.1-dev 1024^2, 1 image, 512 text tokens;
# C3: SD3 1024^2, 4 images with classifier-free guidance, so batch 8 (4096 image + 589 text tokens, image first).
SHAPES = {
    "C4": (4, 4352, 24, 128, "bfloat16", 256),
    "C5": (1, 4608, 24, 128, "bfloat16", 512),
    "C3": (8, 4685, 24, 64, "float16", 4096),
}


def make_case(name, dev):
    """seeded packed q | k | v and a closure that runs the attention once"""
    import torch

    from diffusionkit_b200 import ops

    B, S, heads, d, dt, split = SHAPES[name]
    dtype = getattr(torch, dt)
    g = torch.Generator(device=dev).manual_seed(sum(map(ord, name)))
    qkv = (torch.randn((B * S, 3 * heads * d), generator=g, device=dev) * 2.0).to(dtype)
    out0 = torch.empty((B * split, heads * d), dtype=dtype, device=dev)
    out1 = torch.empty((B * (S - split), heads * d), dtype=dtype, device=dev)
    return (out0, out1), lambda: ops.attention(qkv, B, S, heads, d, out0, split=split, out1=out1)


def run(args):
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_attention.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
    rows = {}
    for name in args.only or list(SHAPES):
        B, S, heads, d, dt, split = SHAPES[name]
        outs, launch = make_case(name, dev)
        launch()
        torch.cuda.synchronize()
        if args.dump:
            words = torch.cat([o.view(torch.int16).flatten() for o in outs]).cpu().numpy()
            np.save(os.path.join(args.dump, f"{name}.npy"), words)
        for _ in range(args.warmup):
            launch()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            launch()
        e1.record()
        torch.cuda.synchronize()
        sec = e0.elapsed_time(e1) / 1e3 / args.iters
        flop = 4.0 * B * S * S * heads * d
        rows[name] = {"B": B, "S": S, "heads": heads, "d": d, "dtype": dt, "split": split,
                      "us": round(sec * 1e6, 1), "tflops": round(flop / sec / 1e12, 1)}
        print(f"{name}  B {B}  S {S}  {heads} x {d}  {dt:8s} {sec * 1e6:9.1f} us  {flop / sec / 1e12:6.1f} TFLOP/s",
              flush=True)
        del outs, launch
        torch.cuda.empty_cache()
    print(json.dumps({"shapes": rows, "iters": args.iters, **card_info()}), flush=True)


def compare(dir_a, dir_b):
    """per shape: 16-bit words that differ, and the largest difference in ulp (bit patterns as ordered ints).  A shape
    dumped in only one directory fails the comparison, and so do two directories with no shape in common."""
    ok, compared = True, 0
    for name in SHAPES:
        pa, pb = os.path.join(dir_a, f"{name}.npy"), os.path.join(dir_b, f"{name}.npy")
        if not (os.path.exists(pa) or os.path.exists(pb)):
            continue
        if not (os.path.exists(pa) and os.path.exists(pb)):
            ok = False
            print(json.dumps({"shape": name, "missing": pb if os.path.exists(pa) else pa}), flush=True)
            continue
        compared += 1
        a, b = np.load(pa).astype(np.int32), np.load(pb).astype(np.int32)
        if a.shape != b.shape:
            ok = False
            print(json.dumps({"shape": name, "elements": [int(a.size), int(b.size)]}), flush=True)
            continue
        # sign-magnitude -> ordered integers, so that neighbouring floats differ by 1
        a = np.where(a < 0, -32768 - a, a)
        b = np.where(b < 0, -32768 - b, b)
        diff = np.abs(a - b)
        n = int((diff != 0).sum())
        ok &= n == 0
        print(json.dumps({"shape": name, "elements": int(a.size), "differ": n, "max_ulp": int(diff.max())}), flush=True)
    if compared == 0:
        print(json.dumps({"compared": 0, "dirs": [dir_a, dir_b]}), flush=True)
    return ok and compared > 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--dump", metavar="DIR", default=None)
    ap.add_argument("--only", nargs="*", choices=sorted(SHAPES))
    ap.add_argument("--compare", nargs=2, metavar=("DIR_A", "DIR_B"))
    args = ap.parse_args()
    if args.compare:
        sys.exit(0 if compare(*args.compare) else 1)
    run(args)


if __name__ == "__main__":
    main()
