#!/usr/bin/env python
"""Times every MMDiT GEMM of the C4 workload (FLUX.1-schnell 1024^2, 4 images) through dk_gemm with its real epilogue.

  python tools/bench_gemm.py [--iters 50] [--warmup 10] [--dump DIR] [--only NAME ...]
  python tools/bench_gemm.py --compare DIR_A DIR_B

Each shape runs with the epilogue, row remap and in-place residual the model gives it.  Inputs are seeded, so with
--dump DIR the output of one launch on fresh inputs is written per shape as DIR/<name>.npy (raw 16-bit words), and
--compare reports, per shape, how many 16-bit words differ between two such directories and by how many ulp at most.
Timing: CUDA events around --iters back-to-back launches after --warmup launches.  The JSON line names the card, its
power limit and the SM clock read in the same run; the aggregate weights each shape by its launches per forward.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

B, H, HEADS, D = 4, 3072, 24, 128     # FLUX.1 width; C4 batch
S_IMG, S_TXT = 4096, 256              # 1024^2 latent -> 64 x 64 patches; text length
S = S_IMG + S_TXT                     # joint sequence, text first
DOUBLE, SINGLE = 19, 38               # blocks per forward

# name: (M, N, K, epilogue, launches per forward)
SHAPES = {
    "double_img_qkv": (B * S_IMG, 3 * H, H, "qk_img", DOUBLE),
    "double_img_o": (B * S_IMG, H, H, "gate_res_img", DOUBLE),
    "double_img_fc1": (B * S_IMG, 4 * H, H, "gelu", DOUBLE),
    "double_img_fc2": (B * S_IMG, H, 4 * H, "gate_res_img", DOUBLE),
    "double_txt_qkv": (B * S_TXT, 3 * H, H, "qk_txt", DOUBLE),
    "double_txt_o": (B * S_TXT, H, H, "gate_res_txt", DOUBLE),
    "double_txt_fc1": (B * S_TXT, 4 * H, H, "gelu", DOUBLE),
    "double_txt_fc2": (B * S_TXT, H, 4 * H, "gate_res_txt", DOUBLE),
    "single_qkv": (B * S, 3 * H, H, "qk_single", SINGLE),
    "single_fc1": (B * S, 4 * H, H, "gelu_cat", SINGLE),
    "single_out": (B * S, H, 5 * H, "gate_res_single", SINGLE),
}


def make_case(name, dev):
    """seeded inputs and a closure that runs the GEMM once and returns its output buffer"""
    import torch

    from diffusionkit_b200 import ops
    from diffusionkit_b200._lib import ACT_GELU_ERF

    M, N, K, epi, _ = SHAPES[name]
    g = torch.Generator(device=dev).manual_seed(sum(map(ord, name)))

    def rnd(shape, scale=1.0):
        return (torch.randn(shape, generator=g, device=dev) * scale).to(torch.bfloat16)

    A = rnd((M, K))
    W = rnd((N, K), 1.0 / math.sqrt(K))
    bias = rnd((N,), 0.5)
    if epi.startswith("qk"):
        rpb, obr, off = {"qk_img": (S_IMG, S, S_TXT), "qk_txt": (S_TXT, S, 0), "qk_single": (S, S, 0)}[epi]
        qw, kw = rnd((D,), 0.1) + 1.0, rnd((D,), 0.1) + 1.0
        ang = torch.rand((S, D // 2), generator=g, device=dev) * 6.28
        rope = torch.stack([torch.cos(ang), torch.sin(ang)], dim=-1).contiguous()
        out = torch.zeros((B * S, N), dtype=torch.bfloat16, device=dev)
        return out, lambda: ops.gemm(A, W, out=out, bias=bias, rows_per_batch=rpb, out_batch_rows=obr,
                                     out_row_off=off, qk=(HEADS, D, qw, kw, rope, 1e-6))
    if epi.startswith("gate_res"):
        rpb = {"gate_res_img": S_IMG, "gate_res_txt": S_TXT, "gate_res_single": S}[epi]
        x = rnd((M, N))
        gate = rnd((B, N), 0.1)
        return x, lambda: ops.gemm(A, W, out=x, bias=bias, gate=gate, res=x, rows_per_batch=rpb, out_batch_rows=rpb)
    if epi == "gelu_cat":
        cat = torch.zeros((M, 5 * H), dtype=torch.bfloat16, device=dev)   # [attention | gelu(fc1)]
        return cat, lambda: ops.gemm(A, W, out=cat[:, H:], bias=bias, act=ACT_GELU_ERF)
    out = torch.empty((M, N), dtype=torch.bfloat16, device=dev)
    return out, lambda: ops.gemm(A, W, out=out, bias=bias, act=ACT_GELU_ERF)


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        line = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm, sm_max = [p.strip() for p in line.split(",")]
        return {"card": name, "power_limit_w": float(power), "sm_mhz": float(sm), "sm_max_mhz": float(sm_max)}
    except Exception as ex:   # reported, not load-bearing
        return {"card": None, "nvidia_smi": f"failed: {ex!r}"}


def run(args):
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    names = args.only or list(SHAPES)
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
    rows, tot_flop, tot_s = {}, 0.0, 0.0
    for name in names:
        M, N, K, epi, per_fwd = SHAPES[name]
        out, launch = make_case(name, dev)
        launch()
        torch.cuda.synchronize()
        if args.dump:
            np.save(os.path.join(args.dump, f"{name}.npy"), out.view(torch.int16).cpu().numpy())
        for _ in range(args.warmup):
            launch()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            launch()
        e1.record()
        torch.cuda.synchronize()
        sec = e0.elapsed_time(e1) / 1e3 / args.iters
        flop = 2.0 * M * N * K
        rows[name] = {"M": M, "N": N, "K": K, "epilogue": epi, "us": round(sec * 1e6, 2),
                      "tflops": round(flop / sec / 1e12, 1)}
        tot_flop += per_fwd * flop
        tot_s += per_fwd * sec
        print(f"{name:16s} {M:6d} x {N:5d} x {K:5d}  {epi:16s} {sec * 1e6:9.1f} us  {flop / sec / 1e12:6.1f} TFLOP/s",
              flush=True)
        del out, launch
        torch.cuda.empty_cache()
    info = card_info()
    print(json.dumps({"shapes": rows, "aggregate_tflops": round(tot_flop / tot_s / 1e12, 1),
                      "gemm_seconds_per_forward": round(tot_s, 4), "iters": args.iters, **info}), flush=True)


def compare(dir_a, dir_b):
    """per shape: 16-bit words that differ, and the largest difference in ulp (bf16 bit patterns as ordered ints)"""
    ok = True
    for name in SHAPES:
        pa, pb = os.path.join(dir_a, f"{name}.npy"), os.path.join(dir_b, f"{name}.npy")
        if not (os.path.exists(pa) and os.path.exists(pb)):
            continue
        a, b = np.load(pa).astype(np.int32), np.load(pb).astype(np.int32)
        # sign-magnitude -> ordered integers, so that neighbouring floats differ by 1
        a = np.where(a < 0, -32768 - a, a)
        b = np.where(b < 0, -32768 - b, b)
        diff = np.abs(a - b)
        n = int((diff != 0).sum())
        ok &= n == 0
        print(json.dumps({"shape": name, "elements": int(a.size), "differ": n, "max_ulp": int(diff.max())}), flush=True)
    return ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--dump", metavar="DIR", default=None)
    ap.add_argument("--only", nargs="*", choices=sorted(SHAPES))
    ap.add_argument("--compare", nargs=2, metavar=("DIR_A", "DIR_B"))
    args = ap.parse_args()
    if args.compare:
        sys.exit(0 if compare(*args.compare) else 1)
    run(args)


if __name__ == "__main__":
    main()
