#!/usr/bin/env python
"""16-bit against FP8 (e4m3) in one process, alternating, on the C4 workload (FLUX.1-schnell 1024^2, 4 images).

  python tools/bench_fp8.py [--iters 30] [--warmup 5] [--rounds 3] [--skip-model]

(i)   every GEMM shape of tools/bench_gemm.py with its real epilogue: 16-bit dk_gemm, dk_gemm_fp8 alone, and dk_gemm_fp8
      plus the quantiser launch that feeds it (dk_ln_modulate_fp8 in place of dk_ln_modulate costs no extra launch, so
      the qkv / fc1 shapes have no feeding quantiser), all as TFLOP/s of the same 2 M N K;
(ii)  dk_quantize_rows_e4m3 and dk_ln_modulate_fp8 as GB/s of the bytes they must move (the data-sheet HBM3 rate of the
      H100 SXM is 3350 GB/s);
(iii) the full-size MMDiT forward (one denoise step, synthetic weights) with FP8 off / on, --rounds alternations.
CUDA events around --iters launches after --warmup.  Prints the card, its power limit and SM clock read in the same
run, and fails when there is no GPU.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_gemm import B, D, H, HEADS, S, S_IMG, S_TXT, SHAPES, card_info  # noqa: E402

# shapes whose input no LayerNorm-modulate produces: a quantiser launch feeds the FP8 GEMM
QUANTISED_INPUT = ("_o", "_fc2", "single_out")


def timed(fn, iters, warmup):
    import torch

    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / iters


def make_case(name, dev):
    """the three launch closures of one shape: 16-bit, FP8 GEMM alone, quantiser + FP8 GEMM (None if LN feeds it)"""
    import torch

    from diffusionkit_b200 import ops
    from diffusionkit_b200._lib import ACT_GELU_ERF

    M, N, K, epi, _ = SHAPES[name]
    g = torch.Generator(device=dev).manual_seed(sum(map(ord, name)))

    def rnd(shape, scale=1.0):
        return (torch.randn(shape, generator=g, device=dev) * scale).to(torch.bfloat16)

    A, W, bias = rnd((M, K)), rnd((N, K), 1.0 / math.sqrt(K)), rnd((N,), 0.5)
    Aq, a_s = ops.quantize_rows_e4m3(A)
    Wq, w_s = ops.quantize_rows_e4m3(W)
    kw = dict(bias=bias)
    if epi.startswith("qk"):
        rpb, obr, off = {"qk_img": (S_IMG, S, S_TXT), "qk_txt": (S_TXT, S, 0), "qk_single": (S, S, 0)}[epi]
        ang = torch.rand((S, D // 2), generator=g, device=dev) * 6.28
        rope = torch.stack([torch.cos(ang), torch.sin(ang)], dim=-1).contiguous()
        kw.update(out=torch.zeros((B * S, N), dtype=torch.bfloat16, device=dev), rows_per_batch=rpb, out_batch_rows=obr,
                  out_row_off=off, qk=(HEADS, D, rnd((D,), 0.1) + 1.0, rnd((D,), 0.1) + 1.0, rope, 1e-6))
    elif epi.startswith("gate_res"):
        rpb = {"gate_res_img": S_IMG, "gate_res_txt": S_TXT, "gate_res_single": S}[epi]
        x = rnd((M, N))
        kw.update(out=x, res=x, gate=rnd((B, N), 0.1), rows_per_batch=rpb, out_batch_rows=rpb)
    elif epi == "gelu_cat":
        kw.update(out=torch.zeros((M, 5 * H), dtype=torch.bfloat16, device=dev)[:, H:], act=ACT_GELU_ERF)
    else:
        kw.update(out=torch.empty((M, N), dtype=torch.bfloat16, device=dev), act=ACT_GELU_ERF)

    def fed():
        ops.quantize_rows_e4m3(A, out=Aq, scale=a_s)
        ops.gemm_fp8(Aq, a_s, Wq, w_s, **kw)

    return (lambda: ops.gemm(A, W, **kw), lambda: ops.gemm_fp8(Aq, a_s, Wq, w_s, **kw),
            fed if name.endswith(QUANTISED_INPUT) else None)


def bench_gemms(args, dev):
    import torch

    rows, tot = {}, {"bf16": 0.0, "fp8": 0.0, "fp8_fed": 0.0}
    for name, (M, N, K, epi, per_fwd) in SHAPES.items():
        f16, f8, fed = make_case(name, dev)
        sec = {"bf16": [], "fp8": [], "fp8_fed": []}
        for _ in range(args.rounds):
            sec["bf16"].append(timed(f16, args.iters, args.warmup))
            sec["fp8"].append(timed(f8, args.iters, args.warmup))
            sec["fp8_fed"].append(timed(fed, args.iters, args.warmup) if fed else sec["fp8"][-1])
        flop = 2.0 * M * N * K
        best = {k: min(v) for k, v in sec.items()}
        rows[name] = {"M": M, "N": N, "K": K, **{k + "_us": round(v * 1e6, 1) for k, v in best.items()},
                      **{k + "_tflops": round(flop / v / 1e12, 1) for k, v in best.items()},
                      "quantiser_launch": fed is not None}
        for k in tot:
            tot[k] += per_fwd * best[k]
        print(f"{name:16s} {M:6d} x {N:5d} x {K:5d}  " + "  ".join(
            f"{k} {best[k] * 1e6:8.1f} us {flop / best[k] / 1e12:6.1f} TFLOP/s" for k in best), flush=True)
        del f16, f8, fed
        torch.cuda.empty_cache()
    return rows, {k + "_gemm_seconds_per_forward": round(v, 4) for k, v in tot.items()}


def bench_elementwise(args, dev):
    import torch

    from diffusionkit_b200 import ops

    out = {}
    for rows, cols in [(B * S_IMG, H), (B * S_IMG, 4 * H), (B * S, 5 * H)]:
        x = torch.randn((rows, cols), device=dev).to(torch.bfloat16)
        q, s = ops.quantize_rows_e4m3(x)
        sec = timed(lambda: ops.quantize_rows_e4m3(x, out=q, scale=s), args.iters, args.warmup)
        out[f"quantize_rows_{rows}x{cols}"] = {"us": round(sec * 1e6, 1), "gb_s": round(rows * (3 * cols + 4) / sec / 1e9)}
    for rows, rpb in [(B * S_IMG, S_IMG), (B * S, S)]:
        x = torch.randn((rows, H), device=dev).to(torch.bfloat16)
        mod = (torch.randn((B, 2 * H), device=dev) * 0.3).to(torch.bfloat16)
        q, s = ops.ln_modulate_fp8(x, mod[:, :H], mod[:, H:], rpb)
        y = torch.empty_like(x)
        sec8 = timed(lambda: ops.ln_modulate_fp8(x, mod[:, :H], mod[:, H:], rpb, out=q, out_scale=s), args.iters,
                     args.warmup)
        sec16 = timed(lambda: ops.ln_modulate(x, mod[:, :H], mod[:, H:], rpb, out=y), args.iters, args.warmup)
        out[f"ln_modulate_fp8_{rows}x{H}"] = {"us": round(sec8 * 1e6, 1), "gb_s": round(rows * (3 * H + 4) / sec8 / 1e9),
                                              "ln_modulate_16bit_us": round(sec16 * 1e6, 1)}
    for k, v in out.items():
        print(k, v, flush=True)
    return out


def bench_model(args, dev):
    import torch

    import diffusionkit_b200 as dk

    pipe = dk.FluxPipeline(w16=True, a16=True, device=dev, load_decoder=False)
    cond, pooled = [t.to(dev) for t in pipe.synthetic_text_embeddings(n_images=B, text_len=S_TXT)]
    m = pipe.mmdit
    m.cache_modulation_params(pooled, [500.0])
    latent = torch.randn((B, 128, 128, 16), device=dev).to(torch.bfloat16)
    t = torch.full((B,), 500.0)
    sec = {"off": [], "on": []}
    for _ in range(args.rounds):
        for mode in ("off", "on"):
            before = torch.cuda.memory_allocated(dev)
            pipe.set_fp8(mode == "on")
            if mode == "on":
                extra = torch.cuda.memory_allocated(dev) - before   # e4m3 weights + scales
            sec[mode].append(timed(lambda: m(latent, cond, t), max(3, args.iters // 6), 2))
    pipe.set_fp8(False)
    res = {"forward_ms_fp8_off": [round(s * 1e3, 2) for s in sec["off"]],
           "forward_ms_fp8_on": [round(s * 1e3, 2) for s in sec["on"]],
           "fp8_weight_bytes": extra, "speedup": round(min(sec["off"]) / min(sec["on"]), 3)}
    print(res, flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-model", action="store_true")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    gemms, totals = bench_gemms(args, dev)
    elem = bench_elementwise(args, dev)
    model = None if args.skip_model else bench_model(args, dev)
    print(json.dumps({"gemm": gemms, **totals, "elementwise": elem, "model": model, "iters": args.iters,
                      "rounds": args.rounds, **card_info()}), flush=True)


if __name__ == "__main__":
    main()
