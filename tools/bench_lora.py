#!/usr/bin/env python
"""Cost of LoRA adapters on full-size FLUX.1-schnell (synthetic weights and adapters that cover every module).

  python tools/bench_lora.py [--ranks 16 64] [--rounds 3] [--images 4] [--latent 128] [--steps 4]

Per rank: the first merge (live copies allocated, every weight merged), a scale change (re-merge in place) and the
unload, each timed with CUDA events around MMDiT.apply_lora after a device synchronise, so host-side factor
preparation counts; the extra HBM the live copies hold (torch.cuda.memory_allocated).  Then denoise step times of
the pipeline (CUDA events of sample_euler) without and with the largest adapter, alternated --rounds times in one run;
each mode runs one untimed denoise first because binding or unbinding live copies drops the captured graphs.  Prints one
JSON line that names the card, its power limit and the SM clock read in the same run.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_gemm import card_info  # noqa: E402


def synthetic_adapter(cfg, rank: int, seed: int) -> dict:
    """PEFT state dict with a rank-`rank` factor pair for every upstream module; ΔW ~ 0.1 / sqrt(fan_in)"""
    import torch

    from diffusionkit_b200.lora import module_table
    from diffusionkit_b200.weights import mmdit_param_specs

    shapes = {n: s for n, s, _ in mmdit_param_specs(cfg)}
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for module, (axis, refs) in module_table(cfg).items():
        outs = [shapes[r][0] for r in refs]
        ins = [math.prod(shapes[r][1:]) for r in refs]
        n_out, n_in = (sum(outs), ins[0]) if axis == 0 else (outs[0], sum(ins))
        sd[module + ".lora_A.weight"] = torch.randn((rank, n_in), generator=g) / math.sqrt(n_in)
        sd[module + ".lora_B.weight"] = torch.randn((n_out, rank), generator=g) * (0.1 / math.sqrt(rank))
    return sd


def run(args):
    import torch

    import diffusionkit_b200 as dk
    from diffusionkit_b200.lora import load_lora

    if not torch.cuda.is_available():
        raise SystemExit("bench_lora.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    pipe = dk.FluxPipeline(w16=True, a16=True, model_version="argmaxinc/mlx-FLUX.1-schnell", load_decoder=False,
                           device=dev)
    m, cfg = pipe.mmdit, pipe.config
    cond, pooled = pipe.synthetic_text_embeddings(n_images=args.images)
    seeds = list(range(args.images))

    def timed_ms(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(dev)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize(dev)
        return round(e0.elapsed_time(e1), 1)

    out = {"workload": f"FLUX.1-schnell synthetic, {args.images} x {8 * args.latent}^2, {args.steps} steps",
           "adapters": {}}
    adapters = {}
    for rank in args.ranks:
        t0 = time.time()
        adapters[rank] = load_lora(synthetic_adapter(cfg, rank, seed=rank), cfg, name=f"rank{rank}")
        n = sum(up.numel() + down.numel() for up, down in adapters[rank].targets.values())
        row = {"targets": len(adapters[rank].targets), "parse_s": round(time.time() - t0, 2)}
        mem0 = torch.cuda.memory_allocated(dev)
        row["apply_ms"] = timed_ms(lambda: m.apply_lora([(adapters[rank], 1.0)]))
        row["extra_hbm_gb"] = round((torch.cuda.memory_allocated(dev) - mem0) / 1e9, 2)
        row["scale_change_ms"] = timed_ms(lambda: m.apply_lora([(adapters[rank], 0.5)]))
        row["unload_ms"] = timed_ms(lambda: m.apply_lora([]))
        row["factor_elements_m"] = round(n / 1e6, 1)
        out["adapters"][f"rank{rank}"] = row
        print(f"rank {rank}: {json.dumps(row)}", flush=True)

    biggest = adapters[max(args.ranks)]
    steps = {"none": [], f"rank{max(args.ranks)}": []}
    for _ in range(args.rounds):
        for mode in steps:
            m.apply_lora([] if mode == "none" else [(biggest, 1.0)])
            kw = dict(num_steps=args.steps, latent_size=(args.latent, args.latent), seed=seeds)
            pipe.denoise_latents(cond, pooled, **kw)
            _, iter_time = pipe.denoise_latents(cond, pooled, **kw)
            steps[mode].append(round(statistics.median(iter_time) * 1e3, 1))
        print(f"step ms (median of {args.steps} per run): {json.dumps(steps)}", flush=True)
    m.apply_lora([])
    out["step_ms"] = steps
    out.update(card_info())
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--ranks", type=int, nargs="+", default=[16, 64])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--images", type=int, default=4)
    ap.add_argument("--latent", type=int, default=128, help="latent height = width (128 -> 1024^2 images)")
    ap.add_argument("--steps", type=int, default=4)
    run(ap.parse_args())


if __name__ == "__main__":
    main()
