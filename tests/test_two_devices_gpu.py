"""-m gpu: two contexts on two GPUs in one process.

A kernel's dynamic shared-memory limit belongs to the kernel as loaded in one device's context.  Every kernel that
needs more than the default 48 KB (the GEMM, attention, the fused convolution, short-sequence attention) must
therefore run on the second device after it has run on the first, and compute the same bits there.
"""
import math

import pytest
import torch

from diffusionkit_b200 import ops

pytestmark = pytest.mark.gpu


def _rand(shape, dtype, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype)


def _run_all(dev, inputs):
    a, w, qkv, x, wc, qkv_s = (t.to(dev) for t in inputs)
    gemm = ops.gemm(a, w)                                                   # N = 3072 over 32 m-blocks: BN = 256
    att = torch.empty((2 * 1024, 8 * 128), dtype=qkv.dtype, device=dev)
    ops.attention(qkv, 2, 1024, 8, 128, att)
    conv = ops.conv3x3_fused(x, wc)
    small = ops.attention_small(qkv_s, 2, 512, 12, 0.125, causal=True)     # S = 512: 132 KB of shared memory
    torch.cuda.synchronize(dev)
    return [t.cpu() for t in (gemm, att, conv, small)]


def test_every_large_smem_kernel_runs_on_both_devices(cuda):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    dt = torch.bfloat16
    inputs = (_rand((4096, 1024), dt, seed=1), _rand((3072, 1024), dt, 1 / math.sqrt(1024), seed=2),
              _rand((2 * 1024, 3 * 8 * 128), dt, seed=3),
              _rand((1, 64, 128, 128), dt, seed=4), _rand((128, 3, 3, 128), dt, 1 / math.sqrt(9 * 128), seed=5),
              _rand((2 * 512, 3 * 12 * 64), dt, seed=6))
    first = _run_all("cuda:0", inputs)
    second = _run_all("cuda:1", inputs)
    for name, a, b in zip(("gemm", "attention", "conv3x3_fused", "attention_small"), first, second):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), name
