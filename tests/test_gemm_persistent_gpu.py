"""-m gpu: what the persistent, 2-CTA-cluster GEMM can get wrong that a one-tile-per-CTA kernel could not.

The grid holds only as many clusters as fit on the device; each walks the cluster tiles (m-block pair, n-block) with
a static stride and shares its W tile with its partner.  A tile's result must not depend on which CTA computes it,
after how many other tiles, or at which ring phase; the idle partner of an odd last m-block must store nothing.
"""
import math

import pytest
import torch

from diffusionkit_b200 import ops
from diffusionkit_b200._lib import ACT_GELU_ERF

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rand(shape, dtype, scale=1.0, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(shape, generator=g, device=DEV) * scale).to(dtype)


def _rel_l2(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-30))


def _sentinel(shape, dtype):
    """a buffer of one fixed, unlikely bit pattern"""
    return torch.full(shape, 0x7A5A, dtype=torch.int16, device=DEV).view(dtype)


def _same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def test_schedule_independence_gate_residual(cuda):
    """rows 0..1023 of the C4 o-projection (16384 x 3072 x 3072, bias + gate + in-place residual) equal the same
    1024-row GEMM run alone, bit for bit"""
    M, N, K, rpb, dt = 16384, 3072, 3072, 4096, torch.bfloat16
    A, W = _rand((M, K), dt, seed=1), _rand((N, K), dt, 1 / math.sqrt(K), seed=2)
    b, gate = _rand((N,), dt, 0.5, seed=3), _rand((4, N), dt, 0.1, seed=4)
    x = _rand((M, N), dt, seed=5)
    x_small = x[:1024].clone()
    ops.gemm(A, W, out=x, bias=b, gate=gate, res=x, rows_per_batch=rpb, out_batch_rows=rpb)
    ops.gemm(A[:1024], W, out=x_small, bias=b, gate=gate, res=x_small, rows_per_batch=rpb, out_batch_rows=rpb)
    assert _same_bits(x[:1024], x_small)


def test_schedule_independence_qkv_fused(cuda):
    """the first 1280 rows of a 17408-row QK-fused QKV (RMSNorm + RoPE) equal the same rows run alone, bit for bit"""
    S, Bt, heads, d, dt = 4352, 4, 24, 128, torch.bfloat16
    h, K = heads * d, 3072
    A, W = _rand((Bt * S, K), dt, seed=6), _rand((3 * h, K), dt, 1 / math.sqrt(K), seed=7)
    bias = _rand((3 * h,), dt, 0.3, seed=8)
    qw, kw = _rand((d,), dt, 0.1, seed=9) + 1.0, _rand((d,), dt, 0.1, seed=10) + 1.0
    ang = torch.rand((S, d // 2), generator=torch.Generator(device=DEV).manual_seed(11), device=DEV) * 6.28
    rope = torch.stack([torch.cos(ang), torch.sin(ang)], dim=-1).contiguous()
    qk = (heads, d, qw, kw, rope, 1e-6)
    big = torch.zeros((Bt * S, 3 * h), dtype=dt, device=DEV)
    ops.gemm(A, W, out=big, bias=bias, rows_per_batch=S, out_batch_rows=S, qk=qk)
    n = 1280
    small = torch.zeros((n, 3 * h), dtype=dt, device=DEV)
    ops.gemm(A[:n], W, out=small, bias=bias, rows_per_batch=S, out_batch_rows=S, qk=qk)
    assert _same_bits(big[:n], small)


def test_odd_num_m_sd3_text_rows_inplace_residual(cuda):
    """M = 4 x 589 (19 m-blocks, batch boundaries inside tiles) scattered into a padded buffer with gate + in-place
    residual: the window is right and every other byte keeps its sentinel"""
    Bt, rpb, pad, off, N, K, dt = 4, 589, 40, 24, 512, 256, torch.float16
    M = Bt * rpb
    A, W = _rand((M, K), dt, seed=12), _rand((N, K), dt, 1 / math.sqrt(K), seed=13)
    b, gate = _rand((N,), dt, 0.5, seed=14), _rand((Bt, N), dt, seed=15)
    buf = _sentinel((Bt * (rpb + pad), N), dt)
    rows = torch.cat([torch.arange(i * (rpb + pad) + off, i * (rpb + pad) + off + rpb) for i in range(Bt)]).to(DEV)
    x0 = _rand((M, N), dt, seed=16)
    buf[rows] = x0
    before = buf.clone()
    ops.gemm(A, W, out=buf, bias=b, gate=gate, res=buf, rows_per_batch=rpb, out_batch_rows=rpb + pad, out_row_off=off,
             res_batch_rows=rpb + pad, res_row_off=off)
    ref = x0.float() + gate.float().repeat_interleave(rpb, 0) * (A.float() @ W.float().t() + b.float())
    assert _rel_l2(buf[rows], ref) <= 4e-3
    other = torch.ones(buf.shape[0], dtype=torch.bool, device=DEV)
    other[rows] = False
    assert _same_bits(buf[other], before[other])


@pytest.mark.parametrize("N", [64, 128, 3072])
def test_odd_num_m_cat_window(cuda, N):
    """M = 300 (3 m-blocks) with GELU into a column window of a wider buffer: the columns left and right of the window
    and the rows below it keep their sentinel"""
    M, K, left, dt = 300, 192, 128, torch.bfloat16
    A, W = _rand((M, K), dt, seed=17), _rand((N, K), dt, 1 / math.sqrt(K), seed=18)
    b = _rand((N,), dt, 0.5, seed=19)
    cat = _sentinel((M + 8, left + N + 64), dt)
    before = cat.clone()
    ops.gemm(A, W, out=cat[:M, left:left + N], bias=b, act=ACT_GELU_ERF)
    ref = torch.nn.functional.gelu(A.float() @ W.float().t() + b.float())
    assert _rel_l2(cat[:M, left:left + N], ref) <= 4e-3
    mask = torch.ones(cat.shape, dtype=torch.bool, device=DEV)
    mask[:M, left:left + N] = False
    assert _same_bits(cat[mask], before[mask])


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("N", [64, 128, 2048], ids=["n64", "n128", "n2048"])
@pytest.mark.parametrize("M", [256, 128 * 132, 128 * 700], ids=["few_tiles", "about_one_wave", "many_waves"])
def test_repeatable(cuda, dtype, N, M):
    """two launches on the same input are bit-identical, for tile counts below, about at and far above the number of
    resident CTAs"""
    K = 256
    A, W = _rand((M, K), dtype, seed=20), _rand((N, K), dtype, 1 / math.sqrt(K), seed=21)
    b = _rand((N,), dtype, 0.5, seed=22)
    one = ops.gemm(A, W, bias=b, act=ACT_GELU_ERF)
    two = ops.gemm(A, W, bias=b, act=ACT_GELU_ERF)
    assert _same_bits(one, two)
    if M == 256:
        ref = torch.nn.functional.gelu(A.float() @ W.float().t() + b.float())
        assert _rel_l2(one, ref) <= 4e-3


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(1, 101, 64, 128, 128), (1, 320, 320, 128, 256)],
                         ids=["odd_num_m", "ragged_x"])
def test_conv3x3_persistent(cuda, B, H, W, Cin, Cout):
    """the implicit-GEMM convolution (4-D TMA boxes, per-tile image / pixel origin) through the persistent loop: 51
    m-blocks (an idle cluster partner) and 960 m-blocks with ragged 128-pixel row tiles"""
    dt = torch.bfloat16
    x = _rand((B, H, W, Cin), dt, seed=23)
    w = _rand((Cout, 3, 3, Cin), dt, 1 / math.sqrt(9 * Cin), seed=24)
    b = _rand((Cout,), dt, 0.5, seed=25)
    r = _rand((B, H, W, Cout), dt, seed=26)
    got = ops.conv3x3(x, w, bias=b, res=r)
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), b.float(),
                                     padding=1).permute(0, 2, 3, 1) + r.float()
    assert _rel_l2(got, ref) <= 4e-3
    assert _same_bits(got, ops.conv3x3(x, w, bias=b, res=r))


def test_w_n_major_persistent(cuda):
    """W given as [K, N] (MN-major operand, each CTA multicasts one of the two 64-column boxes): 333 m-blocks x 3
    n-blocks"""
    M, N, K, dt = 128 * 333 - 40, 384, 256, torch.bfloat16
    A, Wt = _rand((M, K), dt, seed=27), _rand((K, N), dt, 1 / math.sqrt(K), seed=28)
    got = ops.gemm(A, Wt, w_n_major=True)
    assert _rel_l2(got, A.float() @ Wt.float()) <= 4e-3
    assert _same_bits(got, ops.gemm(A, Wt, w_n_major=True))
