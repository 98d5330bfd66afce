"""Typed Python wrappers over the C ABI (torch tensors are only the device-memory containers).

Every function launches hand-written sm_90a kernels from libdkb200.so asynchronously on the current
torch CUDA stream.  Nothing here has a torch / CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional, Tuple

import torch

from . import _lib
from ._lib import ACT_GELU_ERF, ACT_NONE, ACT_QUICK_GELU, ACT_SILU, Context, GemmArgs, dtype_code, ptr

_ctx = {}


def ctx(device: Optional[int] = None) -> Context:
    if device is None:
        device = torch.cuda.current_device()
    c = _ctx.get(device)
    if c is None:
        c = Context(device)
        _ctx[device] = c
    return c


_graph_launches = 0


def note_graph_launches(n: int):
    """kernels replayed from a captured CUDA graph (the C-side counter only sees the capture pass)"""
    global _graph_launches
    _graph_launches += n


def launch_count() -> int:
    return sum(c.launches for c in _ctx.values()) + _graph_launches


def _chk16(t: torch.Tensor, name: str):
    if t.dtype not in (torch.bfloat16, torch.float16):
        raise _lib.DkError(f"{name}: expected a bf16/fp16 tensor, got {t.dtype}")
    if not t.is_cuda:
        raise _lib.DkError(f"{name}: expected a CUDA tensor (there is no CPU fallback)")


def gemm(
    A: torch.Tensor,
    W: torch.Tensor,
    out: Optional[torch.Tensor] = None,
    bias: Optional[torch.Tensor] = None,
    act: int = ACT_NONE,
    gate: Optional[torch.Tensor] = None,
    res: Optional[torch.Tensor] = None,
    rows_per_batch: int = 0,
    out_batch_rows: int = 0,
    out_row_off: int = 0,
    res_batch_rows: Optional[int] = None,
    res_row_off: int = 0,
    w_n_major: bool = False,
    N: Optional[int] = None,
    qk: Optional[tuple] = None,
    fp8_scales: Optional[tuple] = None,
    dtype: Optional[torch.dtype] = None,
) -> torch.Tensor:
    """out = res + gate * act(A @ W.T + bias)   (see include/dkb200.h, dk_gemm).

    A: [M, K] (row stride may exceed K), W: [N, K] (nn.Linear layout) or [K, N] when w_n_major.
    out: 2-D view [rows, >=N] whose row stride is the leading dimension.
    fp8_scales (gemm_fp8 passes it): A and W hold e4m3 bytes, (a_scale [M], w_scale [N]) are their fp32 row scales and
    dtype is the 16-bit type of out (dk_gemm_fp8).
    """
    if fp8_scales is None:
        _chk16(A, "gemm.A")
        _chk16(W, "gemm.W")
        dtype = A.dtype
    else:
        _chk_e4m3(A, "gemm_fp8.A")
        _chk_e4m3(W, "gemm_fp8.W")
        a_scale, w_scale = fp8_scales
        dtype = out.dtype if out is not None else dtype
    assert A.dim() == 2 and W.dim() == 2 and A.stride(1) == 1 and W.stride(1) == 1
    M, K = A.shape
    if w_n_major:
        assert W.shape[0] == K
        n = W.shape[1]
    else:
        assert W.shape[1] == K, f"K mismatch {A.shape} x {W.shape}"
        n = W.shape[0]
    if N is not None:
        n = N
    if out is None:
        out = torch.empty((M, n), dtype=dtype, device=A.device)
    assert out.dim() == 2 and out.stride(1) == 1
    a = GemmArgs()
    a.dtype = dtype_code(dtype)
    a.M, a.N, a.K = M, n, K
    a.A, a.lda = ptr(A), A.stride(0)
    a.W, a.ldw = ptr(W), W.stride(0)
    a.out, a.ldc = ptr(out), out.stride(0)
    a.bias = ptr(bias)
    a.gate = ptr(gate)
    a.gate_ld = gate.stride(0) if gate is not None else 0
    a.res = ptr(res)
    a.ldres = res.stride(0) if res is not None else 0
    a.rows_per_batch = rows_per_batch
    a.out_batch_rows = out_batch_rows if rows_per_batch else 0
    a.out_row_off = out_row_off
    if res_batch_rows is None:
        res_batch_rows = rows_per_batch
    a.res_batch_rows = res_batch_rows if rows_per_batch else 0
    a.res_row_off = res_row_off
    a.act = act
    a.w_n_major = 1 if w_n_major else 0
    if qk is not None:
        # (heads, head_dim, q_norm_weight | None, k_norm_weight | None, rope table | None, eps)
        heads, hd, qw, kw, rope, eps = qk
        a.qk_heads, a.qk_head_dim, a.qk_eps = heads, hd, eps
        a.qk_q_weight, a.qk_k_weight, a.qk_rope = ptr(qw), ptr(kw), ptr(rope)
    c = ctx(A.device.index)
    if fp8_scales is None:
        c.check(c.lib.dk_gemm(c.handle, C.byref(a), c.stream))
    else:
        assert a_scale.dtype == torch.float32 and w_scale.dtype == torch.float32
        assert a_scale.numel() == M and w_scale.numel() >= n and a_scale.is_contiguous() and w_scale.is_contiguous()
        c.check(c.lib.dk_gemm_fp8(c.handle, C.byref(a), ptr(a_scale), ptr(w_scale), c.stream))
    return out


def _chk_e4m3(t: torch.Tensor, name: str):
    if t.dtype != torch.float8_e4m3fn or not t.is_cuda:
        raise _lib.DkError(f"{name}: expected a CUDA torch.float8_e4m3fn tensor, got {t.dtype} on {t.device}")


def gemm_fp8(A, a_scale, W, w_scale, dtype: Optional[torch.dtype] = None, **epilogue) -> torch.Tensor:
    """gemm with row-quantised e4m3 operands: A [M, K] with a_scale [M], W [N, K] with w_scale [N] (as
    quantize_rows_e4m3 / ln_modulate_fp8 produce them); the accumulator is scaled by a_scale[m] * w_scale[n] ahead of
    gemm's epilogue, whose keyword arguments this takes (not w_n_major).  dtype: 16-bit type of out when out is not
    given."""
    return gemm(A, W, fp8_scales=(a_scale, w_scale), dtype=dtype, **epilogue)


def quantize_rows_e4m3(x, out=None, scale=None):
    """x [rows, cols] 16-bit (row stride may exceed cols) -> (q [rows, cols] e4m3, scale [rows] fp32):
    scale = amax|row| / 448 (1 for a zero row), q = e4m3(x / scale)."""
    _chk16(x, "quantize_rows_e4m3.x")
    assert x.dim() == 2 and x.stride(1) == 1
    rows, cols = x.shape
    if out is None:
        out = torch.empty((rows, cols), dtype=torch.float8_e4m3fn, device=x.device)
    if scale is None:
        scale = torch.empty((rows,), dtype=torch.float32, device=x.device)
    _chk_e4m3(out, "quantize_rows_e4m3.out")
    assert out.is_contiguous() and out.shape == (rows, cols) and scale.dtype == torch.float32 and scale.numel() == rows
    c = ctx(x.device.index)
    c.call("dk_quantize_rows_e4m3", dtype_code(x.dtype), ptr(x), x.stride(0), ptr(out), ptr(scale), rows, cols)
    return out, scale


def ln_modulate_fp8(x, shift, scale, rows_per_batch: int, eps: float = 1e-6, out=None, out_scale=None):
    """ln_modulate whose fp32 result row is quantised like quantize_rows_e4m3 -> (q [rows, h] e4m3, scale [rows])."""
    _chk16(x, "ln_modulate_fp8.x")
    rows, h = x.shape
    assert x.is_contiguous() and shift.stride(0) == scale.stride(0) and shift.stride(1) == 1
    if out is None:
        out = torch.empty((rows, h), dtype=torch.float8_e4m3fn, device=x.device)
    if out_scale is None:
        out_scale = torch.empty((rows,), dtype=torch.float32, device=x.device)
    _chk_e4m3(out, "ln_modulate_fp8.out")
    assert out.is_contiguous() and out_scale.dtype == torch.float32 and out_scale.numel() == rows
    c = ctx(x.device.index)
    c.call("dk_ln_modulate_fp8", dtype_code(x.dtype), ptr(x), ptr(out), ptr(out_scale), ptr(shift), ptr(scale),
           shift.stride(0), rows, rows_per_batch, h, eps)
    return out, out_scale


def ln_modulate(x, shift, scale, rows_per_batch: int, eps: float = 1e-6, out=None):
    """y = LN(x) * (1 + scale[b]) + shift[b]; x [rows, h]; shift/scale 2-D views [B, h] (row stride = mod_ld)."""
    _chk16(x, "ln_modulate.x")
    rows, h = x.shape
    assert x.is_contiguous() and shift.stride(0) == scale.stride(0) and shift.stride(1) == 1
    if out is None:
        out = torch.empty_like(x)
    c = ctx(x.device.index)
    c.call("dk_ln_modulate", dtype_code(x.dtype), ptr(x), ptr(out), ptr(shift), ptr(scale), shift.stride(0), rows,
           rows_per_batch, h, eps)
    return out


def qk_norm_rope(qkv, S: int, heads: int, d: int, split: int, q_w=None, k_w=None, q_w2=None, k_w2=None, rope=None,
                 eps: float = 1e-6):
    _chk16(qkv, "qk_norm_rope.qkv")
    assert qkv.is_contiguous() and qkv.shape[1] == 3 * heads * d
    if rope is not None:
        assert rope.dtype == torch.float32 and rope.is_contiguous() and rope.numel() == S * d
    c = ctx(qkv.device.index)
    c.call("dk_qk_norm_rope", dtype_code(qkv.dtype), ptr(qkv), qkv.shape[0], S, heads, d, split, ptr(q_w), ptr(k_w),
           ptr(q_w2), ptr(k_w2), ptr(rope), eps)
    return qkv


def attention(qkv, B: int, S: int, heads: int, d: int, out0, split: Optional[int] = None, out1=None,
              scale: Optional[float] = None):
    """softmax(scale q k^T) v over the packed [B*S, 3*heads*d] buffer; rows < split go to out0, the rest to out1."""
    _chk16(qkv, "attention.qkv")
    assert qkv.is_contiguous() and qkv.shape == (B * S, 3 * heads * d)
    if split is None:
        split = S
    if scale is None:
        scale = 1.0 / math.sqrt(d)
    c = ctx(qkv.device.index)
    c.call("dk_attention_fwd", dtype_code(qkv.dtype), ptr(qkv), B, S, heads, d, scale, split, ptr(out0),
           out0.stride(0) if out0 is not None else 0, ptr(out1), out1.stride(0) if out1 is not None else 0)
    return out0, out1


def silu_add(y, temb, out=None):
    """out[t*B + b] = silu(y[b] + temb[t])."""
    _chk16(y, "silu_add.y")
    B, h = y.shape
    n_t = temb.shape[0]
    if out is None:
        out = torch.empty((n_t * B, h), dtype=y.dtype, device=y.device)
    c = ctx(y.device.index)
    c.call("dk_silu_add", dtype_code(y.dtype), ptr(y), ptr(temb), ptr(out), n_t, B, h)
    return out


def act(x, kind: int, out=None):
    _chk16(x, "act.x")
    if out is None:
        out = torch.empty_like(x)
    c = ctx(x.device.index)
    c.call("dk_act", dtype_code(x.dtype), ptr(x), ptr(out), x.numel(), kind)
    return out


def patchify(latent, order: int, out=None):
    _chk16(latent, "patchify.latent")
    B, H, W, Cc = latent.shape
    if out is None:
        out = torch.empty((B * (H // 2) * (W // 2), 4 * Cc), dtype=latent.dtype, device=latent.device)
    c = ctx(latent.device.index)
    c.call("dk_patchify", dtype_code(latent.dtype), ptr(latent), ptr(out), B, H, W, Cc, order)
    return out


def unpatchify(rows, B: int, H: int, W: int, Cc: int, order: int, out=None):
    _chk16(rows, "unpatchify.rows")
    if out is None:
        out = torch.empty((B, H, W, Cc), dtype=rows.dtype, device=rows.device)
    c = ctx(rows.device.index)
    c.call("dk_unpatchify", dtype_code(rows.dtype), ptr(rows), ptr(out), B, H, W, Cc, order)
    return out


def pos_embed_crop(table, max_hw: int, hp: int, wp: int):
    _chk16(table, "pos_embed_crop.table")
    h = table.shape[1]
    out = torch.empty((hp * wp, h), dtype=table.dtype, device=table.device)
    c = ctx(table.device.index)
    c.call("dk_pos_embed_crop", dtype_code(table.dtype), ptr(table), ptr(out), max_hw, hp, wp, h)
    return out


def copy_rows(src, dst, B: int, rows: int, h: int, dst_rows: int, dst_off: int, src_rows: int, src_off: int):
    _chk16(src, "copy_rows.src")
    c = ctx(src.device.index)
    c.call("dk_copy_rows", dtype_code(src.dtype), ptr(src), ptr(dst), B, rows, h, dst_rows, dst_off, src_rows, src_off)
    return dst


def sampler_prepare(x, xin, reps: int):
    assert x.dtype == torch.float32 and x.is_contiguous()
    c = ctx(x.device.index)
    c.call("dk_sampler_prepare", dtype_code(xin.dtype), ptr(x), ptr(xin), x.numel(), reps)
    return xin


def _slg_entry(name: str, slg: float) -> Tuple[str, tuple]:
    """the plain solver-update entry point for slg == 0, its skip-layer-guidance twin (DESIGN.md §13) otherwise:
    then xin / out hold [positive | negative | positive skipping joint blocks] and D gains slg (D_pos - D_skip)"""
    return (name, ()) if slg == 0.0 else (name + "_slg", (float(slg),))


def sampler_step(x, xin, out, sigma: float, sigma_next: float, cfg_weight: float, slg: float = 0.0):
    assert x.dtype == torch.float32 and x.is_contiguous()
    c = ctx(x.device.index)
    name, extra = _slg_entry("dk_sampler_step", slg)
    c.call(name, dtype_code(xin.dtype), ptr(x), ptr(xin), ptr(out), x.numel(), sigma, sigma_next, cfg_weight, *extra)
    return x


def sampler_heun_predict(x, xin, out, sigma: float, sigma_next: float, cfg_weight: float, d=None, x2=None,
                         slg: float = 0.0):
    """-> (d, x2): the slope at (x, sigma) and the Euler step to sigma_next (fp32, like x); x is not modified"""
    assert x.dtype == torch.float32 and x.is_contiguous()
    d = torch.empty_like(x) if d is None else d
    x2 = torch.empty_like(x) if x2 is None else x2
    assert d.shape == x2.shape == x.shape and d.dtype == x2.dtype == torch.float32
    assert d.is_contiguous() and x2.is_contiguous()
    c = ctx(x.device.index)
    name, extra = _slg_entry("dk_sampler_heun_predict", slg)
    c.call(name, dtype_code(xin.dtype), ptr(x), ptr(xin), ptr(out), ptr(d), ptr(x2), x.numel(), sigma, sigma_next,
           cfg_weight, *extra)
    return d, x2


def sampler_heun_correct(x, d, x2, xin, out, sigma: float, sigma_next: float, cfg_weight: float, slg: float = 0.0):
    """x += (d + d2) / 2 * (sigma_next - sigma), d2 the slope of the forward (xin, out) at (x2, sigma_next)"""
    assert x.dtype == d.dtype == x2.dtype == torch.float32
    assert x.is_contiguous() and d.is_contiguous() and x2.is_contiguous() and d.shape == x2.shape == x.shape
    c = ctx(x.device.index)
    name, extra = _slg_entry("dk_sampler_heun_correct", slg)
    c.call(name, dtype_code(xin.dtype), ptr(x), ptr(d), ptr(x2), ptr(xin), ptr(out), x.numel(), sigma, sigma_next,
           cfg_weight, *extra)
    return x


def sampler_dpmpp_2m(x, d_prev, xin, out, sigma: float, a: float, b: float, c: float, cfg_weight: float,
                     slg: float = 0.0):
    """x = a x + b D + c d_prev, then d_prev = D (both in place); d_prev is not read when c == 0"""
    assert x.dtype == d_prev.dtype == torch.float32 and x.is_contiguous() and d_prev.is_contiguous()
    assert d_prev.shape == x.shape
    cx = ctx(x.device.index)
    name, extra = _slg_entry("dk_sampler_dpmpp_2m", slg)
    cx.call(name, dtype_code(xin.dtype), ptr(x), ptr(d_prev), ptr(xin), ptr(out), x.numel(), sigma, a, b, c,
            cfg_weight, *extra)
    return x


def axpb(x, a: float, b: float, out=None):
    assert x.dtype == torch.float32 and x.is_contiguous()
    if out is None:
        out = torch.empty_like(x)
    c = ctx(x.device.index)
    c.call("dk_axpb_f32", ptr(x), ptr(out), x.numel(), a, b)
    return out


# ------------------------------------------------------------------------------------------------ text encoders
def embedding(table, ids, pos=None, out=None):
    """out[i] = table[ids[i]] (+ pos[i % len(pos)]); ids int32 (any shape, flattened)"""
    _chk16(table, "embedding.table")
    assert table.is_contiguous() and ids.dtype == torch.int32 and ids.is_contiguous() and ids.is_cuda
    n, d = ids.numel(), table.shape[1]
    if out is None:
        out = torch.empty((n, d), dtype=table.dtype, device=table.device)
    c = ctx(table.device.index)
    c.call("dk_embedding", dtype_code(table.dtype), ptr(table), ptr(ids), ptr(pos), ptr(out), n, d, table.shape[0],
           0 if pos is None else pos.shape[0])
    return out


def layernorm(x, weight, bias, eps: float = 1e-5, out=None):
    _chk16(x, "layernorm.x")
    rows, h = x.shape
    assert x.is_contiguous() and weight.is_contiguous() and bias.is_contiguous()
    if out is None:
        out = torch.empty_like(x)
    c = ctx(x.device.index)
    c.call("dk_layernorm", dtype_code(x.dtype), ptr(x), ptr(out), ptr(weight), ptr(bias), rows, h, eps)
    return out


def rmsnorm_f32(x, weight, eps: float = 1e-6, out=None):
    """x fp32 [rows, d] -> 16-bit (weight's dtype) weight * x * rsqrt(mean(x^2) + eps)"""
    _chk16(weight, "rmsnorm_f32.weight")
    assert x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 2
    if out is None:
        out = torch.empty(x.shape, dtype=weight.dtype, device=x.device)
    c = ctx(x.device.index)
    c.call("dk_rmsnorm_f32", dtype_code(weight.dtype), ptr(x), ptr(weight), ptr(out), x.shape[0], x.shape[1], eps)
    return out


def add_f32_16(x, y):
    _chk16(y, "add_f32_16.y")
    assert x.dtype == torch.float32 and x.is_contiguous() and y.is_contiguous() and x.numel() == y.numel()
    c = ctx(x.device.index)
    c.call("dk_add_f32_16", dtype_code(y.dtype), ptr(x), ptr(y), x.numel())
    return x


def glu_gelu(h, out=None):
    _chk16(h, "glu_gelu.h")
    rows, F2 = h.shape
    assert h.is_contiguous() and F2 % 2 == 0
    if out is None:
        out = torch.empty((rows, F2 // 2), dtype=h.dtype, device=h.device)
    c = ctx(h.device.index)
    c.call("dk_glu_gelu", dtype_code(h.dtype), ptr(h), ptr(out), rows, F2 // 2)
    return out


def attention_small(qkv, B: int, S: int, heads: int, scale: float, rel_bias=None, causal: bool = False, out=None):
    """packed (q | k | v) [B*S, 3*heads*64] -> [B*S, heads*64]; rel_bias [heads, 2S-1] or None"""
    _chk16(qkv, "attention_small.qkv")
    assert qkv.is_contiguous() and tuple(qkv.shape) == (B * S, 3 * heads * 64)
    if rel_bias is not None:
        assert rel_bias.dtype == qkv.dtype and rel_bias.is_contiguous() and tuple(rel_bias.shape) == (heads, 2 * S - 1)
    if out is None:
        out = torch.empty((B * S, heads * 64), dtype=qkv.dtype, device=qkv.device)
    c = ctx(qkv.device.index)
    c.call("dk_attention_small", dtype_code(qkv.dtype), ptr(qkv), ptr(rel_bias), ptr(out), B, S, heads, 64, scale,
           1 if causal else 0)
    return out


def dequant_q4(wq, scales, biases, group_size: int = 64, out=None):
    """MLX affine 4-bit weight (wq [N, K/8] uint32 stored as int32/uint32, scales/biases [N, K/group] 16-bit) ->
    dense [N, K] in the scales' dtype"""
    _chk16(scales, "dequant_q4.scales")
    assert wq.dtype in (torch.int32, torch.uint32) and wq.dim() == 2 and wq.is_contiguous() and wq.is_cuda
    assert scales.is_contiguous() and biases.is_contiguous() and biases.dtype == scales.dtype
    N, K = wq.shape[0], wq.shape[1] * 8
    assert tuple(scales.shape) == tuple(biases.shape) == (N, K // group_size)
    if out is None:
        out = torch.empty((N, K), dtype=scales.dtype, device=wq.device)
    c = ctx(wq.device.index)
    c.call("dk_dequant_q4", dtype_code(scales.dtype), ptr(wq), ptr(scales), ptr(biases), ptr(out), N, K, group_size)
    return out


def image_pre(img_u8, dtype, cpad: int = 64):
    """uint8 NHWC [B,H,W,>=3] -> 16-bit NHWC [B,H,W,cpad] in [-1, 1] (channels 3.. zero)"""
    assert img_u8.dtype == torch.uint8 and img_u8.is_contiguous() and img_u8.dim() == 4 and img_u8.is_cuda
    B, H, W, Cs = img_u8.shape
    out = torch.empty((B, H, W, cpad), dtype=dtype, device=img_u8.device)
    c = ctx(img_u8.device.index)
    c.call("dk_image_pre", dtype_code(dtype), ptr(img_u8), ptr(out), B * H * W, Cs, cpad)
    return out


def axpby(x, y, a: float, b: float, out=None):
    assert x.dtype == torch.float32 and y.dtype == torch.float32 and x.is_contiguous() and y.is_contiguous()
    if out is None:
        out = torch.empty_like(x)
    c = ctx(x.device.index)
    c.call("dk_axpby_f32", ptr(x), ptr(y), ptr(out), x.numel(), a, b)
    return out


def vae_sample_latent(hidden, noise, shift: float, scale: float, out=None):
    """hidden NHWC [B,H,W,2C] 16-bit (mean | logvar), noise fp32 [B,H,W,C] -> process_in(mean + std * noise) fp32"""
    _chk16(hidden, "vae_sample_latent.hidden")
    B, H, W, C2 = hidden.shape
    assert hidden.is_contiguous() and noise.dtype == torch.float32 and noise.is_contiguous()
    assert tuple(noise.shape) == (B, H, W, C2 // 2)
    if out is None:
        out = torch.empty((B, H, W, C2 // 2), dtype=torch.float32, device=hidden.device)
    assert out.dtype == torch.float32 and out.is_contiguous()
    c = ctx(hidden.device.index)
    c.call("dk_vae_sample_latent", dtype_code(hidden.dtype), ptr(hidden), ptr(noise), ptr(out), B * H * W, C2 // 2,
           shift, scale)
    return out


def cast_to_16(x, dtype, out=None):
    assert x.dtype == torch.float32 and x.is_contiguous()
    if out is None:
        out = torch.empty(x.shape, dtype=dtype, device=x.device)
    c = ctx(x.device.index)
    c.call("dk_cast_f32_to_16", dtype_code(dtype), ptr(x), ptr(out), x.numel())
    return out


def cast_to_f32(x, out=None):
    _chk16(x, "cast_to_f32.x")
    if out is None:
        out = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    c = ctx(x.device.index)
    c.call("dk_cast_16_to_f32", dtype_code(x.dtype), ptr(x), ptr(out), x.numel())
    return out


def residual_delta(x, base, nseq: int, rows: int, x_seq_rows: Optional[int] = None,
                   b_seq_rows: Optional[int] = None, r_out=None, prev=None, sums=None, ws=None):
    """r = fp32(x) - fp32(base) over nseq sequences of `rows` rows (x, base: 2-D 16-bit views whose row stride is the
    leading dimension; sequence s starts at row s * x_seq_rows, default rows).  r_out [nseq * rows, h] fp32 receives r;
    with prev (same shape), returns sums [nseq, 2] = (Σ|r - prev|, Σ|prev|) per sequence, reduced deterministically."""
    _chk16(x, "residual_delta.x")
    _chk16(base, "residual_delta.base")
    assert x.dim() == 2 and base.dim() == 2 and x.stride(1) == 1 and base.stride(1) == 1 and x.dtype == base.dtype
    h = x.shape[1]
    for t in (r_out, prev):
        assert t is None or (t.dtype == torch.float32 and t.is_contiguous() and t.numel() == nseq * rows * h)
    if prev is not None:
        if sums is None:
            sums = torch.empty((nseq, 2), dtype=torch.float32, device=x.device)
        if ws is None:
            ws = torch.empty((nseq * 512,), dtype=torch.float32, device=x.device)
        assert sums.dtype == torch.float32 and sums.numel() >= 2 * nseq and ws.numel() >= 512 * nseq
    c = ctx(x.device.index)
    c.call("dk_residual_delta", dtype_code(x.dtype), ptr(x), x.stride(0), rows if x_seq_rows is None else x_seq_rows,
           ptr(base), base.stride(0), rows if b_seq_rows is None else b_seq_rows, ptr(r_out), ptr(prev), ptr(sums),
           ptr(ws), nseq, rows, h)
    return sums


def residual_apply(x, r, out=None):
    """out = round16(x + r): x 16-bit, r fp32, both contiguous with the same number of elements; out may be x."""
    _chk16(x, "residual_apply.x")
    assert x.is_contiguous() and r.dtype == torch.float32 and r.is_contiguous() and r.numel() == x.numel()
    if out is None:
        out = torch.empty_like(x)
    assert out.dtype == x.dtype and out.is_contiguous() and out.numel() == x.numel()
    c = ctx(x.device.index)
    c.call("dk_residual_apply", dtype_code(x.dtype), ptr(x), ptr(r), ptr(out), x.numel())
    return out


def groupnorm_stats(x, G: int, eps: float = 1e-5, ws=None):
    """x NHWC [B, H, W, C] -> stats [B, G, 2] (mean, rstd)."""
    _chk16(x, "groupnorm_stats.x")
    B, H, W, Cc = x.shape
    c = ctx(x.device.index)
    n_ws = c.lib.dk_groupnorm_ws_floats(B, G)
    if ws is None:
        ws = torch.empty(n_ws, dtype=torch.float32, device=x.device)
    assert ws.numel() >= n_ws
    stats = torch.empty((B, G, 2), dtype=torch.float32, device=x.device)
    c.call("dk_groupnorm_stats", dtype_code(x.dtype), ptr(x), ptr(stats), ptr(ws), B, H * W, Cc, G, eps)
    return stats


def groupnorm_apply(x, stats, gamma, beta, G: int, silu: bool, out=None):
    _chk16(x, "groupnorm_apply.x")
    B, H, W, Cc = x.shape
    if out is None:
        out = torch.empty_like(x)
    c = ctx(x.device.index)
    c.call("dk_groupnorm_apply", dtype_code(x.dtype), ptr(x), ptr(out), ptr(stats), ptr(gamma), ptr(beta), B, H * W, Cc,
           G, 1 if silu else 0)
    return out


def conv3x3(x, w, bias=None, res=None, out=None):
    """x NHWC [B,H,W,Cin], w [Cout,3,3,Cin] -> NHWC [B,H,W,Cout] (+ res)."""
    _chk16(x, "conv3x3.x")
    B, H, W, Cin = x.shape
    Cout = w.shape[0]
    assert w.shape == (Cout, 3, 3, Cin) and x.is_contiguous() and w.is_contiguous()
    if out is None:
        out = torch.empty((B, H, W, Cout), dtype=x.dtype, device=x.device)
    c = ctx(x.device.index)
    c.call("dk_conv3x3", dtype_code(x.dtype), ptr(x), ptr(w), ptr(bias), ptr(res), ptr(out), B, H, W, Cin, Cout)
    return out


def conv3x3_s2(x, w, bias=None, out=None):
    """stride-2 3x3 conv with bottom/right zero padding: x NHWC [B,H,W,Cin] -> [B,H/2,W/2,Cout]"""
    _chk16(x, "conv3x3_s2.x")
    B, H, W, Cin = x.shape
    Cout = w.shape[0]
    assert w.shape == (Cout, 3, 3, Cin) and x.is_contiguous() and w.is_contiguous()
    if out is None:
        out = torch.empty((B, H // 2, W // 2, Cout), dtype=x.dtype, device=x.device)
    c = ctx(x.device.index)
    c.call("dk_conv3x3_s2", dtype_code(x.dtype), ptr(x), ptr(w), ptr(bias), ptr(out), B, H, W, Cin, Cout)
    return out


def conv_fused_supported(H: int, W: int, Cin: int, Cout: int) -> bool:
    return bool(_lib.load().dk_conv_fused_supported(H, W, Cin, Cout))


def conv_up_weights(w):
    """w [Cout,3,3,Cin] -> phase weights [4*Cout, 4*Cin] of conv3x3(nearest2x(.)) (see dk_conv_up_weights)"""
    _chk16(w, "conv_up_weights.w")
    Cout, _, _, Cin = w.shape
    assert w.shape == (Cout, 3, 3, Cin) and w.is_contiguous()
    wp = torch.empty((4 * Cout, 4 * Cin), dtype=w.dtype, device=w.device)
    c = ctx(w.device.index)
    c.call("dk_conv_up_weights", dtype_code(w.dtype), ptr(w), ptr(wp), Cout, Cin)
    return wp


def conv3x3_fused(x, w, bias=None, res=None, out=None, up: bool = False, gn=None, silu: bool = False,
                  out_partial=None, out_G: int = 32):
    """fused [GroupNorm+SiLU] -> [nearest 2x] -> conv3x3 (+bias, +res) -> out (+ output GroupNorm partial sums).
    gn = (stats [B,G,2] fp32, gamma [Cin], beta [Cin], G) or None; up: w must be conv_up_weights(w3x3)."""
    _chk16(x, "conv3x3_fused.x")
    B, H, W, Cin = x.shape
    if up:
        Cout = w.shape[0] // 4
        assert tuple(w.shape) == (4 * Cout, 4 * Cin)
        Ho, Wo = 2 * H, 2 * W
    else:
        Cout = w.shape[0]
        assert tuple(w.shape) == (Cout, 3, 3, Cin)
        Ho, Wo = H, W
    assert x.is_contiguous() and w.is_contiguous()
    if out is None:
        out = torch.empty((B, Ho, Wo, Cout), dtype=x.dtype, device=x.device)
    assert tuple(out.shape) == (B, Ho, Wo, Cout) and out.is_contiguous()
    if res is not None:
        assert tuple(res.shape) == tuple(out.shape) and res.is_contiguous()
    stats = gamma = beta = None
    G = 0
    if gn is not None:
        stats, gamma, beta, G = gn
        assert stats.dtype == torch.float32 and stats.is_contiguous() and tuple(stats.shape) == (B, G, 2)
    if out_partial is not None:
        assert out_partial.dtype == torch.float32 and out_partial.is_contiguous()
        assert out_partial.numel() >= B * (Ho * Wo // 128) * out_G * 2
    c = ctx(x.device.index)
    c.call("dk_conv3x3_fused", dtype_code(x.dtype), ptr(x), ptr(w), ptr(bias), ptr(res), ptr(out), B, H, W, Cin, Cout,
           1 if up else 0, ptr(stats), ptr(gamma), ptr(beta), G, 1 if silu else 0, ptr(out_partial), out_G)
    return out


def groupnorm_finalize(partial, B: int, G: int, slots: int, count: float, eps: float = 1e-5, stats=None):
    """partial [B, slots, G, 2] (sum, sumsq) -> stats [B, G, 2] (mean, rstd)"""
    assert partial.dtype == torch.float32 and partial.is_contiguous()
    if stats is None:
        stats = torch.empty((B, G, 2), dtype=torch.float32, device=partial.device)
    c = ctx(partial.device.index)
    c.call("dk_groupnorm_finalize", ptr(partial), ptr(stats), B, G, slots, float(count), eps)
    return stats


def upsample_nearest2x(x, out=None):
    _chk16(x, "upsample.x")
    B, H, W, Cc = x.shape
    if out is None:
        out = torch.empty((B, 2 * H, 2 * W, Cc), dtype=x.dtype, device=x.device)
    c = ctx(x.device.index)
    c.call("dk_upsample_nearest2x", dtype_code(x.dtype), ptr(x), ptr(out), B, H, W, Cc)
    return out


def softmax_rows(x, scale: float = 1.0):
    _chk16(x, "softmax_rows.x")
    assert x.dim() == 2 and x.stride(1) == 1
    c = ctx(x.device.index)
    c.call("dk_softmax_rows", dtype_code(x.dtype), ptr(x), x.shape[0], x.shape[1], x.stride(0), scale)
    return x


def image_post(x, want_u8: bool = True):
    """decoder output NHWC [B,H,W,Cpad] -> (float [B,H,W,3] in [0,1], uint8 [B,H,W,3])."""
    _chk16(x, "image_post.x")
    B, H, W, Cp = x.shape
    f = torch.empty((B, H, W, 3), dtype=torch.float32, device=x.device)
    u = torch.empty((B, H, W, 3), dtype=torch.uint8, device=x.device) if want_u8 else None
    c = ctx(x.device.index)
    c.call("dk_image_post", dtype_code(x.dtype), ptr(x), Cp, ptr(f), ptr(u), B * H * W)
    return f, u
