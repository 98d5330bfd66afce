"""GPU checks of the individual sm_90a kernels against plain fp32 torch references of the same op.

Each check_* function is self-contained (used by tests/test_kernels_gpu.py and by tools/run_gpu_checks.py, which
runs every check in its own process so that one trapped kernel cannot poison the others).  A check runs a table of
cases; every case of an op, small or full-size, is compared with that op's one ref_* function.
Tolerances: 16-bit outputs, fp32 accumulation -> relative L2 error <= 4e-3 (bf16 epsilon is 3.9e-3 per element,
the L2 over many elements averages to ~2e-3); attention <= 1e-2.
"""
import math
import os

import numpy as np
import torch

from diffusionkit_b200 import ops
from diffusionkit_b200._lib import ACT_GELU_ERF, ACT_NONE, ACT_QUICK_GELU, ACT_SILU

DEV = "cuda:0"
bf16, fp16 = torch.bfloat16, torch.float16


def _setup():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.manual_seed(0)


def rel_l2(a, b):
    a = a.float()
    b = b.float()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _dump(name, **arrs):
    d = os.environ.get("DK_DUMP_DIR")
    if not d:
        return
    os.makedirs(d, exist_ok=True)
    np.savez_compressed(os.path.join(d, name + ".npz"), **{k: v.float().cpu().numpy() for k, v in arrs.items()})


def _assert_close(name, got, ref, tol):
    err = rel_l2(got, ref)
    finite = bool(torch.isfinite(got.float()).all())
    if not finite or not err <= tol:
        _dump(name, got=got, ref=ref)
        raise AssertionError(f"{name}: rel_l2={err:.3e} (tol {tol:.1e}) finite={finite}")
    return err


def _rand(shape, dtype, scale=1.0):
    return (torch.randn(shape, device=DEV, dtype=torch.float32) * scale).to(dtype)


# ------------------------------------------------------------------------------------------------ fp32 references
def ref_gemm(A, W, bias=None, act=ACT_NONE, gate=None, res=None, *, rows_per_batch=0, res_batch_rows=None,
             res_row_off=0, N=None, w_n_major=False):
    """res + gate * act(A @ W^T + bias) in fp32 with dk_gemm's addressing (include/dkb200.h).  W is [N, K], or [K, N]
    when w_n_major; only its first N output features are used (N: the call's N, default all).  Row m is gated by gate
    row m // rows_per_batch and adds residual row (m / rows_per_batch) * res_batch_rows + res_row_off +
    m % rows_per_batch (res_batch_rows defaults to rows_per_batch; 0 broadcasts the same rows to every batch).  With
    rows_per_batch = 0 all M rows are one batch, except that a gate of G rows then gates G equal row batches (the form
    the table checks use).  The product runs in row chunks: the fp32 copy of a 16384 x 12288 output alone is 805 MB."""
    M = A.shape[0]
    Wt = W.float() if w_n_major else W.float().t()
    if N is not None:
        Wt = Wt[:, :N]
    Wt = Wt.contiguous()
    n = Wt.shape[1]
    y = torch.cat([A[i:i + 4096].float() @ Wt for i in range(0, M, 4096)], 0)
    if bias is not None:
        y += bias.float()[:n]
    if act == ACT_GELU_ERF:
        y = torch.nn.functional.gelu(y)
    elif act == ACT_SILU:
        y = torch.nn.functional.silu(y)
    elif act == ACT_QUICK_GELU:
        y = y * torch.sigmoid(1.702 * y)
    m = torch.arange(M, device=y.device)
    if gate is not None:
        g = gate.float()[:, :n]
        if rows_per_batch:
            y *= g[m // rows_per_batch]
        else:
            y = (y.reshape(g.shape[0], -1, n) * g[:, None]).reshape(y.shape)
    if res is not None:
        if rows_per_batch:
            rbr = rows_per_batch if res_batch_rows is None else res_batch_rows
            rrow = (m // rows_per_batch) * rbr + res_row_off + m % rows_per_batch
        else:
            rrow = res_row_off + m
        y += res.float()[rrow, :n]
    return y


def gemm_out_rows(M, rows_per_batch=0, out_batch_rows=0, out_row_off=0, device=DEV):
    """the output row dk_gemm writes row m of the product to: (m / rows_per_batch) * out_batch_rows + out_row_off +
    m % rows_per_batch (rows_per_batch = 0: out_row_off + m)"""
    m = torch.arange(M, device=device)
    if not rows_per_batch:
        return out_row_off + m
    return (m // rows_per_batch) * out_batch_rows + out_row_off + m % rows_per_batch


def ref_qk_norm_rope(y, pos, heads, d, q_w, k_w, rope, round_to=None, eps=1e-6):
    """QK-RMSNorm + RoPE in fp32 on the q and k thirds of a packed [rows, 3 * heads * d] y; v passes through.
    q_w / k_w: [d] or per-row [rows, 1, d] norm weights, None skips the norm.  rope[pos[row]]: the row's (cos, sin)
    pairs, None skips the rotation.  round_to: the 16-bit type the unfused dk_qk_norm_rope stores the normalised value
    in before it rotates it; the fused GEMM epilogue rotates it unrounded (None)."""
    h = heads * d
    y = y.float()
    ref = y.clone()
    for which, w in enumerate([q_w, k_w]):
        t = y[:, which * h:(which + 1) * h].reshape(-1, heads, d)
        if w is not None:
            t = t * torch.rsqrt((t * t).mean(-1, keepdim=True) + eps) * w.float()
            if round_to is not None:
                t = t.to(round_to).float()
        if rope is not None:
            c, sn = rope[pos][:, None, :, 0], rope[pos][:, None, :, 1]
            x0, x1 = t[..., 0::2], t[..., 1::2]
            t = torch.stack([x0 * c - x1 * sn, x0 * sn + x1 * c], dim=-1).reshape(-1, heads, d)
        ref[:, which * h:(which + 1) * h] = t.reshape(-1, h)
    return ref


def ref_attention(qkv, B, S, heads, d):
    """softmax(q k^T / sqrt(d)) v in fp32 for a packed [B * S, 3 * heads * d] qkv -> [B * S, heads * d], one head at a
    time (a 4685^2 fp32 score matrix is 88 MB)"""
    h = heads * d
    x = qkv.reshape(B, S, 3, heads, d)
    ref = torch.empty((B, S, h), dtype=torch.float32, device=qkv.device)
    for b in range(B):
        for hd in range(heads):
            q, k, v = x[b, :, 0, hd].float(), x[b, :, 1, hd].float(), x[b, :, 2, hd].float()
            ref[b, :, hd * d:(hd + 1) * d] = torch.softmax(q @ k.t() / math.sqrt(d), dim=-1) @ v
    return ref.reshape(B * S, h)


def ref_conv3x3(x, w, b, res=None):
    """3x3 convolution, zero padding 1, of NHWC x with w [Cout, 3, 3, Cin] + b (+ res) in fp32.  It runs in horizontal
    bands with a one-row halo, so a full-size image needs little fp32 scratch."""
    B, H, W, Cin = x.shape
    Cout = w.shape[0]
    wf = w.float().permute(0, 3, 1, 2).contiguous()
    ref = torch.empty((B, H, W, Cout), dtype=torch.float32, device=x.device)
    rows = max(8, (1 << 24) // (W * max(Cin, Cout)))
    for i in range(B):
        for y0 in range(0, H, rows):
            y1 = min(H, y0 + rows)
            xin = x[i, max(0, y0 - 1):min(H, y1 + 1)].float().permute(2, 0, 1)[None]
            xin = torch.nn.functional.pad(xin, (1, 1, 1 if y0 == 0 else 0, 1 if y1 == H else 0))
            ref[i, y0:y1] = torch.nn.functional.conv2d(xin, wf, b.float())[0].permute(1, 2, 0)
    if res is not None:
        ref += res.float()
    return ref


def ref_groupnorm_stats(x, G=32, eps=1e-5):
    """GroupNorm(G) statistics of NHWC x in float64, one image at a time -> (mean [B, G], rstd [B, G]) float64"""
    B, Cc = x.shape[0], x.shape[-1]
    mean = torch.empty((B, G), dtype=torch.float64, device=x.device)
    var = torch.empty_like(mean)
    for i in range(B):
        xd = x[i].reshape(-1, G, Cc // G).double()
        mean[i], var[i] = xd.mean(dim=(0, 2)), xd.var(dim=(0, 2), unbiased=False)
        del xd
    return mean, torch.rsqrt(var + eps)


def ref_groupnorm_apply(x, stats, gamma, beta, G=32, silu=True):
    """(x - mean) * rstd * gamma + beta of NHWC x with the given statistics [B, G, 2] (mean, rstd), rounded to x's
    16-bit type as dk_groupnorm_apply and the fused convolution round it, then SiLU -> fp32"""
    B, Cc = x.shape[0], x.shape[-1]
    y = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    for i in range(B):
        xg = x[i].reshape(-1, G, Cc // G).float()
        xn = (xg - stats[i, :, 0].float()[None, :, None]) * stats[i, :, 1].float()[None, :, None]
        v = (xn.reshape(x[i].shape) * gamma.float() + beta.float()).to(x.dtype).float()
        y[i] = torch.nn.functional.silu(v) if silu else v
    return y


def ref_groupnorm_silu(x, gamma, beta, G=32, eps=1e-5):
    """GroupNorm(G) + SiLU of NHWC x with float64 statistics (ref_groupnorm_stats, ref_groupnorm_apply).
    Returns (y fp32, mean [B, G], rstd [B, G])."""
    mean, rstd = ref_groupnorm_stats(x, G, eps)
    y = ref_groupnorm_apply(x, torch.stack([mean, rstd], -1), gamma, beta, G, True)
    return y, mean.float(), rstd.float()


def ref_conv3x3_s2(x, w, b):
    """the encoder's downsample: pad bottom/right by one, then 3x3 stride 2 without padding (mlx/vae.py:142-144)"""
    xp = torch.nn.functional.pad(x.float().permute(0, 3, 1, 2), (0, 1, 0, 1))
    return torch.nn.functional.conv2d(xp, w.float().permute(0, 3, 1, 2), b.float(), stride=2).permute(0, 2, 3, 1)


def ref_conv_up_weights(w):
    """phase weights [4 * Cout, 4 * Cin] of conv3x3(nearest2x(.)) from w [Cout, 3, 3, Cin]: row phase * Cout + n,
    column tap * Cin + c, phase = 2 py + px, tap = 2 a + b; tap (a, b) of phase (py, px) sums the 3x3 taps that land on
    the same source pixel (py = 0: a = 0 <- ky {0}, a = 1 <- ky {1, 2}; py = 1: a = 0 <- ky {0, 1}, a = 1 <- ky {2};
    the same in x), in fp32, rounded once"""
    Cout, _, _, Cin = w.shape
    rng = {(0, 0): (0, 1), (0, 1): (1, 3), (1, 0): (0, 2), (1, 1): (2, 3)}     # (phase bit, tap bit) -> ky range
    wf = w.float()
    wp = torch.zeros((4, Cout, 4, Cin), dtype=torch.float32, device=w.device)
    for py in range(2):
        for px in range(2):
            for a in range(2):
                for b in range(2):
                    (y0, y1), (x0, x1) = rng[(py, a)], rng[(px, b)]
                    for ky in range(y0, y1):                        # the kernel's summation order
                        for kx in range(x0, x1):
                            wp[2 * py + px, :, 2 * a + b] += wf[:, ky, kx]
    return wp.reshape(4 * Cout, 4 * Cin).to(w.dtype)


def ref_conv_partial_stats(y, G=32, up=False):
    """the fused convolution's output statistics: per image, per slot of 128 stored output pixels and per group,
    (sum, sum of squares) of the stored NHWC y in float64 -> [B, H * W / 128, G, 2].  A slot is 128 consecutive pixels
    of an output row, or with up (nearest 2x) the 128 pixels of one column phase of a 256-pixel row segment."""
    B, H, W, Cc = y.shape
    if up:
        y = y.reshape(B, H, W // 256, 128, 2, Cc).permute(0, 1, 2, 4, 3, 5)
    yd = y.reshape(B, -1, 128, G, Cc // G).double()
    return torch.stack([yd.sum(dim=(2, 4)), yd.square().sum(dim=(2, 4))], -1)


def ref_groupnorm_finalize(partial, count, eps=1e-5):
    """partial [B, slots, G, 2] (sum, sum of squares) -> [B, G, 2] (mean, rstd), folded in float64"""
    s = partial.double().sum(dim=1)
    mean = s[..., 0] / count
    var = s[..., 1] / count - mean * mean
    return torch.stack([mean, torch.rsqrt(var + eps)], -1)


def ref_ln_modulate(x, shift, scale, rows_per_batch, eps=1e-6):
    """LN(x) * (1 + scale[b]) + shift[b] in fp32, b = row // rows_per_batch; shift / scale [>= B, h] (any row stride)"""
    b = torch.arange(x.shape[0], device=x.device) // rows_per_batch
    ln = torch.nn.functional.layer_norm(x.float(), (x.shape[1],), eps=eps)
    return ln * (1 + scale.float()[b]) + shift.float()[b]


def ref_layernorm(x, weight, bias, eps=1e-5):
    return torch.nn.functional.layer_norm(x.float(), (x.shape[-1],), weight.float(), bias.float(), eps)


def ref_rmsnorm_f32(x, weight, eps=1e-6):
    """T5's RMSNorm of the fp32 residual stream: weight * x * rsqrt(mean(x^2) + eps)"""
    return weight.float() * x * torch.rsqrt(x.square().mean(-1, keepdim=True) + eps)


def ref_glu_gelu(h):
    """gelu(h[:, :F]) * h[:, F:] for h [rows, 2F]"""
    F = h.shape[1] // 2
    return torch.nn.functional.gelu(h.float()[:, :F]) * h.float()[:, F:]


def ref_silu_add(y, temb):
    """out[t * B + b] = silu(round16(y[b] + temb[t]))"""
    return torch.nn.functional.silu((y.float()[None] + temb.float()[:, None]).to(y.dtype).float()).reshape(
        -1, y.shape[1])


def ref_act(x, kind):
    if kind == ACT_SILU:
        return torch.nn.functional.silu(x.float())
    if kind == ACT_GELU_ERF:
        return torch.nn.functional.gelu(x.float())
    if kind == ACT_QUICK_GELU:
        return x.float() * torch.sigmoid(1.702 * x.float())
    return x.float()


def ref_attention_small(qkv, B, S, heads, scale, rel_bias=None, causal=False):
    """softmax(scale q k^T + rel_bias[h, j - i + S - 1] (+ causal mask)) v in fp32 over a packed [B * S, 3 * heads * 64]
    qkv -> [B * S, heads * 64]"""
    q, k, v = [t.reshape(B, S, heads, 64).permute(0, 2, 1, 3).float() for t in qkv.split(heads * 64, dim=1)]
    s = scale * (q @ k.transpose(-1, -2))
    i = torch.arange(S, device=qkv.device)
    if rel_bias is not None:
        s = s + rel_bias.float()[:, (i[None, :] - i[:, None]) + S - 1][None]
    if causal:
        s = s + (i[:, None] < i[None]).float() * -6e4
    return (torch.softmax(s, dim=-1) @ v).permute(0, 2, 1, 3).reshape(B * S, heads * 64)


def ref_softmax_rows(x, scale=1.0):
    """row softmax of scale * x in fp32, in row chunks (a 16384^2 fp32 score matrix is 1 GB)"""
    return torch.cat([torch.softmax(x[i:i + 2048].float() * scale, dim=-1) for i in range(0, x.shape[0], 2048)], 0)


def ref_image_post(x):
    """decoder output NHWC [B, H, W, Cpad] -> (float [B, H, W, 3] in [0, 1], uint8), rounded as dk_image_post rounds"""
    dt = x.dtype
    v = ((x[..., :3].float() * 0.5).to(dt).float() + 0.5).to(dt).float().clamp(0, 1)
    return v, (v * 255).to(dt).float().to(torch.uint8)


def ref_image_pre(img_u8, dtype, cpad=64):
    """uint8 NHWC -> 16-bit [B, H, W, cpad] in [-1, 1], channels 3.. zero.  Evaluated on the CPU: torch's CUDA
    division by a scalar multiplies by the reciprocal, the reference (and dk_image_pre) divide."""
    ref = torch.zeros((*img_u8.shape[:3], cpad), dtype=torch.float32)
    ref[..., :3] = img_u8.cpu()[..., :3].float() / 255 * 2 - 1.0
    return ref.to(dtype).to(img_u8.device)


def ref_vae_sample_latent(hidden, noise, shift, scale):
    """(mean + exp(0.5 clamp(logvar, -30, 20)) * noise - shift) * scale, hidden = (mean | logvar)"""
    mean, logvar = hidden.float().split(hidden.shape[-1] // 2, dim=-1)
    return (mean + torch.exp(0.5 * logvar.clamp(-30.0, 20.0)) * noise - shift) * scale


def ref_patchify(latent, order):
    """[B, H, W, C] -> rows [B * H/2 * W/2, 4C]: order 0 (FLUX) packs (c, ph, pw), order 1 (SD3) (ph, pw, c)"""
    B, H, W, Cc = latent.shape
    t = latent.reshape(B, H // 2, 2, W // 2, 2, Cc)
    t = t.permute(0, 1, 3, 5, 2, 4) if order == 0 else t.permute(0, 1, 3, 2, 4, 5)
    return t.reshape(B * (H // 2) * (W // 2), 4 * Cc)


def ref_unpatchify(rows, B, H, W, Cc, order):
    if order == 0:
        t = rows.reshape(B, H // 2, W // 2, Cc, 2, 2).permute(0, 1, 4, 2, 5, 3)
    else:
        t = rows.reshape(B, H // 2, W // 2, 2, 2, Cc).permute(0, 1, 3, 2, 4, 5)
    return t.reshape(B, H, W, Cc)


def ref_pos_embed_crop(table, max_hw, hp, wp):
    """the centred hp x wp window of a max_hw x max_hw position table (reference mmdit.py:334-349)"""
    y0, x0 = (max_hw - hp) // 2, (max_hw - wp) // 2
    return table.reshape(max_hw, max_hw, -1)[y0:y0 + hp, x0:x0 + wp].reshape(hp * wp, -1)


def ref_embedding(table, ids, pos=None):
    """table[ids] (+ pos[i % len(pos)], summed in fp32 and rounded once)"""
    rows = table[ids.long().reshape(-1)]
    if pos is None:
        return rows
    i = torch.arange(rows.shape[0], device=table.device) % pos.shape[0]
    return (rows.float() + pos.float()[i]).to(table.dtype)


def ref_denoised(xin, out, sigma, cfg, n, slg=0.0):
    """the CFG (+ skip-layer guidance) mixed denoised estimate D every sampler kernel computes, in fp32: D = xin -
    out * sigma of [positive | negative | positive skipping layers] rows, D_neg + cfg (D_pos - D_neg) + slg (D_pos -
    D_skip)"""
    den = xin.reshape(-1).float() - out.reshape(-1).float() * sigma
    if cfg <= 0:
        return den[:n]
    mixed = den[n:2 * n] + cfg * (den[:n] - den[n:2 * n])
    if slg != 0.0:
        mixed = mixed + slg * (den[:n] - den[2 * n:3 * n])
    return mixed


def ref_sampler_step(x, xin, out, sigma, sigma_next, cfg, slg=0.0):
    """Euler: x + (x - D) / sigma * (sigma_next - sigma)"""
    d = (x - ref_denoised(xin, out, sigma, cfg, x.numel(), slg).reshape(x.shape)) / sigma
    return x + d * (sigma_next - sigma)


def ref_heun_predict(x, xin, out, sigma, sigma_next, cfg, slg=0.0):
    """-> (d, x2): the slope at (x, sigma) and the Euler step to sigma_next"""
    d = (x - ref_denoised(xin, out, sigma, cfg, x.numel(), slg).reshape(x.shape)) / sigma
    return d, x + d * (sigma_next - sigma)


def ref_heun_correct(x, d, x2, xin, out, sigma, sigma_next, cfg, slg=0.0):
    """x + (d + d2) / 2 * (sigma_next - sigma), d2 the slope of (xin, out) at (x2, sigma_next)"""
    d2 = (x2 - ref_denoised(xin, out, sigma_next, cfg, x.numel(), slg).reshape(x.shape)) / sigma_next
    return x + (d + d2) / 2 * (sigma_next - sigma)


def ref_dpmpp_2m(x, d_prev, xin, out, sigma, a, b, c, cfg, slg=0.0):
    """-> (a x + b D + c d_prev, D); d_prev is not read when c == 0"""
    den = ref_denoised(xin, out, sigma, cfg, x.numel(), slg).reshape(x.shape)
    return (a * x + b * den + (c * d_prev if c != 0.0 else 0.0)), den


def ref_residual_delta(x, base, nseq, rows, x_seq, b_seq, prev=None):
    """the step cache's residual r = fp32(x) - fp32(base) of nseq sequences of `rows` rows (sequence s at row s * x_seq
    of x, s * b_seq of base) -> (r [nseq * rows, h] fp32, with prev: float64 sums [nseq, 2] = (sum |r - prev|,
    sum |prev|) per sequence, else None)"""
    h = x.shape[1]
    xs = torch.stack([x[s * x_seq:s * x_seq + rows] for s in range(nseq)]).float()
    bs = torch.stack([base[s * b_seq:s * b_seq + rows] for s in range(nseq)]).float()
    r = (xs - bs).reshape(nseq * rows, h)
    if prev is None:
        return r, None
    pv = prev.reshape(nseq, rows, h).double()
    rd = r.reshape(nseq, rows, h).double()
    return r, torch.stack([(rd - pv).abs().sum(dim=(1, 2)), pv.abs().sum(dim=(1, 2))], dim=1)


# ------------------------------------------------------------------------------------------------ GEMM
def _gemm_case(M, N, K, dtype, epi="", block_tol=None):
    """dk_gemm vs ref_gemm.  epi lists the epilogue terms: bias, gelu | silu | quick_gelu, gate, res (out of place),
    inplace (residual read from and written to the output), remap (two batches of M / 2 rows scattered at row offset
    24 into 40-row-padded batches), window (a column window of a wider buffer, the FLUX single-block concat buffer),
    n_major (W given as [K, N]).  Bytes of a remap / window buffer outside the output must keep their sentinel."""
    e = set(epi.split())
    act = (ACT_GELU_ERF if "gelu" in e else ACT_SILU if "silu" in e else ACT_QUICK_GELU if "quick_gelu" in e
           else ACT_NONE)
    Bt = 2 if "remap" in e else 1
    A = _rand((M, K), dtype)
    W = _rand((K, N) if "n_major" in e else (N, K), dtype, 1 / math.sqrt(K))
    b = _rand((N,), dtype, 0.5) if "bias" in e else None
    g = _rand((Bt, N), dtype) if "gate" in e else None
    r = _rand((M, N), dtype) if e & {"res", "inplace"} else None
    ref = ref_gemm(A, W.t() if "n_major" in e else W, b, act, g, r)
    name = f"gemm_{M}x{N}x{K}_{str(dtype)[6:]}_{'_'.join(epi.split()) or 'plain'}"
    out, buf, kw = (r if "inplace" in e else None), None, {}
    if "remap" in e:
        rpb, out_rows, off = M // Bt, M // Bt + 40, 24
        buf = out = torch.full((Bt * out_rows, N), 7.0, dtype=dtype, device=DEV)
        rows = torch.cat([torch.arange(i * out_rows + off, i * out_rows + off + rpb) for i in range(Bt)]).to(DEV)
        window = (rows, slice(0, N))
        kw = dict(rows_per_batch=rpb, out_batch_rows=out_rows, out_row_off=off)
    elif "window" in e:
        buf = torch.full((M + 8, 1024), 7.0, dtype=dtype, device=DEV)
        window = (slice(0, M), slice(256, 256 + N))
        out = buf[window]
    got = ops.gemm(A, W, out=out, bias=b, act=act, gate=g, res=r, w_n_major="n_major" in e, **kw)
    if buf is not None:
        got = buf[window]
        outside = torch.ones(buf.shape, dtype=torch.bool, device=DEV)
        outside[window] = False
        assert bool((buf[outside] == 7.0).all()), f"{name}: bytes outside the output window were written"
    if block_tol is not None:
        return _assert_close_blocks(name, got, ref, 4e-3, block_tol)
    return _assert_close(name, got, ref, 4e-3)


def _gemm_table(cases):
    _setup()
    return {f"{M}x{N}x{K}_{epi}": _gemm_case(M, N, K, dt, epi) for (M, N, K, dt, epi) in cases}


def check_gemm_single_tile():
    _setup()
    return {"err": _gemm_case(128, 256, 64, bf16)}


def check_gemm_multi_k():
    _setup()
    return {"err": _gemm_case(128, 256, 512, bf16)}


def check_gemm_one_m_pair():
    """M = 256: one m-block pair, so both CTAs of a cluster own rows and share the W tile; one and several K steps"""
    return _gemm_table([(256, 256, 64, bf16, ""), (256, 512, 512, bf16, "")])


def check_gemm_shapes():
    """ragged M / N / K, tiny and tall problems"""
    return _gemm_table([(256, 512, 256, bf16, ""), (300, 264, 200, bf16, ""), (77, 64, 64, bf16, ""),
                        (1000, 3072, 1536, bf16, ""), (20, 1024, 3072, bf16, ""), (4352, 768, 3072, bf16, ""),
                        (128, 128, 128, bf16, "")])


def check_gemm_persistent_large():
    """more tiles than SMs: more than one wave of clusters and the smem ring wrap-around"""
    return _gemm_table([(4096, 4608, 1024, bf16, "bias"), (8192, 4608, 1024, bf16, "bias"),
                        (4096, 3072, 512, bf16, "bias")])


def check_gemm_epilogues():
    return _gemm_table([(384, 512, 256, bf16, "bias"), (384, 512, 256, bf16, "bias gelu"),
                        (384, 512, 256, bf16, "bias silu"), (384, 512, 256, bf16, "bias gate res"),
                        (600, 512, 256, bf16, "bias gate res remap"), (77, 512, 256, bf16, "bias quick_gelu")])


def check_gemm_gate_residual():
    """bias + gate + residual on multi-tile problems, one with N = 1152 (not a multiple of the 256-wide tile)"""
    return _gemm_table([(1024, 1152, 256, bf16, "bias gate res"), (2048, 1536, 512, bf16, "bias gate res")])


def check_gemm_output_window():
    """GELU output into a column window of a wider buffer (the FLUX single-block concat buffer), M and N not tile
    multiples: every byte left, right and below the window keeps its sentinel"""
    return _gemm_table([(1000, 520, 256, bf16, "gelu window")])


def check_gemm_fp16():
    return _gemm_table([(300, 512, 320, fp16, "bias gelu"), (300, 512, 320, fp16, "bias")])


def check_gemm_inplace_residual():
    return _gemm_table([(256, 256, 128, bf16, "inplace"), (1000, 520, 256, bf16, "gate inplace")])


def check_gemm_w_n_major():
    return _gemm_table([(128, 128, 64, bf16, "n_major"), (256, 384, 256, bf16, "n_major"),
                        (200, 136, 72, bf16, "n_major")])


# ------------------------------------------------------------------------------------------------ conv
def _conv_case(B, H, W, Cin, Cout, dtype, res=False, block_tol=None):
    x = _rand((B, H, W, Cin), dtype)
    w = _rand((Cout, 3, 3, Cin), dtype, 1 / math.sqrt(9 * Cin))
    b = _rand((Cout,), dtype, 0.5)
    r = _rand((B, H, W, Cout), dtype) if res else None
    ref = ref_conv3x3(x, w, b, r)
    got = ops.conv3x3(x, w, bias=b, res=r)
    name = f"conv_{B}x{H}x{W}_{Cin}to{Cout}_{str(dtype)[6:]}" + ("_res" if res else "")
    if block_tol is not None:
        return _assert_close_blocks(name, got.reshape(-1, Cout), ref.reshape(-1, Cout), 4e-3, block_tol,
                                    bc=min(128, Cout))
    return _assert_close(name, got, ref, 4e-3)


def check_conv3x3():
    _setup()
    return {f"{B}x{H}x{W}_{Cin}to{Cout}": _conv_case(B, H, W, Cin, Cout, dt, res)
            for (B, H, W, Cin, Cout, dt, res) in [(2, 16, 16, 64, 64, bf16, False), (1, 8, 32, 128, 128, bf16, True),
                                                  (2, 12, 20, 64, 72, bf16, False), (1, 64, 256, 128, 256, bf16, True),
                                                  (1, 32, 32, 64, 16, fp16, False)]}


def _conv_s2_case(B, H, W, Cin, Cout, dtype):
    x = _rand((B, H, W, Cin), dtype)
    w = _rand((Cout, 3, 3, Cin), dtype, 1 / math.sqrt(9 * Cin))
    b = _rand((Cout,), dtype, 0.5)
    ref = ref_conv3x3_s2(x, w, b)
    got = ops.conv3x3_s2(x, w, bias=b)
    assert got.shape == (B, H // 2, W // 2, Cout)
    return _assert_close(f"convs2_{B}x{H}x{W}_{Cin}to{Cout}_{str(dtype)[6:]}", got, ref, 4e-3)


def check_conv3x3_s2():
    """the encoder's stride-2 downsample: same implicit-GEMM kernel, TMA box with element stride 2"""
    _setup()
    return {f"{B}x{H}x{W}_{Cin}to{Cout}": _conv_s2_case(B, H, W, Cin, Cout, dt)
            for (B, H, W, Cin, Cout, dt) in [(2, 32, 32, 64, 64, bf16),        # TW=16, TH=8
                                             (1, 16, 64, 128, 128, bf16),      # TW=32, TH=4
                                             (2, 24, 40, 64, 72, bf16),        # TW=128 ragged
                                             (1, 64, 512, 128, 128, bf16),     # box 256 wide
                                             (1, 32, 32, 64, 16, fp16)]}


def check_img2img_kernels():
    """dk_image_pre, dk_vae_sample_latent, dk_axpby_f32 (read_image / posterior sample / noise_scaling)"""
    _setup()
    out = {}
    for dt in (torch.bfloat16, torch.float16):
        for cs in (3, 4):
            img = torch.randint(0, 256, (2, 8, 12, cs), dtype=torch.uint8, device=DEV)
            got = ops.image_pre(img, dt, 64)
            assert torch.equal(got, ref_image_pre(img, dt, 64)), f"image_pre {dt} {cs}"
    hidden = _rand((1, 8, 8, 32), torch.bfloat16, 2.0)
    hidden[0, 0, 0, 16] = 50.0       # logvar clipped at 20
    hidden[0, 0, 1, 16] = -80.0      # ... and at -30
    noise = torch.randn((1, 8, 8, 16), device=DEV)
    out["sample"] = _assert_close("vae_sample", ops.vae_sample_latent(hidden, noise, 0.0, 1.0),
                                  ref_vae_sample_latent(hidden, noise, 0.0, 1.0), 1e-5)
    out["sample_in"] = _assert_close("vae_sample_in", ops.vae_sample_latent(hidden, noise, 0.1159, 0.3611),
                                     ref_vae_sample_latent(hidden, noise, 0.1159, 0.3611), 1e-5)
    a, b = torch.randn(1000, device=DEV), torch.randn(1000, device=DEV)
    out["axpby"] = _assert_close("axpby", ops.axpby(a, b, 0.7, 0.3), 0.7 * a + 0.3 * b, 1e-6)
    return out


def check_dequant_q4():
    """dk_dequant_q4 vs the numpy restatement of MLX's dequantisation rule: bit-exact in both 16-bit types"""
    import numpy as np

    from oracle import quant_ref as qr

    _setup()
    out = {}
    rng = np.random.RandomState(3)
    for (N, K, dt) in [(64, 256, torch.bfloat16), (200, 3072, torch.bfloat16), (72, 128, torch.float16)]:
        w = (rng.randn(N, K) / math.sqrt(K)).astype(np.float32)
        wq, sc, bi = qr.quantize_q4(w)
        sc16, bi16 = torch.from_numpy(sc).to(dt), torch.from_numpy(bi).to(dt)
        want = torch.from_numpy(qr.dequantize_q4(wq, sc16.float().numpy(), bi16.float().numpy())).to(dt)
        got = ops.dequant_q4(torch.from_numpy(wq.view(np.int32)).to(DEV), sc16.to(DEV), bi16.to(DEV))
        assert got.dtype == dt and torch.equal(got.cpu(), want), f"dequant_q4 {N}x{K} {dt}"
        out[f"{N}x{K}"] = rel_l2(got.cpu(), torch.from_numpy(w))       # quantisation error itself, for the record
    return out


def check_text_kernels():
    """csrc/text.cu: embedding, LayerNorm(affine), T5 RMSNorm over fp32, fp32 += 16-bit, gated GELU (the quick-GELU GEMM
    epilogue is a row of check_gemm_epilogues)"""
    _setup()
    out = {}
    for dt in (torch.bfloat16, torch.float16):
        table, pos = _rand((50, 128), dt), _rand((7, 128), dt)
        ids = torch.randint(0, 50, (3, 7), dtype=torch.int32, device=DEV)
        got = ops.embedding(table, ids.reshape(-1).contiguous(), pos=pos)
        assert torch.equal(got, ref_embedding(table, ids, pos)), f"embedding+pos {dt}"
        assert torch.equal(ops.embedding(table, ids.reshape(-1).contiguous()), ref_embedding(table, ids))
    for (rows, h, dt) in [(77, 768, torch.bfloat16), (154, 1280, torch.float16), (5, 128, torch.bfloat16)]:
        x, w, b = _rand((rows, h), dt, 2.0), _rand((h,), dt, 0.5) + 1.0, _rand((h,), dt, 0.3)
        ref = ref_layernorm(x, w, b, 1e-5)
        out[f"ln_{h}"] = _assert_close(f"layernorm_{h}", ops.layernorm(x, w, b, 1e-5), ref, 4e-3)
    for (rows, d, dt) in [(64, 4096, torch.bfloat16), (9, 256, torch.bfloat16), (3, 1000, torch.float16)]:
        x = torch.randn((rows, d), device=DEV) * 30.0
        w = _rand((d,), dt, 0.2) + 1.0
        ref = ref_rmsnorm_f32(x, w, 1e-6)
        out[f"rms_{d}"] = _assert_close(f"rmsnorm_f32_{d}", ops.rmsnorm_f32(x, w, 1e-6), ref, 4e-3)
    x32, y16 = torch.randn(4096, device=DEV), _rand((4096,), torch.bfloat16)
    assert torch.equal(ops.add_f32_16(x32.clone(), y16), x32 + y16.float())
    hgl = _rand((33, 2 * 512), torch.bfloat16, 2.0)
    out["glu"] = _assert_close("glu_gelu", ops.glu_gelu(hgl), ref_glu_gelu(hgl), 4e-3)
    return out


def _attention_small_case(B, S, heads, dt, causal, rel, scale, name):
    qkv = _rand((B * S, 3 * heads * 64), dt)
    rel_bias = _rand((heads, 2 * S - 1), dt, 2.0) if rel else None
    ref = ref_attention_small(qkv, B, S, heads, scale, rel_bias, causal)
    got = ops.attention_small(qkv, B, S, heads, scale, rel_bias=rel_bias, causal=causal)
    return _assert_close(name, got, ref, 6e-3)


def check_attention_small():
    """short-sequence attention (text encoders): CLIP causal mask, T5 relative bias, ragged and maximum lengths"""
    _setup()
    out = {}
    out["clip_77"] = _attention_small_case(2, 77, 12, torch.bfloat16, True, False, 0.125, "atts_clip77")
    out["clip_fp16_20h"] = _attention_small_case(1, 77, 20, torch.float16, True, False, 0.125, "atts_clip_fp16")
    out["t5_256"] = _attention_small_case(1, 256, 8, torch.bfloat16, False, True, 1.0, "atts_t5_256")
    out["t5_512"] = _attention_small_case(2, 512, 4, torch.bfloat16, False, True, 1.0, "atts_t5_512")
    out["ragged_33"] = _attention_small_case(1, 33, 2, torch.bfloat16, True, True, 0.5, "atts_33")
    out["one_token"] = _attention_small_case(1, 1, 1, torch.bfloat16, False, False, 1.0, "atts_1")
    c = ops.ctx(0)
    qkv = _rand((513, 192), torch.bfloat16)
    o = torch.empty((513, 64), dtype=torch.bfloat16, device=DEV)
    rc = c.lib.dk_attention_small(c.handle, 0, ops.ptr(qkv), None, ops.ptr(o), 1, 513, 1, 64, 1.0, 0, None)
    assert rc != 0 and b"512" in c.lib.dk_last_error()
    return out


# ------------------------------------------------------------------------------------------------ attention
def _attention_case(B, S, heads, d, dtype, split=None, out1_pad=64, block_tol=None, twice=False):
    """dk_attention_fwd vs ref_attention.  With a split, rows >= split of each sequence go to out1, a view whose rows
    are out1_pad elements longer than heads * d.  twice: a second launch on the same input must be bit-identical to
    the first (the K/V steps and the quad reductions run in a fixed order)."""
    h = heads * d
    qkv = _rand((B * S, 3 * h), dtype)

    def launch():
        if split is None:
            out = torch.zeros((B * S, h), dtype=dtype, device=DEV)
            ops.attention(qkv, B, S, heads, d, out)
            return out
        o0 = torch.zeros((B * split, h), dtype=dtype, device=DEV)
        o1 = torch.zeros((B * (S - split), h + out1_pad), dtype=dtype, device=DEV)[:, :h]
        ops.attention(qkv, B, S, heads, d, o0, split=split, out1=o1)
        return torch.cat([o0.reshape(B, split, h), o1.reshape(B, S - split, h)], dim=1).reshape(B * S, h)

    name = f"att_d{d}_{B}x{S}x{heads}_{str(dtype)[6:]}" + (f"_split{split}" if split is not None else "")
    got = launch()
    if twice:
        assert torch.equal(got, launch()), f"{name}: two launches on the same input differ"
    ref = ref_attention(qkv, B, S, heads, d)
    if block_tol is not None:
        return _assert_close_blocks(name, got, ref, 1e-2, block_tol, bc=d)
    return _assert_close(name, got, ref, 1e-2)


def _attention_table(cases):
    _setup()
    return {f"{B}x{S}x{heads}_split{split}": _attention_case(B, S, heads, d, dt, split)
            for (B, S, heads, d, dt, split) in cases}


def check_attention_d128_one_tile():
    _setup()
    return {"err": _attention_case(1, 128, 1, 128, bf16)}


def check_attention_d128():
    return _attention_table([(2, 300, 2, 128, bf16, None), (1, 1280, 3, 128, bf16, 256)])


def check_attention_d64():
    return _attention_table([(1, 128, 1, 64, fp16, None), (2, 1178, 2, 64, fp16, 1024), (1, 333, 2, 64, bf16, None)])


def check_attention_short():
    """a half-filled K/V tile and two full ones"""
    return _attention_table([(1, 64, 1, 128, bf16, None), (1, 256, 2, 128, bf16, None)])


def check_attention_long():
    """many K/V steps with a ragged last tile, with and without split outputs"""
    return _attention_table([(2, 1300, 2, 128, bf16, 1024), (1, 4400, 2, 128, bf16, None)])


def check_attention_many_ctas():
    """more (batch, head, query tile) work items than SMs, at both head dims"""
    return _attention_table([(3, 700, 24, 128, bf16, 100), (2, 1500, 24, 64, fp16, 1024)])


def check_attention_determinism():
    """long ragged sequences at both head dims: a second launch on the same input is bit-identical to the first"""
    _setup()
    return {"d128_S1300": _attention_case(2, 1300, 2, 128, bf16, twice=True),
            "d64_S1178": _attention_case(2, 1178, 2, 64, fp16, twice=True)}


def check_attention_large_scores():
    """rows whose running max keeps growing: exercises the lazy O rescale path."""
    _setup()
    B, S, heads, d = 1, 1024, 1, 128
    h = heads * d
    qkv = _rand((B * S, 3 * h), torch.bfloat16)
    # make later keys progressively more aligned with the queries
    ramp = torch.linspace(0.2, 6.0, S, device=DEV).unsqueeze(1)
    base = _rand((1, d), torch.bfloat16).float()
    qkv[:, :h] = (base * 2.0 + 0.3 * qkv[:, :h].float()).to(torch.bfloat16)
    qkv[:, h:2 * h] = (base * ramp + 0.3 * qkv[:, h:2 * h].float()).to(torch.bfloat16)
    out = torch.zeros((B * S, h), dtype=torch.bfloat16, device=DEV)
    ops.attention(qkv, B, S, heads, d, out)
    return {"err": _assert_close("att_rescale", out, ref_attention(qkv, B, S, heads, d), 1e-2)}


# ------------------------------------------------------------------------------------------------ elementwise
def check_ln_modulate():
    _setup()
    out = {}
    for (B, S, h, dt) in [(2, 37, 3072, torch.bfloat16), (1, 64, 1536, torch.float16), (3, 5, 128, torch.bfloat16)]:
        x = _rand((B * S, h), dt, 2.0) + 0.5
        mod = _rand((B, 6 * h), dt, 0.3)
        shift, scale = mod[:, 0:h], mod[:, h:2 * h]
        ref = ref_ln_modulate(x, shift, scale, S, 1e-6)
        got = ops.ln_modulate(x, shift, scale, S, 1e-6)
        out[f"{B}x{S}x{h}"] = _assert_close(f"ln_{h}", got, ref, 4e-3)
    return out


def _rope_table(S, d, device):
    ang = torch.rand((S, d // 2), device=device) * 6.28
    return torch.stack([torch.cos(ang), torch.sin(ang)], dim=-1).contiguous()


def check_qk_norm_rope():
    """the unfused dk_qk_norm_rope: rows before split use the first pair of norm weights, the rest the second"""
    _setup()
    out = {}
    for (B, S, heads, d, dt, use_norm, use_rope) in [(2, 50, 3, 128, torch.bfloat16, True, True),
                                                     (1, 33, 2, 64, torch.float16, True, False),
                                                     (1, 40, 2, 128, torch.bfloat16, False, True)]:
        qkv = _rand((B * S, 3 * heads * d), dt)
        split = S // 3
        ws = [(_rand((d,), dt, 0.1) + 1.0) for _ in range(4)] if use_norm else [None] * 4
        rope = _rope_table(S, d, DEV) if use_rope else None
        pos = torch.arange(B * S, device=DEV) % S
        first = (pos < split)[:, None, None]
        qw, kw = ([torch.where(first, w1.float(), w2.float()) for w1, w2 in ((ws[0], ws[2]), (ws[1], ws[3]))]
                  if use_norm else (None, None))
        ref = ref_qk_norm_rope(qkv, pos, heads, d, qw, kw, rope, round_to=dt)
        got = ops.qk_norm_rope(qkv.clone(), S, heads, d, split, ws[0], ws[1], ws[2], ws[3], rope)
        out[f"d{d}_{use_norm}_{use_rope}"] = _assert_close(f"qknr_{d}", got, ref, 4e-3)
    return out


def check_gemm_fused_qk_norm_rope():
    """packed QKV projection with the QK-RMSNorm + RoPE epilogue == plain GEMM followed by dk_qk_norm_rope,
    and == an fp32 torch evaluation"""
    _setup()
    out = {}
    for (Bt, Ss, off, S, heads, d, dt, use_norm, use_rope) in [(2, 100, 28, 128, 2, 128, torch.bfloat16, True, True),
                                                               (1, 300, 0, 300, 4, 64, torch.float16, True, True),
                                                               (2, 77, 5, 90, 2, 128, torch.bfloat16, False, True)]:
        h = heads * d
        K = 192
        A = _rand((Bt * Ss, K), dt)
        W = _rand((3 * h, K), dt, 1 / math.sqrt(K))
        bias = _rand((3 * h,), dt, 0.3)
        qw = (_rand((d,), dt, 0.1) + 1.0) if use_norm else None
        kw = (_rand((d,), dt, 0.1) + 1.0) if use_norm else None
        rope = _rope_table(S, d, DEV) if use_rope else None
        fused = torch.zeros((Bt * S, 3 * h), dtype=dt, device=DEV)
        ops.gemm(A, W, out=fused, bias=bias, rows_per_batch=Ss, out_batch_rows=S, out_row_off=off,
                 qk=(heads, d, qw, kw, rope, 1e-6))
        plain = torch.zeros((Bt * S, 3 * h), dtype=dt, device=DEV)
        ops.gemm(A, W, out=plain, bias=bias, rows_per_batch=Ss, out_batch_rows=S, out_row_off=off)
        ops.qk_norm_rope(plain, S, heads, d, S, qw, kw, None, None, rope)
        rows = torch.cat([torch.arange(b * S + off, b * S + off + Ss) for b in range(Bt)]).to(DEV)
        out[f"vs_unfused_d{d}_{use_norm}"] = _assert_close(f"fusedqk_{d}", fused[rows], plain[rows], 3e-3)
        other = torch.ones(Bt * S, dtype=torch.bool, device=DEV)
        other[rows] = False
        if bool(other.any()):
            assert float(fused[other].float().abs().max()) == 0.0, "rows outside the scatter window were written"
        pos = (torch.arange(Bt * Ss, device=DEV) % Ss) + off
        ref = ref_qk_norm_rope(ref_gemm(A, W, bias), pos, heads, d, qw, kw, rope)
        out[f"vs_fp32_d{d}_{use_norm}"] = _assert_close(f"fusedqk_ref_{d}", fused[rows], ref, 6e-3)
    return out


def check_layout_kernels():
    _setup()
    out = {}
    dt = torch.bfloat16
    B, H, W, Cc = 2, 8, 12, 16
    lat = _rand((B, H, W, Cc), dt)
    # FLUX order (c, ph, pw) — reference mmdit.py:292-302
    ref0 = ref_patchify(lat, 0)
    got0 = ops.patchify(lat, 0)
    assert torch.equal(got0, ref0), "patchify order 0"
    # SD3 order (ph, pw, c)
    ref1 = ref_patchify(lat, 1)
    got1 = ops.patchify(lat, 1)
    assert torch.equal(got1, ref1), "patchify order 1"
    assert torch.equal(ops.unpatchify(got0, B, H, W, Cc, 0), lat), "unpatchify order 0"
    assert torch.equal(ops.unpatchify(got1, B, H, W, Cc, 1), lat), "unpatchify order 1"
    assert torch.equal(ref_unpatchify(ref0, B, H, W, Cc, 0), lat) and torch.equal(ref_unpatchify(ref1, B, H, W, Cc, 1), lat)
    # pos-embed crop — reference mmdit.py:334-349
    max_hw, hp, wp, h = 12, 4, 6, 64
    table = _rand((max_hw * max_hw, h), dt)
    refc = ref_pos_embed_crop(table, max_hw, hp, wp)
    assert torch.equal(ops.pos_embed_crop(table, max_hw, hp, wp), refc), "pos_embed_crop"
    # copy_rows
    src = _rand((2, 5, 64), dt)
    dst = torch.zeros((2, 9, 64), dtype=dt, device=DEV)
    ops.copy_rows(src, dst, 2, 5, 64, 9, 3, 5, 0)
    assert torch.equal(dst[:, 3:8], src) and float(dst[:, :3].float().abs().max()) == 0
    # silu_add / act
    y = _rand((3, 128), dt)
    temb = _rand((4, 128), dt)
    out["silu_add"] = _assert_close("silu_add", ops.silu_add(y, temb), ref_silu_add(y, temb), 4e-3)
    out["act_silu"] = _assert_close("act_silu", ops.act(y, ACT_SILU), ref_act(y, ACT_SILU), 4e-3)
    # upsample
    x = _rand((2, 3, 5, 16), dt)
    refu = x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    assert torch.equal(ops.upsample_nearest2x(x), refu), "upsample"
    return out


def check_sampler_kernels():
    _setup()
    dt = torch.bfloat16
    n = 2 * 8 * 8 * 16
    x = torch.randn(n, device=DEV)
    out = {}
    for cfg in (0.0, 5.0):
        reps = 2 if cfg > 0 else 1
        xin = torch.empty(reps * n, dtype=dt, device=DEV)
        ops.sampler_prepare(x, xin, reps)
        assert torch.equal(xin[:n], x.to(dt)) and torch.equal(xin[-n:], x.to(dt))
        mo = _rand((reps * n,), dt)
        sigma, sigma_next = 0.75, 0.5
        ref = ref_sampler_step(x, xin, mo, sigma, sigma_next, cfg)
        got = ops.sampler_step(x.clone(), xin, mo, sigma, sigma_next, cfg)
        out[f"cfg{cfg}"] = _assert_close(f"sampler_{cfg}", got, ref, 1e-5)
    out["axpb"] = _assert_close("axpb", ops.axpb(x, 1 / 0.3611, 0.1159), x / 0.3611 + 0.1159, 1e-6)
    assert torch.equal(ops.cast_to_16(x, dt), x.to(dt))
    assert torch.equal(ops.cast_to_f32(x.to(dt)), x.to(dt).float())
    return out


def _groupnorm_case(B, H, W, Cc, dt, mean=0.7, std=1.5):
    """dk_groupnorm_stats and dk_groupnorm_apply (+ SiLU) vs ref_groupnorm_silu, each image compared on its own"""
    x = _rand((B, H, W, Cc), dt, std) + mean
    gamma = _rand((Cc,), dt, 0.1) + 1.0
    beta = _rand((Cc,), dt, 0.1)
    ref, mean, rstd = ref_groupnorm_silu(x, gamma, beta, 32, 1e-5)
    stats = ops.groupnorm_stats(x, 32, 1e-5)
    name = f"gn_{B}x{H}x{W}x{Cc}_{str(dt)[6:]}"
    out = {"mean": _assert_close(name + "_mean", stats[..., 0], mean, 1e-4),
           "rstd": _assert_close(name + "_rstd", stats[..., 1], rstd, 1e-4)}
    got = ops.groupnorm_apply(x, stats, gamma, beta, 32, True)
    for i in range(B):
        out[f"apply_{i}"] = _assert_close(f"{name}_apply_{i}", got[i], ref[i], 4e-3)
    return out


def check_groupnorm():
    _setup()
    return {f"{B}x{H}x{W}x{Cc}": _groupnorm_case(B, H, W, Cc, dt)
            for (B, H, W, Cc, dt) in [(2, 16, 16, 128, bf16), (1, 9, 7, 512, bf16), (1, 32, 32, 256, fp16)]}


def check_groupnorm_offset():
    """groups whose mean is 32x their standard deviation: the single-pass sum(x^2) - sum(x)^2 / n statistics lose
    about log2(32^2) = 10 bits to cancellation there, so their fp32 partial sums must still leave mean and rstd within
    1e-4 of float64 statistics.  The standalone kernel, and the fused convolution's output statistics (a bias of 48
    on outputs of standard deviation ~1.5)."""
    _setup()
    out = {"standalone": _groupnorm_case(1, 64, 64, 256, bf16, mean=48.0, std=1.5)}
    out["fused"] = _conv_fused_case(1, 8, 256, 128, 128, bf16, True, False, False, True, 6e-3, bias_mean=48.0)
    return out


def check_softmax_image_post():
    _setup()
    dt = torch.bfloat16
    x = _rand((37, 1024), dt, 3.0)
    ref = ref_softmax_rows(x, 0.25)
    got = ops.softmax_rows(x.clone(), 0.25)
    out = {"softmax": _assert_close("softmax", got, ref, 4e-3)}
    img = _rand((2, 8, 8, 8), dt, 1.5)
    f, u = ops.image_post(img)
    v, v8 = ref_image_post(img)
    assert torch.equal(f, v), "image_post float"
    assert torch.equal(u, v8), "image_post uint8"
    return out


def check_edge_cases():
    """smallest / most ragged shapes every kernel accepts"""
    _setup()
    out = {}
    out["gemm_1x8x8"] = _gemm_case(1, 8, 8, torch.bfloat16, "bias")
    out["gemm_129x72x24"] = _gemm_case(129, 72, 24, torch.float16, "bias silu")
    out["att_S1"] = _attention_case(2, 1, 2, 128, torch.bfloat16)
    out["att_S129"] = _attention_case(1, 129, 1, 64, torch.float16)
    out["att_S257_split1"] = _attention_case(1, 257, 2, 128, torch.bfloat16, split=1)
    out["conv_1x1"] = _conv_case(1, 1, 1, 64, 8, torch.bfloat16)
    out["conv_3x5"] = _conv_case(2, 3, 5, 64, 24, torch.bfloat16, res=True)
    x = _rand((3, 64), torch.bfloat16, 2.0)
    mod = _rand((3, 128), torch.bfloat16, 0.3)
    ref = ref_ln_modulate(x, mod[:, :64], mod[:, 64:], 1, 1e-6)
    out["ln_h64"] = _assert_close("ln_h64", ops.ln_modulate(x, mod[:, :64], mod[:, 64:], 1, 1e-6), ref, 4e-3)
    g = _rand((1, 1, 1, 64), torch.bfloat16)
    st = ops.groupnorm_stats(g, 32, 1e-5)
    assert bool(torch.isfinite(st).all())
    return out


def check_error_paths():
    """invalid arguments are refused with an error code + message (no launch, no crash)"""
    _setup()
    from diffusionkit_b200._lib import DkError

    A = _rand((16, 64), torch.bfloat16)
    W = _rand((16, 64), torch.bfloat16)
    cases = {
        "N not multiple of 8": lambda: ops.gemm(A, _rand((12, 64), torch.bfloat16)),
        "K not multiple of 8": lambda: ops.gemm(_rand((16, 12), torch.bfloat16), _rand((16, 12), torch.bfloat16)),
        "misaligned A": lambda: ops.gemm(_rand((16, 72), torch.bfloat16)[:, 4:68], W),
        "head dim 96": lambda: ops.attention(_rand((8, 3 * 96), torch.bfloat16), 1, 8, 1, 96,
                                             torch.empty((8, 96), dtype=torch.bfloat16, device=DEV)),
        "conv Cin 48": lambda: ops.conv3x3(_rand((1, 4, 4, 48), torch.bfloat16), _rand((8, 3, 3, 48), torch.bfloat16)),
        "fp32 input": lambda: ops.gemm(A.float(), W.float()),
        "cpu tensor": lambda: ops.gemm(A.cpu(), W.cpu()),
        "ln h too wide": lambda: ops.ln_modulate(_rand((2, 8192), torch.bfloat16), _rand((2, 8192), torch.bfloat16),
                                                 _rand((2, 8192), torch.bfloat16), 1),
    }
    for name, fn in cases.items():
        try:
            fn()
        except DkError as e:
            assert len(str(e)) > 0
            continue
        raise AssertionError(f"{name}: accepted")
    # the context is still healthy afterwards
    return {"after": _gemm_case(128, 128, 64, torch.bfloat16)}


# ------------------------------------------------------------------------------------------------ fused VAE conv (K7f)
def _conv_fused_case(B, H, W, Cin, Cout, dtype, norm, up, res, want_stats, tol, bias_mean=0.0):
    """[GroupNorm+SiLU] -> [nearest 2x] -> conv3x3 (+bias, +skip) in one kernel vs the same chain of fp32 references
    (reference mlx/vae.py:60-101 ResnetBlock2D, :20-25/:146-147 upsample stage); with want_stats, the output
    statistics it folds into its epilogue vs float64 statistics of the stored output"""
    G = 32
    x = _rand((B, H, W, Cin), dtype, 1.5) + 0.3
    w = _rand((Cout, 3, 3, Cin), dtype, 1 / math.sqrt(9 * Cin))
    b = (_rand((Cout,), dtype, 0.5).float() + bias_mean).to(dtype)
    Ho, Wo = (2 * H, 2 * W) if up else (H, W)
    r = _rand((B, Ho, Wo, Cout), dtype) if res else None
    xin, gn = x, None
    if norm:
        gamma, beta = _rand((Cin,), dtype, 0.1) + 1.0, _rand((Cin,), dtype, 0.1)
        gn = (ops.groupnorm_stats(x, G, 1e-5), gamma, beta, G)
        xin = ref_groupnorm_silu(x, gamma, beta, G, 1e-5)[0].to(dtype)     # the conv reads the activation in 16 bits
    if up:
        xin = xin.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    ref = ref_conv3x3(xin, w, b, r)
    wk = ops.conv_up_weights(w) if up else w
    slots = Ho * Wo // 128
    part = torch.full((B, slots, G, 2), float("nan"), dtype=torch.float32, device=DEV) if want_stats else None
    got = ops.conv3x3_fused(x, wk, bias=b, res=r, up=up, gn=gn, silu=norm, out_partial=part, out_G=G)
    name = f"cf_{B}x{H}x{W}_{Cin}to{Cout}_{str(dtype)[6:]}" + "".join(
        f"_{k}" for k, v in (("norm", norm), ("up", up), ("res", res)) if v)
    out = {"rel_l2": _assert_close(name, got, ref, tol)}
    if want_stats:
        st = ops.groupnorm_finalize(part, B, G, slots, float(Ho * Wo * (Cout // G)), 1e-5)
        mean, rstd = ref_groupnorm_stats(got, G, 1e-5)        # float64 statistics of the STORED tensor
        assert bool(torch.isfinite(part).all()), f"{name}: unwritten partial-statistics slots"
        if bias_mean:
            sd = 1.0 / rstd
            out["mean_over_std"] = float((mean.abs() / sd).min())
            assert out["mean_over_std"] >= 25.0, f"{name}: group mean only {out['mean_over_std']:.1f} std"
        out["partial"] = _assert_close(name + "_partial", part, ref_conv_partial_stats(got, G, up), 1e-5)
        out["mean"] = _assert_close(name + "_mean", st[..., 0], mean, 1e-4)
        out["rstd"] = _assert_close(name + "_rstd", st[..., 1], rstd, 1e-4)
    return out


def _conv_fused_table(cases):
    _setup()
    out = {}
    for (B, H, W, Cin, Cout, dt, norm, up, res, want_stats, tol) in cases:
        key = f"{B}x{H}x{W}_{Cin}to{Cout}_norm{norm:d}_up{up:d}_res{res:d}"
        out[key] = _conv_fused_case(B, H, W, Cin, Cout, dt, norm, up, res, want_stats, tol)
    return out


def check_conv_fused():
    # (B, H, W, Cin, Cout, dtype, norm, up, res, want_stats, tol); the 128 -> 8 case is the narrow output tile of
    # conv_out (3 real channels padded to 8; weight rows beyond Cout zero-filled by TMA)
    return _conv_fused_table([(1, 8, 128, 64, 128, bf16, False, False, False, False, 4e-3),
                              (2, 16, 256, 128, 256, bf16, False, False, True, True, 4e-3),
                              (2, 8, 128, 128, 128, bf16, True, False, False, True, 6e-3),
                              (1, 12, 256, 512, 256, bf16, True, False, True, True, 6e-3),
                              (1, 8, 128, 256, 256, bf16, False, True, False, True, 6e-3),
                              (2, 4, 256, 512, 512, bf16, False, True, False, False, 6e-3),
                              (1, 8, 128, 64, 128, fp16, True, False, True, True, 4e-3),
                              (2, 8, 256, 128, 8, bf16, True, False, False, False, 6e-3),
                              (1, 4, 128, 64, 64, bf16, False, False, True, False, 4e-3)])


def check_fullsize_conv_fused():
    """the fused ResNet-path convolution at the 1024^2 decode's real extents"""
    return _conv_fused_table([(1, 1024, 1024, 128, 128, bf16, True, False, True, True, 6e-3),
                              (2, 512, 512, 256, 256, bf16, True, False, False, True, 6e-3),
                              (1, 512, 512, 256, 256, bf16, False, True, False, True, 6e-3)])


# ------------------------------------------------------------------------------------------------ BASELINE shapes
# Parity at the shapes bench.py times (BASELINE.json C3/C4/C5): every kernel against fp32 torch at full size, with a
# per-block error map on top of the global rel-L2 so that ONE wrong output tile (a tile-index decode slip, a barrier phase slip,
# a tail tile) cannot hide in the average.
def _assert_close_blocks(name, got, ref, tol, block_tol, br=128, bc=128, floor=0.0):
    """global rel-L2 <= tol AND every br x bc block's rel-L2 (vs the block's own reference norm) <= block_tol.
    floor > 0: a block's reference norm counts as at least floor x the typical block norm (the tensor's norm over the
    square root of its block count), so a block of near-zero reference values (padded channels, zero rows) is judged
    by its absolute error at the tensor's scale instead of by a ratio of two tiny numbers"""
    err = _assert_close(name, got, ref, tol)
    g, r = got.reshape(-1, got.shape[-1]), ref.reshape(-1, ref.shape[-1])
    R, Cc = g.shape
    Rp, Cp = (R + br - 1) // br * br, (Cc + bc - 1) // bc * bc
    typical = float(torch.linalg.vector_norm(r, dtype=torch.float32)) / math.sqrt((Rp // br) * (Cp // bc))
    worst = 0.0
    step = max(br, (1 << 26) // max(Cp, 1) // br * br)      # ~64 M elements of fp32 scratch at a time
    for r0 in range(0, R, step):
        r1 = min(R, r0 + step)
        dg = torch.zeros((((r1 - r0) + br - 1) // br * br, Cp), dtype=torch.float32, device=g.device)
        dr = torch.zeros_like(dg)
        dg[:r1 - r0, :Cc] = g[r0:r1].float() - r[r0:r1].float()
        dr[:r1 - r0, :Cc] = r[r0:r1].float()
        nb = dg.shape[0] // br
        e = dg.reshape(nb, br, Cp // bc, bc).square().sum(dim=(1, 3)).sqrt()
        n = dr.reshape(nb, br, Cp // bc, bc).square().sum(dim=(1, 3)).sqrt()
        worst = max(worst, float((e / (n.clamp(min=floor * typical) + 1e-20)).max()))
        del dg, dr
    if not worst <= block_tol:
        raise AssertionError(f"{name}: worst {br}x{bc} block rel_l2={worst:.3e} (tol {block_tol:.1e}), global {err:.3e}")
    return {"rel_l2": err, "worst_block": worst}


def check_fullsize_gemm_fc1():
    """FLUX fc1 at the C4 bench shape: 16384 x 12288 x 3072, bias + GELU-erf (reference mlx/mmdit.py:827-835)"""
    _setup()
    return _gemm_case(16384, 12288, 3072, bf16, "bias gelu", block_tol=1.2e-2)


def check_fullsize_gemm_single_out():
    """FLUX single-block output projection at the C4 shape: 17408 x 3072 x 15360 with x + gate * (.) in place
    (reference mlx/mmdit.py:736-751; K = [attn | gelu(fc1)] = 5h)"""
    _setup()
    B, S, N, K = 4, 4352, 3072, 15360
    M = B * S
    A, W, b = _rand((M, K), torch.bfloat16), _rand((N, K), torch.bfloat16, 1 / math.sqrt(K)), _rand((N,), torch.bfloat16, 0.5)
    x, g = _rand((M, N), torch.bfloat16), _rand((B, N), torch.bfloat16)
    ref = ref_gemm(A, W, b, gate=g, res=x)
    got = ops.gemm(A, W, out=x, bias=b, gate=g, res=x, rows_per_batch=S, out_batch_rows=S)
    return _assert_close_blocks("full_single_out", got, ref, 4e-3, 1.2e-2)


def check_fullsize_gemm_qkv_fused():
    """FLUX image-stream QKV at the C4 shape: 4 x 4096 rows scattered behind 256 text rows of a 4 x 4352 joint buffer,
    K = 3072 -> 9216, QK-RMSNorm + RoPE fused (reference mlx/mmdit.py:477-488,594-606,934-942)"""
    _setup()
    Bt, Ss, off, S, heads, d = 4, 4096, 256, 4352, 24, 128
    h, K, dt = heads * d, 3072, torch.bfloat16
    A, W, bias = _rand((Bt * Ss, K), dt), _rand((3 * h, K), dt, 1 / math.sqrt(K)), _rand((3 * h,), dt, 0.3)
    qw, kw = _rand((d,), dt, 0.1) + 1.0, _rand((d,), dt, 0.1) + 1.0
    rope = _rope_table(S, d, DEV)
    fused = torch.zeros((Bt * S, 3 * h), dtype=dt, device=DEV)
    ops.gemm(A, W, out=fused, bias=bias, rows_per_batch=Ss, out_batch_rows=S, out_row_off=off,
             qk=(heads, d, qw, kw, rope, 1e-6))
    rows = torch.cat([torch.arange(b * S + off, b * S + off + Ss) for b in range(Bt)]).to(DEV)
    pos = (torch.arange(Bt * Ss, device=DEV) % Ss) + off
    ref = ref_qk_norm_rope(ref_gemm(A, W, bias), pos, heads, d, qw, kw, rope)
    other = torch.ones(Bt * S, dtype=torch.bool, device=DEV)
    other[rows] = False
    assert float(fused[other].float().abs().max()) == 0.0, "rows outside the scatter window were written"
    return _assert_close_blocks("full_qkv_fused", fused[rows], ref, 6e-3, 1.5e-2)


def check_fullsize_attention():
    """joint attention at the bench sequence lengths, all 24 heads: FLUX d=128 S=4352 (C4: 17 x 256 exactly) and
    S=4608 (C5), SD3 d=64 fp16 S=4685 (C3: ragged tail), outputs split at the text/image boundary as the model does
    (reference mlx/mmdit.py:594-657)"""
    _setup()
    return {"flux_S4352": _attention_case(2, 4352, 24, 128, bf16, 256, out1_pad=0, block_tol=3e-2),
            "flux_S4608": _attention_case(1, 4608, 24, 128, bf16, 512, out1_pad=0, block_tol=3e-2),
            "sd3_S4685": _attention_case(2, 4685, 24, 64, fp16, 4096, out1_pad=0, block_tol=3e-2)}


def check_fullsize_conv():
    """VAE decoder convs at the 1024^2 decode's real extents (reference mlx/vae.py:60-101,146-149):
    1024 x 1024 x 128 -> 128 (+ skip), 512 x 512 x 256 -> 256, and the 512 -> 256 channel change at 512^2"""
    _setup()
    return {"1024_128": _conv_case(1, 1024, 1024, 128, 128, bf16, True, block_tol=1.2e-2),
            "512_256": _conv_case(2, 512, 512, 256, 256, bf16, False, block_tol=1.2e-2),
            "512_512to256": _conv_case(1, 512, 512, 512, 256, bf16, False, block_tol=1.2e-2)}


def check_fullsize_groupnorm():
    """GroupNorm(32) + SiLU at 1024 x 1024 x 128 and 512 x 512 x 256, batch 2 (reference mlx/vae.py:72-80)"""
    _setup()
    return {f"{H}x{W}x{Cc}": _groupnorm_case(B, H, W, Cc, bf16) for (B, H, W, Cc) in [(2, 1024, 1024, 128),
                                                                                     (2, 512, 512, 256)]}


FULLSIZE_CHECKS = [check_fullsize_gemm_fc1, check_fullsize_gemm_single_out, check_fullsize_gemm_qkv_fused,
                   check_fullsize_attention, check_fullsize_conv, check_fullsize_groupnorm, check_fullsize_conv_fused]


ALL_CHECKS = [
    check_gemm_single_tile, check_gemm_multi_k, check_gemm_one_m_pair, check_gemm_shapes, check_gemm_persistent_large,
    check_gemm_epilogues, check_gemm_gate_residual, check_gemm_output_window, check_gemm_fp16,
    check_gemm_inplace_residual, check_gemm_w_n_major, check_gemm_fused_qk_norm_rope,
    check_conv3x3, check_conv3x3_s2, check_img2img_kernels, check_dequant_q4, check_text_kernels, check_attention_small,
    check_attention_d128_one_tile, check_attention_d128, check_attention_d64, check_attention_short,
    check_attention_long, check_attention_many_ctas, check_attention_determinism, check_attention_large_scores,
    check_conv_fused, check_groupnorm_offset,
    check_ln_modulate, check_qk_norm_rope, check_layout_kernels, check_sampler_kernels, check_groupnorm,
    check_softmax_image_post, check_edge_cases, check_error_paths,
] + FULLSIZE_CHECKS
