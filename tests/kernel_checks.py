"""GPU checks of the individual sm_90a kernels against plain fp32 torch references of the same op.

Each check_* function is self-contained (used by tests/test_kernels_gpu.py and by tools/run_gpu_checks.py, which
runs every check in its own process so that one trapped kernel cannot poison the others).
Tolerances: 16-bit outputs, fp32 accumulation -> relative L2 error <= 4e-3 (bf16 epsilon is 3.9e-3 per element,
the L2 over many elements averages to ~2e-3); attention <= 1e-2.
"""
import math
import os

import numpy as np
import torch

from diffusionkit_b200 import ops
from diffusionkit_b200._lib import ACT_GELU_ERF, ACT_NONE, ACT_SILU

DEV = "cuda:0"


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


# ------------------------------------------------------------------------------------------------ GEMM
def _gemm_case(M, N, K, dtype, bias=False, act=ACT_NONE, gate=False, res=False, remap=False, name=""):
    A = _rand((M, K), dtype)
    W = _rand((N, K), dtype, 1.0 / math.sqrt(K))
    b = _rand((N,), dtype, 0.5) if bias else None
    ref = A.float() @ W.float().t()
    if bias:
        ref = ref + b.float()
    if act == ACT_GELU_ERF:
        ref = torch.nn.functional.gelu(ref)
    elif act == ACT_SILU:
        ref = torch.nn.functional.silu(ref)
    kw = {}
    out = None
    if remap:
        # M = Bt * rpb rows scattered into a [Bt * out_rows, N] buffer at row offset off
        Bt = 2
        assert M % Bt == 0
        rpb = M // Bt
        out_rows, off = rpb + 40, 24
        out = torch.zeros((Bt * out_rows, N), dtype=dtype, device=DEV)
        kw.update(rows_per_batch=rpb, out_batch_rows=out_rows, out_row_off=off)
        g = _rand((Bt, N), dtype) if gate else None
        r = _rand((Bt * rpb, N), dtype) if res else None
        if gate:
            ref = ref * g.float().repeat_interleave(rpb, 0)
        if res:
            ref = ref + r.float()
        got = ops.gemm(A, W, out=out, bias=b, act=act, gate=g, res=r, **kw)
        got_rows = torch.cat([got[i * out_rows + off:i * out_rows + off + rpb] for i in range(Bt)], 0)
        untouched = torch.cat([got[i * out_rows:i * out_rows + off] for i in range(Bt)], 0)
        assert float(untouched.float().abs().max()) == 0.0, f"{name}: rows outside the remap window were written"
        return _assert_close(name, got_rows, ref, 4e-3)
    g = _rand((1, N), dtype) if gate else None
    r = _rand((M, N), dtype) if res else None
    if gate:
        ref = ref * g.float()
    if res:
        ref = ref + r.float()
    got = ops.gemm(A, W, bias=b, act=act, gate=g, res=r)
    return _assert_close(name, got, ref, 4e-3)


def check_gemm_single_tile():
    _setup()
    return {"err": _gemm_case(128, 256, 64, torch.bfloat16, name="gemm_128x256x64")}


def check_gemm_multi_k():
    _setup()
    return {"err": _gemm_case(128, 256, 512, torch.bfloat16, name="gemm_128x256x512")}


def check_gemm_shapes():
    _setup()
    out = {}
    for (M, N, K) in [(256, 512, 256), (300, 264, 200), (77, 64, 64), (1000, 3072, 1536), (20, 1024, 3072),
                      (4352, 768, 3072), (128, 128, 128)]:
        out[f"{M}x{N}x{K}"] = _gemm_case(M, N, K, torch.bfloat16, name=f"gemm_{M}x{N}x{K}")
    return out


def check_gemm_persistent_large():
    _setup()
    # more tiles than SMs: exercises more than one wave of CTAs and the smem ring wrap-around
    return {"err": _gemm_case(4096, 4608, 1024, torch.bfloat16, bias=True, name="gemm_4096x4608x1024")}


def check_gemm_epilogues():
    _setup()
    out = {}
    out["bias"] = _gemm_case(384, 512, 256, torch.bfloat16, bias=True, name="gemm_bias")
    out["gelu"] = _gemm_case(384, 512, 256, torch.bfloat16, bias=True, act=ACT_GELU_ERF, name="gemm_gelu")
    out["silu"] = _gemm_case(384, 512, 256, torch.bfloat16, bias=True, act=ACT_SILU, name="gemm_silu")
    out["gate_res"] = _gemm_case(384, 512, 256, torch.bfloat16, bias=True, gate=True, res=True, name="gemm_gate_res")
    out["remap"] = _gemm_case(600, 512, 256, torch.bfloat16, bias=True, gate=True, res=True, remap=True,
                              name="gemm_remap")
    return out


def check_gemm_fp16():
    _setup()
    return {"err": _gemm_case(300, 512, 320, torch.float16, bias=True, act=ACT_GELU_ERF, name="gemm_fp16")}


def check_gemm_inplace_residual():
    _setup()
    M, N, K = 256, 256, 128
    A = _rand((M, K), torch.bfloat16)
    W = _rand((N, K), torch.bfloat16, 1 / math.sqrt(K))
    x = _rand((M, N), torch.bfloat16)
    ref = x.float() + A.float() @ W.float().t()
    got = ops.gemm(A, W, out=x, res=x)
    return {"err": _assert_close("gemm_inplace", got, ref, 4e-3)}


def check_gemm_w_n_major():
    _setup()
    out = {}
    for (M, N, K) in [(128, 128, 64), (256, 384, 256), (200, 136, 72)]:
        A = _rand((M, K), torch.bfloat16)
        Wt = _rand((K, N), torch.bfloat16, 1 / math.sqrt(K))  # [K, N] row-major
        ref = A.float() @ Wt.float()
        got = ops.gemm(A, Wt, w_n_major=True)
        out[f"{M}x{N}x{K}"] = _assert_close(f"gemm_nmajor_{M}x{N}x{K}", got, ref, 4e-3)
    return out


# ------------------------------------------------------------------------------------------------ conv
def _conv_case(B, H, W, Cin, Cout, dtype, bias=True, res=False, name=""):
    x = _rand((B, H, W, Cin), dtype)
    w = _rand((Cout, 3, 3, Cin), dtype, 1 / math.sqrt(9 * Cin))
    b = _rand((Cout,), dtype, 0.5) if bias else None
    r = _rand((B, H, W, Cout), dtype) if res else None
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2),
                                     b.float() if bias else None, padding=1).permute(0, 2, 3, 1)
    if res:
        ref = ref + r.float()
    got = ops.conv3x3(x, w, bias=b, res=r)
    return _assert_close(name, got, ref, 4e-3)


def check_conv3x3():
    _setup()
    out = {}
    out["16x16"] = _conv_case(2, 16, 16, 64, 64, torch.bfloat16, name="conv_16x16")
    out["8x32_res"] = _conv_case(1, 8, 32, 128, 128, torch.bfloat16, res=True, name="conv_8x32")
    out["12x20_ragged"] = _conv_case(2, 12, 20, 64, 72, torch.bfloat16, name="conv_12x20")
    out["64x256"] = _conv_case(1, 64, 256, 128, 256, torch.bfloat16, res=True, name="conv_64x256")
    out["fp16"] = _conv_case(1, 32, 32, 64, 16, torch.float16, name="conv_fp16")
    return out


def _conv_s2_case(B, H, W, Cin, Cout, dtype, name=""):
    x = _rand((B, H, W, Cin), dtype)
    w = _rand((Cout, 3, 3, Cin), dtype, 1 / math.sqrt(9 * Cin))
    b = _rand((Cout,), dtype, 0.5)
    # reference downsample: pad bottom/right by one, then 3x3 stride 2 without padding (mlx/vae.py:142-144)
    xp = torch.nn.functional.pad(x.float().permute(0, 3, 1, 2), (0, 1, 0, 1))
    ref = torch.nn.functional.conv2d(xp, w.float().permute(0, 3, 1, 2), b.float(), stride=2).permute(0, 2, 3, 1)
    got = ops.conv3x3_s2(x, w, bias=b)
    assert got.shape == (B, H // 2, W // 2, Cout)
    return _assert_close(name, got, ref, 4e-3)


def check_conv3x3_s2():
    """the encoder's stride-2 downsample: same implicit-GEMM kernel, TMA box with element stride 2"""
    _setup()
    out = {}
    out["32x32"] = _conv_s2_case(2, 32, 32, 64, 64, torch.bfloat16, name="convs2_32x32")          # TW=16, TH=8
    out["16x64"] = _conv_s2_case(1, 16, 64, 128, 128, torch.bfloat16, name="convs2_16x64")        # TW=32, TH=4
    out["24x40_ragged"] = _conv_s2_case(2, 24, 40, 64, 72, torch.bfloat16, name="convs2_24x40")   # TW=128 ragged
    out["64x512"] = _conv_s2_case(1, 64, 512, 128, 128, torch.bfloat16, name="convs2_64x512")     # box 256 wide
    out["fp16"] = _conv_s2_case(1, 32, 32, 64, 16, torch.float16, name="convs2_fp16")
    return out


def check_img2img_kernels():
    """dk_image_pre, dk_vae_sample_latent, dk_axpby_f32 (read_image / posterior sample / noise_scaling)"""
    _setup()
    out = {}
    for dt in (torch.bfloat16, torch.float16):
        for cs in (3, 4):
            img = torch.randint(0, 256, (2, 8, 12, cs), dtype=torch.uint8, device=DEV)
            got = ops.image_pre(img, dt, 64)
            # reference arithmetic on the CPU: torch's CUDA div-by-scalar multiplies by the reciprocal, the reference
            # (and dk_image_pre) divide
            ref = torch.zeros((2, 8, 12, 64), dtype=torch.float32)
            ref[..., :3] = img.cpu()[..., :3].float() / 255 * 2 - 1.0
            assert torch.equal(got.cpu(), ref.to(dt)), f"image_pre {dt} {cs}"
    hidden = _rand((1, 8, 8, 32), torch.bfloat16, 2.0)
    hidden[0, 0, 0, 16] = 50.0       # logvar clipped at 20
    hidden[0, 0, 1, 16] = -80.0      # ... and at -30
    noise = torch.randn((1, 8, 8, 16), device=DEV)
    mean, logvar = hidden.float().split(16, dim=-1)
    z = mean + torch.exp(0.5 * logvar.clamp(-30.0, 20.0)) * noise
    out["sample"] = _assert_close("vae_sample", ops.vae_sample_latent(hidden, noise, 0.0, 1.0), z, 1e-5)
    out["sample_in"] = _assert_close("vae_sample_in", ops.vae_sample_latent(hidden, noise, 0.1159, 0.3611),
                                     (z - 0.1159) * 0.3611, 1e-5)
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
    """csrc/text.cu: embedding, LayerNorm(affine), T5 RMSNorm over fp32, fp32 += 16-bit, gated GELU, quick-GELU epilogue"""
    from diffusionkit_b200._lib import ACT_QUICK_GELU

    _setup()
    out = {}
    for dt in (torch.bfloat16, torch.float16):
        table, pos = _rand((50, 128), dt), _rand((7, 128), dt)
        ids = torch.randint(0, 50, (3, 7), dtype=torch.int32, device=DEV)
        got = ops.embedding(table, ids.reshape(-1).contiguous(), pos=pos)
        want = (table.float()[ids.long()] + pos.float()[None]).to(dt).reshape(21, 128)
        assert torch.equal(got, want), f"embedding+pos {dt}"
        assert torch.equal(ops.embedding(table, ids.reshape(-1).contiguous()), table[ids.long().reshape(-1)])
    for (rows, h, dt) in [(77, 768, torch.bfloat16), (154, 1280, torch.float16), (5, 128, torch.bfloat16)]:
        x, w, b = _rand((rows, h), dt, 2.0), _rand((h,), dt, 0.5) + 1.0, _rand((h,), dt, 0.3)
        ref = torch.nn.functional.layer_norm(x.float(), (h,), w.float(), b.float(), 1e-5)
        out[f"ln_{h}"] = _assert_close(f"layernorm_{h}", ops.layernorm(x, w, b, 1e-5), ref, 4e-3)
    for (rows, d, dt) in [(64, 4096, torch.bfloat16), (9, 256, torch.bfloat16), (3, 1000, torch.float16)]:
        x = torch.randn((rows, d), device=DEV) * 30.0
        w = _rand((d,), dt, 0.2) + 1.0
        ref = w.float() * x * torch.rsqrt(x.square().mean(-1, keepdim=True) + 1e-6)
        out[f"rms_{d}"] = _assert_close(f"rmsnorm_f32_{d}", ops.rmsnorm_f32(x, w, 1e-6), ref, 4e-3)
    x32, y16 = torch.randn(4096, device=DEV), _rand((4096,), torch.bfloat16)
    assert torch.equal(ops.add_f32_16(x32.clone(), y16), x32 + y16.float())
    hgl = _rand((33, 2 * 512), torch.bfloat16, 2.0)
    ref = torch.nn.functional.gelu(hgl.float()[:, :512]) * hgl.float()[:, 512:]
    out["glu"] = _assert_close("glu_gelu", ops.glu_gelu(hgl), ref, 4e-3)
    a, wq = _rand((77, 256), torch.bfloat16), _rand((512, 256), torch.bfloat16, 1 / 16)
    bq = _rand((512,), torch.bfloat16, 0.5)
    z = a.float() @ wq.float().t() + bq.float()
    out["quick_gelu"] = _assert_close("gemm_quick_gelu", ops.gemm(a, wq, bias=bq, act=ACT_QUICK_GELU),
                                      z * torch.sigmoid(1.702 * z), 4e-3)
    return out


def _attention_small_case(B, S, heads, dt, causal, rel, scale, name):
    qkv = _rand((B * S, 3 * heads * 64), dt)
    q, k, v = [t.reshape(B, S, heads, 64).permute(0, 2, 1, 3).float() for t in qkv.split(heads * 64, dim=1)]
    s = scale * (q @ k.transpose(-1, -2))
    rel_bias = None
    if rel:
        rel_bias = _rand((heads, 2 * S - 1), dt, 2.0)
        idx = (torch.arange(S, device=DEV)[None, :] - torch.arange(S, device=DEV)[:, None]) + S - 1     # j - i + S - 1
        s = s + rel_bias.float()[:, idx][None]
    if causal:
        i = torch.arange(S, device=DEV)
        s = s + (i[:, None] < i[None]).float() * -6e4
    ref = (torch.softmax(s, dim=-1) @ v).permute(0, 2, 1, 3).reshape(B * S, heads * 64)
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
def _attention_case(B, S, heads, d, dtype, split=None, name=""):
    h = heads * d
    qkv = _rand((B * S, 3 * h), dtype)
    q, k, v = [t.reshape(B, S, heads, d).permute(0, 2, 1, 3).float() for t in qkv.split(h, dim=1)]
    ref = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(d), dim=-1) @ v
    ref = ref.permute(0, 2, 1, 3).reshape(B, S, h)
    if split is None:
        out = torch.zeros((B * S, h), dtype=dtype, device=DEV)
        ops.attention(qkv, B, S, heads, d, out)
        got = out.reshape(B, S, h)
    else:
        o0 = torch.zeros((B * split, h), dtype=dtype, device=DEV)
        o1 = torch.zeros((B * (S - split), h + 64), dtype=dtype, device=DEV)[:, :h]  # non-trivial leading dim
        ops.attention(qkv, B, S, heads, d, o0, split=split, out1=o1)
        got = torch.cat([o0.reshape(B, split, h), o1.reshape(B, S - split, h)], dim=1)
    return _assert_close(name, got, ref, 1e-2)


def check_attention_d128_one_tile():
    _setup()
    return {"err": _attention_case(1, 128, 1, 128, torch.bfloat16, name="att_d128_S128")}


def check_attention_d128():
    _setup()
    out = {}
    out["S300"] = _attention_case(2, 300, 2, 128, torch.bfloat16, name="att_d128_S300")
    out["S1280_split"] = _attention_case(1, 1280, 3, 128, torch.bfloat16, split=256, name="att_d128_S1280")
    return out


def check_attention_d64():
    _setup()
    out = {}
    out["S128"] = _attention_case(1, 128, 1, 64, torch.float16, name="att_d64_S128")
    out["S1178_split"] = _attention_case(2, 1178, 2, 64, torch.float16, split=1024, name="att_d64_S1178")
    out["bf16_S333"] = _attention_case(1, 333, 2, 64, torch.bfloat16, name="att_d64_S333")
    return out


def check_attention_v3_explicit():
    """split outputs with a ragged tail at d = 64 (fp16 and bf16), two batches at d = 128, rescale"""
    _setup()
    out = {"d64_S1178_split": _attention_case(2, 1178, 2, 64, torch.float16, split=1024, name="att3_d64_S1178"),
           "d64_S333": _attention_case(1, 333, 2, 64, torch.bfloat16, name="att3_d64_S333"),
           "d128_S300": _attention_case(2, 300, 2, 128, torch.bfloat16, name="att3_d128_S300")}
    out["rescale"] = check_attention_large_scores()["err"]
    return out


def check_attention_v3_variants():
    """long ragged sequences at both head dims against the fp32 reference, and the kernel is deterministic: a second
    launch on the same input is bit-identical to the first (the K/V steps and the quad reductions run in a fixed order)"""
    _setup()
    out = {}
    for d, dt, S in ((128, torch.bfloat16, 1300), (64, torch.float16, 1178)):
        name = f"att_d{d}_S{S}"
        out[name] = _attention_case(2, S, 2, d, dt, split=1024, name=name)
        qkv = _rand((2 * S, 3 * 2 * d), dt)
        o1 = torch.zeros((2 * S, 2 * d), dtype=dt, device=DEV)
        o2 = torch.zeros((2 * S, 2 * d), dtype=dt, device=DEV)
        ops.attention(qkv, 2, S, 2, d, o1)
        ops.attention(qkv, 2, S, 2, d, o2)
        assert torch.equal(o1, o2), f"{name}: two launches on the same input differ"
    return out


def check_attention_v3s_kernel():
    """one full K/V tile, ragged tails, split outputs at both head dims, a one-token sequence, rescale"""
    _setup()
    out = {"d128_S128": _attention_case(1, 128, 1, 128, torch.bfloat16, name="att3s_d128_S128"),
           "d128_S300": _attention_case(2, 300, 2, 128, torch.bfloat16, name="att3s_d128_S300"),
           "d128_S1280_split": _attention_case(1, 1280, 3, 128, torch.bfloat16, split=256, name="att3s_d128_S1280"),
           "d64_S1178_split": _attention_case(2, 1178, 2, 64, torch.float16, split=1024, name="att3s_d64_S1178"),
           "S1": _attention_case(2, 1, 2, 128, torch.bfloat16, name="att3s_S1")}
    out["rescale"] = check_attention_large_scores()["err"]
    return out


def check_attention_v5_kernel():
    """more CTAs than SMs, odd/even K/V tile counts, tails, both head dims, split outputs, rescale"""
    _setup()
    out = {"d128_S128": _attention_case(1, 128, 1, 128, torch.bfloat16, name="att5_d128_S128"),
           "d128_S256": _attention_case(1, 256, 2, 128, torch.bfloat16, name="att5_d128_S256"),
           "d128_S300": _attention_case(2, 300, 2, 128, torch.bfloat16, name="att5_d128_S300"),
           "d128_S1280_split": _attention_case(1, 1280, 3, 128, torch.bfloat16, split=256, name="att5_d128_S1280"),
           "d64_S1178_split": _attention_case(2, 1178, 2, 64, torch.float16, split=1024, name="att5_d64_S1178"),
           "d64_S333": _attention_case(1, 333, 2, 64, torch.bfloat16, name="att5_d64_S333"),
           "S1": _attention_case(2, 1, 2, 128, torch.bfloat16, name="att5_S1"),
           "many_items": _attention_case(3, 700, 24, 128, torch.bfloat16, split=100, name="att5_many"),     # 216 items
           "many_items_d64": _attention_case(2, 1500, 24, 64, torch.float16, split=1024, name="att5_many64")}
    out["rescale"] = check_attention_large_scores()["err"]
    return out


def check_attention_v6_kernel():
    """one and many K/V steps, odd / even step counts, ragged tails (incl. tiles with a fully masked half), both head
    dims, split outputs, rescale"""
    _setup()
    out = {"d128_S64": _attention_case(1, 64, 1, 128, torch.bfloat16, name="att6_d128_S64"),
           "d128_S128": _attention_case(1, 128, 1, 128, torch.bfloat16, name="att6_d128_S128"),
           "d128_S300": _attention_case(2, 300, 2, 128, torch.bfloat16, name="att6_d128_S300"),
           "d128_S1280_split": _attention_case(1, 1280, 3, 128, torch.bfloat16, split=256, name="att6_d128_S1280"),
           "d128_S4400": _attention_case(1, 4400, 2, 128, torch.bfloat16, name="att6_d128_S4400"),
           "d64_S1178_split": _attention_case(2, 1178, 2, 64, torch.float16, split=1024, name="att6_d64_S1178"),
           "d64_S333": _attention_case(1, 333, 2, 64, torch.bfloat16, name="att6_d64_S333"),
           "S1": _attention_case(2, 1, 2, 128, torch.bfloat16, name="att6_S1")}
    out["rescale"] = check_attention_large_scores()["err"]
    return out


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
    q, k, v = [t.reshape(B, S, heads, d).permute(0, 2, 1, 3).float() for t in qkv.split(h, dim=1)]
    ref = (torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(d), dim=-1) @ v).permute(0, 2, 1, 3).reshape(B * S, h)
    out = torch.zeros((B * S, h), dtype=torch.bfloat16, device=DEV)
    ops.attention(qkv, B, S, heads, d, out)
    return {"err": _assert_close("att_rescale", out, ref, 1e-2)}


# ------------------------------------------------------------------------------------------------ elementwise
def check_ln_modulate():
    _setup()
    out = {}
    for (B, S, h, dt) in [(2, 37, 3072, torch.bfloat16), (1, 64, 1536, torch.float16), (3, 5, 128, torch.bfloat16)]:
        x = _rand((B * S, h), dt, 2.0) + 0.5
        mod = _rand((B, 6 * h), dt, 0.3)
        shift, scale = mod[:, 0:h], mod[:, h:2 * h]
        xf = x.float()
        ln = torch.nn.functional.layer_norm(xf, (h,), eps=1e-6)
        ref = ln * (1 + scale.float().repeat_interleave(S, 0)) + shift.float().repeat_interleave(S, 0)
        got = ops.ln_modulate(x, shift, scale, S, 1e-6)
        out[f"{B}x{S}x{h}"] = _assert_close(f"ln_{h}", got, ref, 4e-3)
    return out


def _rope_table(S, d, device):
    ang = torch.rand((S, d // 2), device=device) * 6.28
    return torch.stack([torch.cos(ang), torch.sin(ang)], dim=-1).contiguous()


def check_qk_norm_rope():
    _setup()
    out = {}
    for (B, S, heads, d, dt, use_norm, use_rope) in [(2, 50, 3, 128, torch.bfloat16, True, True),
                                                     (1, 33, 2, 64, torch.float16, True, False),
                                                     (1, 40, 2, 128, torch.bfloat16, False, True)]:
        h = heads * d
        qkv = _rand((B * S, 3 * h), dt)
        split = S // 3
        ws = [(_rand((d,), dt, 0.1) + 1.0) for _ in range(4)] if use_norm else [None] * 4
        rope = _rope_table(S, d, DEV) if use_rope else None
        ref = qkv.float().clone()
        pos = torch.arange(B * S, device=DEV) % S
        for which, (w1, w2) in enumerate([(ws[0], ws[2]), (ws[1], ws[3])]):
            t = ref[:, which * h:(which + 1) * h].reshape(B * S, heads, d)
            if use_norm:
                w = torch.where((pos < split)[:, None, None], w1.float()[None, None], w2.float()[None, None])
                t = t * torch.rsqrt((t * t).mean(-1, keepdim=True) + 1e-6) * w
                t = t.to(dt).float()
            if use_rope:
                c = rope[pos][:, None, :, 0]
                s = rope[pos][:, None, :, 1]
                x0, x1 = t[..., 0::2], t[..., 1::2]
                t = torch.stack([x0 * c - x1 * s, x0 * s + x1 * c], dim=-1).reshape(B * S, heads, d)
            ref[:, which * h:(which + 1) * h] = t.reshape(B * S, h)
        got = ops.qk_norm_rope(qkv.clone(), S, heads, d, split, ws[0], ws[1], ws[2], ws[3], rope)
        out[f"d{d}_{use_norm}_{use_rope}"] = _assert_close(f"qknr_{d}", got, ref, 4e-3)
    return out


def check_gemm_pair_kernel():
    """large and ragged shapes (256- and 128-wide tiles): ragged M/N/K, every epilogue, more tiles than SMs, strided
    output windows, in-place residual, the fused QK epilogue"""
    _setup()
    out = {}
    for (M, N, K) in [(256, 256, 64), (256, 512, 512), (300, 264, 200), (77, 64, 64), (1000, 3072, 1536),
                      (4352, 768, 3072), (20, 1024, 3072)]:
        out[f"{M}x{N}x{K}"] = _gemm_case(M, N, K, torch.bfloat16, name=f"pair_{M}x{N}x{K}")
    out["large"] = _gemm_case(8192, 4608, 1024, torch.bfloat16, bias=True, name="pair_8192x4608x1024")
    out["n3072"] = _gemm_case(4096, 3072, 512, torch.bfloat16, bias=True, name="pair_4096x3072x512")
    out["bn128"] = _gemm_case(1024, 1152, 256, torch.bfloat16, bias=True, gate=True, res=True, name="pair_1024x1152")
    out["gelu"] = _gemm_case(384, 512, 256, torch.bfloat16, bias=True, act=ACT_GELU_ERF, name="pair_gelu")
    out["remap"] = _gemm_case(600, 512, 256, torch.bfloat16, bias=True, gate=True, res=True, remap=True,
                              name="pair_remap")
    out["fp16"] = _gemm_case(300, 512, 320, torch.float16, bias=True, name="pair_fp16")
    out.update(_pair_store_cases())
    out.update({"qk_" + k: v for k, v in check_gemm_fused_qk_norm_rope().items()})
    return out


def _pair_store_cases():
    """outputs the GEMM epilogue has to get right: a strided column window of a wider buffer (the FLUX single-block
    concat buffer), rows/columns that are not tile multiples next to data that must survive, in-place residual"""
    out = {}
    M, N, K, ld, c0 = 1000, 520, 256, 1024, 256
    A, W = _rand((M, K), torch.bfloat16), _rand((N, K), torch.bfloat16, 1 / math.sqrt(K))
    buf = torch.full((M + 8, ld), 7.0, dtype=torch.bfloat16, device=DEV)
    view = buf[:M, c0:c0 + N]
    ops.gemm(A, W, out=view, act=ACT_GELU_ERF)
    out["window"] = _assert_close("pair_window", view, torch.nn.functional.gelu(A.float() @ W.float().t()), 4e-3)
    keep = buf.clone()
    keep[:M, c0:c0 + N] = 7.0
    assert bool((keep == 7.0).all()), "pair_window: bytes outside the output window were written"
    x = _rand((M, N), torch.bfloat16)
    g = _rand((1, N), torch.bfloat16)
    ref = x.float() + g.float() * (A.float() @ W.float().t())
    out["inplace"] = _assert_close("pair_inplace", ops.gemm(A, W, out=x, res=x, gate=g), ref, 4e-3)
    return out


def check_gemm_pair_legacy_store():
    """the epilogue's register -> global stores with bias, gate and in-place-able residual on a multi-tile problem and a
    ragged one, plus the output-window cases"""
    _setup()
    out = {"large": _gemm_case(2048, 1536, 512, torch.bfloat16, bias=True, gate=True, res=True, name="pairleg_large"),
           "ragged": _gemm_case(300, 264, 200, torch.bfloat16, name="pairleg_ragged")}
    out.update(_pair_store_cases())
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
        # fp32 reference
        y = (A.float() @ W.float().t() + bias.float())
        pos = (torch.arange(Bt * Ss, device=DEV) % Ss) + off
        ref = y.clone()
        for which, w in enumerate([qw, kw]):
            t = y[:, which * h:(which + 1) * h].reshape(-1, heads, d)
            if use_norm:
                t = t * torch.rsqrt((t * t).mean(-1, keepdim=True) + 1e-6) * w.float()
            if use_rope:
                c, sn = rope[pos][:, None, :, 0], rope[pos][:, None, :, 1]
                x0, x1 = t[..., 0::2], t[..., 1::2]
                t = torch.stack([x0 * c - x1 * sn, x0 * sn + x1 * c], dim=-1).reshape(-1, heads, d)
            ref[:, which * h:(which + 1) * h] = t.reshape(-1, h)
        out[f"vs_fp32_d{d}_{use_norm}"] = _assert_close(f"fusedqk_ref_{d}", fused[rows], ref, 6e-3)
    return out


def check_layout_kernels():
    _setup()
    out = {}
    dt = torch.bfloat16
    B, H, W, Cc = 2, 8, 12, 16
    lat = _rand((B, H, W, Cc), dt)
    # FLUX order (c, ph, pw) — reference mmdit.py:292-302
    ref0 = lat.reshape(B, H // 2, 2, W // 2, 2, Cc).permute(0, 1, 3, 5, 2, 4).reshape(B * (H // 2) * (W // 2), 4 * Cc)
    got0 = ops.patchify(lat, 0)
    assert torch.equal(got0, ref0), "patchify order 0"
    # SD3 order (ph, pw, c)
    ref1 = lat.reshape(B, H // 2, 2, W // 2, 2, Cc).permute(0, 1, 3, 2, 4, 5).reshape(B * (H // 2) * (W // 2), 4 * Cc)
    got1 = ops.patchify(lat, 1)
    assert torch.equal(got1, ref1), "patchify order 1"
    assert torch.equal(ops.unpatchify(got0, B, H, W, Cc, 0), lat), "unpatchify order 0"
    assert torch.equal(ops.unpatchify(got1, B, H, W, Cc, 1), lat), "unpatchify order 1"
    # pos-embed crop — reference mmdit.py:334-349
    max_hw, hp, wp, h = 12, 4, 6, 64
    table = _rand((max_hw * max_hw, h), dt)
    y0, x0 = (max_hw - hp) // 2, (max_hw - wp) // 2
    refc = table.reshape(max_hw, max_hw, h)[y0:y0 + hp, x0:x0 + wp].reshape(hp * wp, h)
    assert torch.equal(ops.pos_embed_crop(table, max_hw, hp, wp), refc), "pos_embed_crop"
    # copy_rows
    src = _rand((2, 5, 64), dt)
    dst = torch.zeros((2, 9, 64), dtype=dt, device=DEV)
    ops.copy_rows(src, dst, 2, 5, 64, 9, 3, 5, 0)
    assert torch.equal(dst[:, 3:8], src) and float(dst[:, :3].float().abs().max()) == 0
    # silu_add / act
    y = _rand((3, 128), dt)
    temb = _rand((4, 128), dt)
    refs = torch.nn.functional.silu((y.float()[None] + temb.float()[:, None]).to(dt).float()).reshape(12, 128)
    out["silu_add"] = _assert_close("silu_add", ops.silu_add(y, temb), refs, 4e-3)
    out["act_silu"] = _assert_close("act_silu", ops.act(y, ACT_SILU), torch.nn.functional.silu(y.float()), 4e-3)
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
        den = xin.float() - mo.float() * sigma
        if cfg > 0:
            den = den[n:] + cfg * (den[:n] - den[n:])
        ref = x + (x - den) / sigma * (sigma_next - sigma)
        got = ops.sampler_step(x.clone(), xin, mo, sigma, sigma_next, cfg)
        out[f"cfg{cfg}"] = _assert_close(f"sampler_{cfg}", got, ref, 1e-5)
    out["axpb"] = _assert_close("axpb", ops.axpb(x, 1 / 0.3611, 0.1159), x / 0.3611 + 0.1159, 1e-6)
    assert torch.equal(ops.cast_to_16(x, dt), x.to(dt))
    assert torch.equal(ops.cast_to_f32(x.to(dt)), x.to(dt).float())
    return out


def check_groupnorm():
    _setup()
    out = {}
    for (B, H, W, Cc, dt) in [(2, 16, 16, 128, torch.bfloat16), (1, 9, 7, 512, torch.bfloat16),
                              (1, 32, 32, 256, torch.float16)]:
        x = _rand((B, H, W, Cc), dt, 1.5) + 0.7
        gamma = _rand((Cc,), dt, 0.1) + 1.0
        beta = _rand((Cc,), dt, 0.1)
        stats = ops.groupnorm_stats(x, 32, 1e-5)
        xf = x.float().reshape(B, H * W, 32, Cc // 32)
        mean = xf.mean(dim=(1, 3))
        var = xf.var(dim=(1, 3), unbiased=False)
        out[f"stats_{Cc}"] = _assert_close("gn_mean", stats[..., 0], mean, 1e-4)
        _assert_close("gn_rstd", stats[..., 1], torch.rsqrt(var + 1e-5), 1e-4)
        ref = torch.nn.functional.group_norm(x.float().permute(0, 3, 1, 2), 32, gamma.float(), beta.float(), 1e-5)
        ref = torch.nn.functional.silu(ref.permute(0, 2, 3, 1).to(dt).float())
        got = ops.groupnorm_apply(x, stats, gamma, beta, 32, True)
        out[f"apply_{Cc}"] = _assert_close("gn_apply", got, ref, 4e-3)
    return out


def check_softmax_image_post():
    _setup()
    dt = torch.bfloat16
    x = _rand((37, 1024), dt, 3.0)
    ref = torch.softmax(x.float() * 0.25, dim=-1)
    got = ops.softmax_rows(x.clone(), 0.25)
    out = {"softmax": _assert_close("softmax", got, ref, 4e-3)}
    img = _rand((2, 8, 8, 8), dt, 1.5)
    f, u = ops.image_post(img)
    v = ((img[..., :3].float() * 0.5).to(dt).float() + 0.5).to(dt).float().clamp(0, 1)
    assert torch.equal(f, v), "image_post float"
    assert torch.equal(u, (v * 255).to(dt).float().to(torch.uint8)), "image_post uint8"
    return out


def check_edge_cases():
    """smallest / most ragged shapes every kernel accepts"""
    _setup()
    out = {}
    out["gemm_1x8x8"] = _gemm_case(1, 8, 8, torch.bfloat16, bias=True, name="gemm_1x8x8")
    out["gemm_129x72x24"] = _gemm_case(129, 72, 24, torch.float16, bias=True, act=ACT_SILU, name="gemm_129x72x24")
    out["att_S1"] = _attention_case(2, 1, 2, 128, torch.bfloat16, name="att_S1")
    out["att_S129"] = _attention_case(1, 129, 1, 64, torch.float16, name="att_S129")
    out["att_S257_split1"] = _attention_case(1, 257, 2, 128, torch.bfloat16, split=1, name="att_S257")
    out["conv_1x1"] = _conv_case(1, 1, 1, 64, 8, torch.bfloat16, name="conv_1x1")
    out["conv_3x5"] = _conv_case(2, 3, 5, 64, 24, torch.bfloat16, res=True, name="conv_3x5")
    x = _rand((3, 64), torch.bfloat16, 2.0)
    mod = _rand((3, 128), torch.bfloat16, 0.3)
    ref = torch.nn.functional.layer_norm(x.float(), (64,), eps=1e-6) * (1 + mod[:, 64:].float()) + mod[:, :64].float()
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
    return {"after": _gemm_case(128, 128, 64, torch.bfloat16, name="gemm_after_errors")}


# ------------------------------------------------------------------------------------------------ fused VAE conv (K7f)
def _conv_fused_case(B, H, W, Cin, Cout, dtype, norm, up, res, want_stats, name, tol=4e-3):
    """[GroupNorm+SiLU] -> [nearest 2x] -> conv3x3 (+bias, +skip) in one kernel vs the same chain in fp32 torch
    (reference mlx/vae.py:60-101 ResnetBlock2D, :20-25/:146-147 upsample stage)"""
    G = 32
    x = _rand((B, H, W, Cin), dtype, 1.5) + 0.3
    w = _rand((Cout, 3, 3, Cin), dtype, 1 / math.sqrt(9 * Cin))
    b = _rand((Cout,), dtype, 0.5)
    Ho, Wo = (2 * H, 2 * W) if up else (H, W)
    r = _rand((B, Ho, Wo, Cout), dtype) if res else None
    xin = x.float()
    gn = None
    if norm:
        gamma, beta = _rand((Cin,), dtype, 0.1) + 1.0, _rand((Cin,), dtype, 0.1)
        stats = ops.groupnorm_stats(x, G, 1e-5)
        gn = (stats, gamma, beta, G)
        xn = torch.nn.functional.group_norm(xin.permute(0, 3, 1, 2), G, gamma.float(), beta.float(), 1e-5)
        xin = torch.nn.functional.silu(xn.permute(0, 2, 3, 1).to(dtype).float()).to(dtype).float()
    if up:
        xin = xin.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    ref = torch.nn.functional.conv2d(xin.permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), b.float(),
                                     padding=1).permute(0, 2, 3, 1)
    if res:
        ref = ref + r.float()
    wk = ops.conv_up_weights(w) if up else w
    slots = Ho * Wo // 128
    part = torch.full((B, slots, G, 2), float("nan"), dtype=torch.float32, device=DEV) if want_stats else None
    got = ops.conv3x3_fused(x, wk, bias=b, res=r, up=up, gn=gn, silu=norm, out_partial=part, out_G=G)
    out = {"rel_l2": _assert_close(name, got, ref, tol)}
    if want_stats:
        st = ops.groupnorm_finalize(part, B, G, slots, float(Ho * Wo * (Cout // G)), 1e-5)
        st_ref = ops.groupnorm_stats(got, G, 1e-5)           # statistics of the STORED tensor, standalone kernel
        assert bool(torch.isfinite(part).all()), f"{name}: unwritten partial-statistics slots"
        out["mean"] = _assert_close(name + "_mean", st[..., 0], st_ref[..., 0], 1e-4)
        out["rstd"] = _assert_close(name + "_rstd", st[..., 1], st_ref[..., 1], 1e-4)
    return out


def check_conv_fused():
    _setup()
    out = {}
    bf = torch.bfloat16
    out["plain_64to128"] = _conv_fused_case(1, 8, 128, 64, 128, bf, False, False, False, False, "cf_plain")
    out["plain_res_256"] = _conv_fused_case(2, 16, 256, 128, 256, bf, False, False, True, True, "cf_res256")
    out["norm_silu"] = _conv_fused_case(2, 8, 128, 128, 128, bf, True, False, False, True, "cf_norm", tol=6e-3)
    out["norm_silu_res_512to256"] = _conv_fused_case(1, 12, 256, 512, 256, bf, True, False, True, True, "cf_norm512",
                                                     tol=6e-3)
    out["up_256"] = _conv_fused_case(1, 8, 128, 256, 256, bf, False, True, False, True, "cf_up", tol=6e-3)
    out["up_b2_512"] = _conv_fused_case(2, 4, 256, 512, 512, bf, False, True, False, False, "cf_up512", tol=6e-3)
    out["fp16_norm"] = _conv_fused_case(1, 8, 128, 64, 128, torch.float16, True, False, True, True, "cf_fp16")
    # narrow output tile (conv_out: 3 real channels padded to 8; weight rows beyond Cout zero-filled by TMA)
    out["narrow_norm_128to8"] = _conv_fused_case(2, 8, 256, 128, 8, bf, True, False, False, False, "cf_narrow8", tol=6e-3)
    out["narrow_plain_64to64"] = _conv_fused_case(1, 4, 128, 64, 64, bf, False, False, True, False, "cf_narrow64")
    return out


def check_fullsize_conv_fused():
    """the fused ResNet-path convolution at the 1024^2 decode's real extents"""
    _setup()
    bf = torch.bfloat16
    return {"1024_128_norm_res": _conv_fused_case(1, 1024, 1024, 128, 128, bf, True, False, True, True, "cf_full_1024",
                                                  tol=6e-3),
            "512_256_norm": _conv_fused_case(2, 512, 512, 256, 256, bf, True, False, False, True, "cf_full_512", tol=6e-3),
            "up_512to1024_256": _conv_fused_case(1, 512, 512, 256, 256, bf, False, True, False, True, "cf_full_up",
                                                 tol=6e-3)}


# ------------------------------------------------------------------------------------------------ BASELINE shapes
# Parity at the shapes bench.py times (BASELINE.json C3/C4/C5): every kernel against fp32 torch at full size, with a
# per-block error map on top of the global rel-L2 so that ONE wrong output tile (a tile-index decode slip, a barrier phase slip,
# a tail tile) cannot hide in the average.
def _assert_close_blocks(name, got, ref, tol, block_tol, br=128, bc=128):
    """global rel-L2 <= tol AND every br x bc block's rel-L2 (vs the block's own reference norm) <= block_tol"""
    err = _assert_close(name, got, ref, tol)
    g, r = got.reshape(-1, got.shape[-1]), ref.reshape(-1, ref.shape[-1])
    R, Cc = g.shape
    Rp, Cp = (R + br - 1) // br * br, (Cc + bc - 1) // bc * bc
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
        worst = max(worst, float((e / (n + 1e-20)).max()))
        del dg, dr
    if not worst <= block_tol:
        raise AssertionError(f"{name}: worst {br}x{bc} block rel_l2={worst:.3e} (tol {block_tol:.1e}), global {err:.3e}")
    return {"rel_l2": err, "worst_block": worst}


def _ref_matmul(A, W):
    """fp32 reference product in row chunks (the fp32 copy of a 16384 x 12288 output alone is 805 MB)"""
    Wt = W.float().t().contiguous()
    return torch.cat([A[i:i + 4096].float() @ Wt for i in range(0, A.shape[0], 4096)], 0)


def check_fullsize_gemm_fc1():
    """FLUX fc1 at the C4 bench shape: 16384 x 12288 x 3072, bias + GELU-erf (reference mlx/mmdit.py:827-835)"""
    _setup()
    M, N, K = 16384, 12288, 3072
    A, W, b = _rand((M, K), torch.bfloat16), _rand((N, K), torch.bfloat16, 1 / math.sqrt(K)), _rand((N,), torch.bfloat16, 0.5)
    ref = torch.nn.functional.gelu(_ref_matmul(A, W) + b.float())
    got = ops.gemm(A, W, bias=b, act=ACT_GELU_ERF)
    return _assert_close_blocks("full_fc1", got, ref, 4e-3, 1.2e-2)


def check_fullsize_gemm_single_out():
    """FLUX single-block output projection at the C4 shape: 17408 x 3072 x 15360 with x + gate * (.) in place
    (reference mlx/mmdit.py:736-751; K = [attn | gelu(fc1)] = 5h)"""
    _setup()
    B, S, N, K = 4, 4352, 3072, 15360
    M = B * S
    A, W, b = _rand((M, K), torch.bfloat16), _rand((N, K), torch.bfloat16, 1 / math.sqrt(K)), _rand((N,), torch.bfloat16, 0.5)
    x, g = _rand((M, N), torch.bfloat16), _rand((B, N), torch.bfloat16)
    ref = x.float() + g.float().repeat_interleave(S, 0) * (_ref_matmul(A, W) + b.float())
    got = ops.gemm(A, W, out=x, bias=b, gate=g, res=x, rows_per_batch=S, out_batch_rows=S)
    return _assert_close_blocks("full_single_out", got, ref, 4e-3, 1.2e-2)


def _ref_qk_norm_rope(y, pos, h, heads, d, qw, kw, rope):
    ref = y.clone()
    for which, w in enumerate([qw, kw]):
        t = y[:, which * h:(which + 1) * h].reshape(-1, heads, d)
        if w is not None:
            t = t * torch.rsqrt((t * t).mean(-1, keepdim=True) + 1e-6) * w.float()
        if rope is not None:
            c, sn = rope[pos][:, None, :, 0], rope[pos][:, None, :, 1]
            x0, x1 = t[..., 0::2], t[..., 1::2]
            t = torch.stack([x0 * c - x1 * sn, x0 * sn + x1 * c], dim=-1).reshape(-1, heads, d)
        ref[:, which * h:(which + 1) * h] = t.reshape(-1, h)
    return ref


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
    y = _ref_matmul(A, W) + bias.float()
    pos = (torch.arange(Bt * Ss, device=DEV) % Ss) + off
    ref = _ref_qk_norm_rope(y, pos, h, heads, d, qw, kw, rope)
    other = torch.ones(Bt * S, dtype=torch.bool, device=DEV)
    other[rows] = False
    assert float(fused[other].float().abs().max()) == 0.0, "rows outside the scatter window were written"
    return _assert_close_blocks("full_qkv_fused", fused[rows], ref, 6e-3, 1.5e-2)


def _attention_full_case(B, S, heads, d, dtype, split, name):
    """fp32 reference one head at a time (a 4685^2 fp32 score matrix is 88 MB)"""
    h = heads * d
    qkv = _rand((B * S, 3 * h), dtype)
    o0 = torch.zeros((B * split, h), dtype=dtype, device=DEV)
    o1 = torch.zeros((B * (S - split), h), dtype=dtype, device=DEV)
    ops.attention(qkv, B, S, heads, d, o0, split=split, out1=o1)
    got = torch.cat([o0.reshape(B, split, h), o1.reshape(B, S - split, h)], dim=1)
    ref = torch.empty((B, S, h), dtype=torch.float32, device=DEV)
    x = qkv.reshape(B, S, 3, heads, d)
    for b in range(B):
        for hd in range(heads):
            q, k, v = x[b, :, 0, hd].float(), x[b, :, 1, hd].float(), x[b, :, 2, hd].float()
            ref[b, :, hd * d:(hd + 1) * d] = torch.softmax(q @ k.t() / math.sqrt(d), dim=-1) @ v
    return _assert_close_blocks(name, got.reshape(B * S, h), ref.reshape(B * S, h), 1e-2, 3e-2, br=128, bc=d)


def check_fullsize_attention():
    """joint attention at the bench sequence lengths, all 24 heads: FLUX d=128 S=4352 (C4: 17 x 256 exactly) and
    S=4608 (C5), SD3 d=64 fp16 S=4685 (C3: ragged tail), outputs split at the text/image boundary as the model does
    (reference mlx/mmdit.py:594-657)"""
    _setup()
    return {"flux_S4352": _attention_full_case(2, 4352, 24, 128, torch.bfloat16, 256, "full_att_4352"),
            "flux_S4608": _attention_full_case(1, 4608, 24, 128, torch.bfloat16, 512, "full_att_4608"),
            "sd3_S4685": _attention_full_case(2, 4685, 24, 64, torch.float16, 4096, "full_att_4685")}


def _conv_full_case(B, H, W, Cin, Cout, dtype, res, name):
    x = _rand((B, H, W, Cin), dtype)
    w = _rand((Cout, 3, 3, Cin), dtype, 1 / math.sqrt(9 * Cin))
    b = _rand((Cout,), dtype, 0.5)
    r = _rand((B, H, W, Cout), dtype) if res else None
    got = ops.conv3x3(x, w, bias=b, res=r)
    wf = w.float().permute(0, 3, 1, 2).contiguous()
    ref = torch.empty((B, H, W, Cout), dtype=torch.float32, device=DEV)
    rows = max(8, (1 << 24) // (W * max(Cin, Cout)))       # reference in horizontal bands with a one-row halo
    for b_ in range(B):
        for y0 in range(0, H, rows):
            y1 = min(H, y0 + rows)
            ya, yb = max(0, y0 - 1), min(H, y1 + 1)
            xin = x[b_, ya:yb].float().permute(2, 0, 1)[None]
            xin = torch.nn.functional.pad(xin, (1, 1, 1 if y0 == 0 else 0, 1 if y1 == H else 0))
            o = torch.nn.functional.conv2d(xin, wf, b.float())[0].permute(1, 2, 0)
            ref[b_, y0:y1] = o
    if res:
        ref += r.float()
    return _assert_close_blocks(name, got.reshape(-1, Cout), ref.reshape(-1, Cout), 4e-3, 1.2e-2, br=128, bc=min(128, Cout))


def check_fullsize_conv():
    """VAE decoder convs at the 1024^2 decode's real extents (reference mlx/vae.py:60-101,146-149):
    1024 x 1024 x 128 -> 128 (+ skip), 512 x 512 x 256 -> 256, and the 512 -> 256 channel change at 512^2"""
    _setup()
    return {"1024_128": _conv_full_case(1, 1024, 1024, 128, 128, torch.bfloat16, True, "full_conv_1024"),
            "512_256": _conv_full_case(2, 512, 512, 256, 256, torch.bfloat16, False, "full_conv_512"),
            "512_512to256": _conv_full_case(1, 512, 512, 512, 256, torch.bfloat16, False, "full_conv_512to256")}


def check_fullsize_groupnorm():
    """GroupNorm(32) + SiLU at 1024 x 1024 x 128 and 512 x 512 x 256, batch 2 (reference mlx/vae.py:72-80)"""
    _setup()
    out = {}
    for (B, H, W, Cc) in [(2, 1024, 1024, 128), (2, 512, 512, 256)]:
        dt = torch.bfloat16
        x = _rand((B, H, W, Cc), dt, 1.5) + 0.7
        gamma, beta = _rand((Cc,), dt, 0.1) + 1.0, _rand((Cc,), dt, 0.1)
        stats = ops.groupnorm_stats(x, 32, 1e-5)
        mean = torch.empty((B, 32), device=DEV, dtype=torch.float64)
        var = torch.empty((B, 32), device=DEV, dtype=torch.float64)
        for b_ in range(B):
            xf = x[b_].reshape(H * W, 32, Cc // 32).double()
            mean[b_] = xf.mean(dim=(0, 2))
            var[b_] = xf.var(dim=(0, 2), unbiased=False)
        out[f"mean_{Cc}"] = _assert_close("full_gn_mean", stats[..., 0], mean.float(), 1e-4)
        out[f"rstd_{Cc}"] = _assert_close("full_gn_rstd", stats[..., 1], torch.rsqrt(var + 1e-5).float(), 1e-4)
        got = ops.groupnorm_apply(x, stats, gamma, beta, 32, True)
        for b_ in range(B):
            xn = (x[b_].float().reshape(H * W, 32, Cc // 32) - mean[b_].float()[None, :, None]) * \
                torch.rsqrt(var[b_] + 1e-5).float()[None, :, None]
            ref = torch.nn.functional.silu((xn.reshape(H * W, Cc) * gamma.float() + beta.float()).to(dt).float())
            out[f"apply_{Cc}_{b_}"] = _assert_close("full_gn_apply", got[b_].reshape(H * W, Cc), ref, 4e-3)
    return out


FULLSIZE_CHECKS = [check_fullsize_gemm_fc1, check_fullsize_gemm_single_out, check_fullsize_gemm_qkv_fused,
                   check_fullsize_attention, check_fullsize_conv, check_fullsize_groupnorm, check_fullsize_conv_fused]


ALL_CHECKS = [
    check_gemm_single_tile, check_gemm_multi_k, check_gemm_shapes, check_gemm_persistent_large, check_gemm_epilogues,
    check_gemm_fp16, check_gemm_inplace_residual, check_gemm_w_n_major, check_gemm_fused_qk_norm_rope,
    check_gemm_pair_kernel, check_gemm_pair_legacy_store, check_conv3x3, check_conv3x3_s2, check_img2img_kernels, check_dequant_q4,
    check_text_kernels, check_attention_small,
    check_attention_d128_one_tile, check_attention_d128, check_attention_d64, check_attention_large_scores,
    check_attention_v3_explicit, check_attention_v3s_kernel, check_attention_v3_variants, check_attention_v5_kernel, check_attention_v6_kernel,
    check_conv_fused,
    check_ln_modulate, check_qk_norm_rope, check_layout_kernels, check_sampler_kernels, check_groupnorm,
    check_softmax_image_post, check_edge_cases, check_error_paths,
] + FULLSIZE_CHECKS

EXPERIMENTAL_CHECKS = []

