"""GPU checks of the opt-in FP8 (e4m3) linears.  Every reference contains the same quantisation as the kernels, so no
tolerance here depends on how much accuracy e4m3 costs: the quantiser is checked bit for bit, the GEMM against an fp32
product of the dequantised operands, the models against the fake-quantised oracle (tests/fp8_ref.py)."""
import ctypes as C
import math
from dataclasses import replace

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
bf16, fp16, e4m3 = torch.bfloat16, torch.float16, torch.float8_e4m3fn


@pytest.fixture(scope="module")
def kc():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    from tests import kernel_checks

    kernel_checks._setup()
    return kernel_checks


def _deq(q, scale):
    return q.float() * scale[:, None]


# ------------------------------------------------------------------------------------------------ quantiser
@pytest.mark.parametrize("dtype", [bf16, fp16])
@pytest.mark.parametrize("cols", [16, 64, 3072, 12288, 15360])
def test_quantize_rows_bit_exact(kc, dtype, cols):
    from diffusionkit_b200 import ops
    from tests.fp8_ref import quantize_rows_e4m3

    rows = 37
    buf = kc._rand((rows, cols + 24), dtype, 3.0)
    buf[5] = 0                                            # an all-zero row
    buf[7, 3] = 448.0 * 4                                 # a row whose maximum is 448 * 2^k
    buf[9] *= 1e-3
    x = buf[:, 8:8 + cols]                                # strided rows, 16-byte aligned
    q, s = ops.quantize_rows_e4m3(x)
    q2, s2 = ops.quantize_rows_e4m3(x)
    want_q, want_s = quantize_rows_e4m3(x.cpu())
    assert torch.equal(s.cpu(), want_s)
    assert torch.equal(q.float().cpu(), want_q)
    assert torch.equal(q.view(torch.uint8), q2.view(torch.uint8)) and torch.equal(s, s2)
    assert float(s[5]) == 1.0 and float(q[5].float().abs().max()) == 0.0


@pytest.mark.parametrize("B,S,h,dtype", [(2, 37, 3072, bf16), (1, 64, 1536, fp16), (3, 5, 128, bf16), (1, 9, 4096, bf16)])
def test_ln_modulate_fp8(kc, B, S, h, dtype):
    from diffusionkit_b200 import ops

    x = kc._rand((B * S, h), dtype, 2.0) + 0.5
    mod = kc._rand((B, 6 * h), dtype, 0.3)
    shift, scale = mod[:, 0:h], mod[:, h:2 * h]
    ln = torch.nn.functional.layer_norm(x.float(), (h,), eps=1e-6)
    ref = ln * (1 + scale.float().repeat_interleave(S, 0)) + shift.float().repeat_interleave(S, 0)
    q, s = ops.ln_modulate_fp8(x, shift, scale, S, 1e-6)
    want_s = ref.abs().amax(dim=1) / 448.0
    assert float(((s - want_s).abs() / want_s).max()) <= 1e-5
    # half an e4m3 ulp of each element (3 mantissa bits, subnormal step 2^-9) times the row's scale, plus the slack of
    # evaluating LayerNorm in fp32 in another order
    y = ref / s[:, None]
    ulp = torch.floor(torch.log2(y.abs().clamp(2.0 ** -6, 448.0))).exp2() * 2.0 ** -3
    err = (_deq(q, s) - ref).abs()
    bound = (0.5 * ulp + 1e-4 * y.abs() + 1e-4) * s[:, None]
    assert bool((err <= bound).all()), float((err / bound).max())


# ------------------------------------------------------------------------------------------------ GEMM
def _quant_pair(kc, M, N, K, dtype, spread=False):
    """e4m3 operands + scales as the quantiser makes them.  spread: row / column magnitudes from 2^-20 to 2^20."""
    from diffusionkit_b200 import ops

    A = kc._rand((M, K + 16), torch.float32)             # a row stride wider than K
    W = kc._rand((N, K), torch.float32, 1 / math.sqrt(K))
    Aq, a_s = ops.quantize_rows_e4m3(A.to(dtype)[:, :K])
    Wq, w_s = ops.quantize_rows_e4m3(W.to(dtype))
    if spread:
        a_s = a_s * torch.exp2(torch.randint(-20, 21, (M,), device=DEV).float())
        w_s = w_s * torch.exp2(torch.randint(-20, 21, (N,), device=DEV).float())
        keep = 2.0 ** -6 / (a_s[:, None] * w_s[None, :]).abs().max()      # keep the 16-bit output finite
        a_s = (a_s * keep).contiguous()
    return Aq, a_s, Wq, w_s


def _gemm_fp8_case(kc, M, N, K, dtype, epi="", spread=False):
    """dk_gemm_fp8 against ref_gemm of the dequantised operands; epi as in tests/kernel_checks._gemm_case"""
    from diffusionkit_b200 import ops

    e = set(epi.split())
    act = (kc.ACT_GELU_ERF if "gelu" in e else kc.ACT_SILU if "silu" in e else kc.ACT_NONE)
    Bt = 2 if "remap" in e else 1
    Aq, a_s, Wq, w_s = _quant_pair(kc, M, N, K, dtype, spread=spread)
    b = kc._rand((N,), dtype, 0.5 if not spread else 1e-3) if "bias" in e else None
    g = kc._rand((Bt, N), dtype) if "gate" in e else None
    r = kc._rand((M, N), dtype) if e & {"res", "inplace"} else None
    ref = kc.ref_gemm(_deq(Aq, a_s), _deq(Wq, w_s), b, act, g, r)
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
    got = ops.gemm_fp8(Aq, a_s, Wq, w_s, dtype=dtype, out=out, bias=b, act=act, gate=g, res=r, **kw)
    if buf is not None:
        got = buf[window]
        outside = torch.ones(buf.shape, dtype=torch.bool, device=DEV)
        outside[window] = False
        assert bool((buf[outside] == 7.0).all()), "bytes outside the output window were written"
    return kc._assert_close(f"gemm_fp8_{M}x{N}x{K}_{epi}", got, ref, 4e-3)


GEMM_CASES = [
    (128, 256, 128, bf16, ""), (128, 256, 1024, bf16, ""),                      # single tile, multi-k
    (256, 512, 400, bf16, ""), (300, 264, 208, bf16, ""), (77, 64, 64, bf16, ""),   # K % 128 != 0, ragged M, BN 64
    (1000, 3072, 1536, bf16, ""), (20, 1024, 3072, bf16, ""), (128, 128, 128, bf16, ""),
    (4096, 4608, 1024, bf16, "bias"), (8192, 4608, 1024, bf16, "bias"),          # more tiles than resident clusters
    (384, 512, 256, bf16, "bias"), (384, 512, 256, bf16, "bias gelu"), (384, 512, 256, bf16, "bias silu"),
    (384, 512, 256, bf16, "bias gate res"), (600, 512, 256, bf16, "bias gate res remap"),
    (1024, 1152, 256, bf16, "bias gate res"), (1000, 520, 256, bf16, "gelu window"),
    (256, 256, 128, bf16, "inplace"), (1000, 520, 256, bf16, "gate inplace"),
    (300, 512, 320, fp16, "bias gelu"), (300, 512, 320, fp16, "bias"),
]


@pytest.mark.parametrize("M,N,K,dtype,epi", GEMM_CASES)
def test_gemm_fp8(kc, M, N, K, dtype, epi):
    _gemm_fp8_case(kc, M, N, K, dtype, epi)


@pytest.mark.parametrize("M,N,K,dtype,epi", [(384, 512, 256, bf16, "bias"), (300, 264, 208, fp16, ""),
                                             (1000, 520, 256, bf16, "gate res")])
def test_gemm_fp8_scales_apply_per_row_and_column(kc, M, N, K, dtype, epi):
    _gemm_fp8_case(kc, M, N, K, dtype, epi, spread=True)


@pytest.mark.parametrize("M,N,K,epi", [(16384, 12288, 3072, "bias gelu"), (17408, 3072, 15360, "bias gate inplace")])
def test_gemm_fp8_full_size(kc, M, N, K, epi):
    """the FLUX fc1 and single-block out projection shapes; K = 15360 is the accumulation-precision case"""
    _gemm_fp8_case(kc, M, N, K, bf16, epi)


def test_gemm_fp8_deterministic(kc):
    from diffusionkit_b200 import ops

    Aq, a_s, Wq, w_s = _quant_pair(kc, 1000, 1536, 3072, bf16)
    a = ops.gemm_fp8(Aq, a_s, Wq, w_s, dtype=bf16)
    b = ops.gemm_fp8(Aq, a_s, Wq, w_s, dtype=bf16)
    assert torch.equal(a, b)


@pytest.mark.parametrize("Bt,Ss,off,S,heads,d,dtype,use_norm", [(2, 100, 28, 128, 2, 128, bf16, True),
                                                               (1, 300, 0, 300, 4, 64, fp16, True),
                                                               (2, 77, 5, 90, 2, 128, bf16, False),
                                                               (1, 4352, 0, 4352, 24, 128, bf16, True)])
def test_gemm_fp8_fused_qk_norm_rope(kc, Bt, Ss, off, S, heads, d, dtype, use_norm):
    from diffusionkit_b200 import ops

    h, K = heads * d, (3072 if S == 4352 else 192)
    Aq, a_s, Wq, w_s = _quant_pair(kc, Bt * Ss, 3 * h, K, dtype)
    bias = kc._rand((3 * h,), dtype, 0.3)
    qw = (kc._rand((d,), dtype, 0.1) + 1.0) if use_norm else None
    kw = (kc._rand((d,), dtype, 0.1) + 1.0) if use_norm else None
    rope = kc._rope_table(S, d, DEV)
    fused = torch.zeros((Bt * S, 3 * h), dtype=dtype, device=DEV)
    ops.gemm_fp8(Aq, a_s, Wq, w_s, out=fused, bias=bias, rows_per_batch=Ss, out_batch_rows=S, out_row_off=off,
                 qk=(heads, d, qw, kw, rope, 1e-6))
    rows = torch.cat([torch.arange(b * S + off, b * S + off + Ss) for b in range(Bt)]).to(DEV)
    other = torch.ones(Bt * S, dtype=torch.bool, device=DEV)
    other[rows] = False
    if bool(other.any()):
        assert float(fused[other].float().abs().max()) == 0.0, "rows outside the scatter window were written"
    pos = (torch.arange(Bt * Ss, device=DEV) % Ss) + off
    ref = kc.ref_qk_norm_rope(kc.ref_gemm(_deq(Aq, a_s), _deq(Wq, w_s), bias), pos, heads, d, qw, kw, rope)
    kc._assert_close(f"gemm_fp8_fusedqk_{d}", fused[rows], ref, 6e-3)   # the bound of the 16-bit fused check


def test_gemm_fp8_error_paths(kc):
    from diffusionkit_b200 import _lib, ops

    c = ops.ctx(0)
    Aq, a_s, Wq, w_s = _quant_pair(kc, 128, 128, 128, bf16)
    out = torch.empty((128, 128), dtype=bf16, device=DEV)
    n0 = c.launches

    def call(a_scale=a_s, w_scale=w_s, **over):
        a = _lib.GemmArgs()
        a.dtype, a.M, a.N, a.K = _lib.DK_BF16, 128, 128, 128
        a.A, a.lda, a.W, a.ldw, a.out, a.ldc = Aq.data_ptr(), 128, Wq.data_ptr(), 128, out.data_ptr(), 128
        for k, v in over.items():
            setattr(a, k, v)
        rc = c.lib.dk_gemm_fp8(c.handle, C.byref(a), _lib.ptr(a_scale), _lib.ptr(w_scale), c.stream)
        return rc, c.lib.dk_last_error().decode()

    for kw, word in [(dict(w_n_major=1), "w_n_major"), (dict(a_scale=None), "required"),
                     (dict(w_scale=None), "required"), (dict(K=120), "K (120)"), (dict(lda=136), "lda"),
                     (dict(ldw=72), "ldw"), (dict(A=Aq.data_ptr() + 8), "aligned"),
                     (dict(a_scale=a_s[1:]), "aligned"), (dict(dtype=5), "dtype")]:
        rc, msg = call(**kw)
        assert rc != 0 and "dk_gemm_fp8" in msg and word in msg, (kw.keys(), rc, msg)
    assert c.launches == n0
    with pytest.raises(_lib.DkError):
        ops.gemm_fp8(Aq.view(torch.uint8), a_s, Wq, w_s, dtype=bf16)


# ------------------------------------------------------------------------------------------------ models
def _mmdit_setup(cfg, dtype, B, lat, T, seed=7):
    import diffusionkit_b200 as dk
    from diffusionkit_b200.weights import init_params, mmdit_param_specs

    p16 = {k: v.to(dtype) for k, v in init_params(mmdit_param_specs(cfg), seed=seed, dtype=torch.float32).items()}
    gen = torch.Generator().manual_seed(5)
    latent = torch.randn((B, lat[0], lat[1], 16), generator=gen).to(dtype)
    text = torch.randn((B, T, cfg.token_level_text_embed_dim), generator=gen).to(dtype)
    pooled = torch.randn((B, cfg.pooled_text_embed_dim), generator=gen).to(dtype)
    m = dk.MMDiT(cfg, {k: v.to(DEV) for k, v in p16.items()})
    m.cache_modulation_params(pooled.to(DEV), [752.0, 0.0])

    def run():
        out = m(latent_image_embeddings=latent.to(DEV), token_level_text_embeddings=text.to(DEV).unsqueeze(2),
                timestep=torch.full((B,), 752.0))
        torch.cuda.synchronize()
        return out.clone()

    return m, run, p16, (latent, text, pooled)


def _oracles(cfg, p16, inputs):
    from diffusionkit_b200.mmdit import fp8_covered_linears
    from oracle.mmdit_ref import MMDiTRef
    from tests.fp8_ref import FakeQuantMMDiTRef
    from tests.oracle_bridge import ref_config

    latent, text, pooled = inputs
    t = torch.tensor([752.0])
    p = {k: v.float() for k, v in p16.items()}
    outs = []
    for ref in (FakeQuantMMDiTRef(ref_config(cfg), p, fp8_covered_linears(cfg)), MMDiTRef(ref_config(cfg), p)):
        ref.cache_modulation_params(pooled.float(), t)
        outs.append(ref(latent.float(), text.float(), t.repeat(latent.shape[0])))
    return outs


# e4m3 rounding is discontinuous: where the engine's 16-bit activations differ from the oracle's fp32 ones by a 16-bit
# ulp, a few per cent of the elements fall on the neighbouring e4m3 value, an eighth of their magnitude away.  So the
# fake-quantised oracle cannot bound the FP8 forward as tightly as the plain oracle bounds the 16-bit one (2e-2); the
# PSNR bound is the 16-bit one.  Measured on an H100: see DESIGN.md "FP8 linears".
FQ_REL_L2 = 5e-2


def _mmdit_fp8_case(cfg, dtype, B, lat, T):
    from tests.model_checks import psnr, rel_l2

    m, run, p16, inputs = _mmdit_setup(cfg, dtype, B, lat, T)
    m.set_fp8(True)
    got = run()
    want_fq, want_plain = _oracles(cfg, p16, inputs)
    assert bool(torch.isfinite(got.float()).all())
    r, ps = rel_l2(got, want_fq), psnr(want_fq, got)
    print(f"fp8 mmdit vs fake-quantised oracle rel_l2={r:.3e} psnr={ps:.1f}; vs unquantised oracle "
          f"rel_l2={rel_l2(got, want_plain):.3e} psnr={psnr(want_plain, got):.1f}")
    assert r <= FQ_REL_L2 and ps >= 35.0, f"fp8 mmdit rel_l2={r:.3e} psnr={ps:.1f}"


def test_mmdit_fp8_flux_tiny(kc):
    from diffusionkit_b200.config import tiny_flux_config

    _mmdit_fp8_case(tiny_flux_config(), bf16, 2, (8, 12), 16)


def test_mmdit_fp8_sd3_tiny(kc):
    from diffusionkit_b200.config import tiny_sd3_config

    _mmdit_fp8_case(tiny_sd3_config(), fp16, 2, (8, 8), 24)


def test_mmdit_fp8_sd35_tiny(kc):
    from diffusionkit_b200.config import tiny_sd35_config

    _mmdit_fp8_case(tiny_sd35_config(), fp16, 2, (8, 12), 24)


def test_mmdit_fp8_fullwidth_flux(kc):
    """FLUX.1-schnell's real width and sequence (h = 3072, S = 4096 + 256), one double and one single block"""
    from diffusionkit_b200.config import MODEL_CONFIGS

    full = MODEL_CONFIGS["argmaxinc/mlx-FLUX.1-schnell"]
    cfg = replace(full, depth_multimodal=1, depth_unified=1, hidden_size_override=full.hidden_size)
    _mmdit_fp8_case(cfg, bf16, 1, (128, 128), 256)


@pytest.mark.parametrize("kind", ["flux", "sd3"])
def test_pipeline_fp8(kc, kind):
    """the tiny FLUX and CFG SD3 pipelines with FP8 on: finite, switchable, and on -> off restores the 16-bit result"""
    import diffusionkit_b200 as dk
    from diffusionkit_b200.config import VAEDecoderConfig, tiny_flux_config, tiny_sd3_config
    from diffusionkit_b200.weights import init_params, mmdit_param_specs, vae_decoder_param_specs
    from tests.model_checks import psnr, rel_l2

    if kind == "flux":
        cfg, dtype, steps, cfgw, shift, T = tiny_flux_config(), bf16, 4, 0.0, 1.0, 16
        Pipe, mv = dk.FluxPipeline, "argmaxinc/mlx-FLUX.1-schnell"
    else:
        cfg, dtype, steps, cfgw, shift, T = tiny_sd3_config(), fp16, 6, 5.0, 3.0, 24
        Pipe, mv = dk.DiffusionPipeline, "argmaxinc/mlx-stable-diffusion-3-medium"
    p = init_params(mmdit_param_specs(cfg), seed=7, dtype=dtype, device=DEV)
    vp = init_params(vae_decoder_param_specs(VAEDecoderConfig()), seed=8, dtype=dtype, device=DEV)
    pipe = Pipe(w16=True, a16=True, shift=shift, model_version=mv, mmdit_config=cfg, params=p, vae_params=vp)
    assert pipe.fp8 is False
    cond, pooled = pipe.synthetic_text_embeddings(n_images=2, text_len=T)

    def run():
        lat, _ = pipe.denoise_latents(cond, pooled, num_steps=steps, cfg_weight=cfgw, latent_size=(8, 12), seed=[11, 12])
        return lat.clone(), pipe.decode_latents_to_image(lat).clone()

    lat16, img16 = run()
    pipe.set_fp8(True)
    assert pipe.fp8 is True
    lat8, img8 = run()
    pipe.set_fp8(False)
    lat16b, img16b = run()
    pipe.set_fp8(True)
    lat8b, img8b = run()
    assert torch.equal(lat16, lat16b) and torch.equal(img16, img16b)
    assert torch.equal(lat8, lat8b) and torch.equal(img8, img8b)
    assert not torch.equal(lat8, lat16)
    ps = psnr(img16, img8)
    print(f"{kind} fp8 vs 16-bit pipeline: latent rel_l2={rel_l2(lat8, lat16):.3e} decoded RGB psnr={ps:.1f}")
    assert bool(torch.isfinite(lat8).all()) and ps >= 20.0


def test_switch_drops_and_recaptures_graphs(kc):
    from diffusionkit_b200.config import tiny_flux_config

    m, run, _, _ = _mmdit_setup(tiny_flux_config(), bf16, 2, (8, 12), 16)
    m.use_cuda_graphs = True
    never = run()
    state = next(iter(m._shapes._states.values()))
    assert "graph" in state and "ws8" not in state
    m.set_fp8(True)
    assert "graph" not in state
    on = run()
    assert "graph" in state and "ws8" in state
    assert torch.equal(on, run())                         # replay
    m.set_fp8(False)
    assert "graph" not in state and "ws8" not in state and not m._fp8_w
    assert torch.equal(never, run())
    m.set_fp8(True)
    assert torch.equal(on, run())
    m.use_cuda_graphs = False
    assert torch.equal(on, run())                         # eager == captured


def test_lora_under_fp8(kc):
    from diffusionkit_b200.config import tiny_flux_config
    from diffusionkit_b200.lora import LoRA

    cfg = tiny_flux_config()
    g = torch.Generator().manual_seed(3)
    h = cfg.hidden_size
    names = {"multimodal_transformer_blocks.0.image_transformer_block.attn.q_proj.weight": (h, h),
             "unified_transformer_blocks.0.transformer_block.mlp.fc2.weight": (h, cfg.mlp_ratio * h),
             "final_layer.linear.weight": None}
    m, run, _, _ = _mmdit_setup(cfg, bf16, 2, (8, 12), 16)
    names["final_layer.linear.weight"] = tuple(m.w_final.shape)
    lora = LoRA("a", {n: (torch.randn((o, 4), generator=g) * 0.2, torch.randn((4, i), generator=g) * 0.2)
                      for n, (o, i) in names.items()})
    m.set_fp8(True)
    base = run()
    ptrs = {k: (q.data_ptr(), s.data_ptr()) for k, (q, s) in m._fp8_w.items()}
    m.apply_lora([(lora, 1.0)])
    merged = run()
    assert not torch.equal(base, merged)
    # the same adapters merged first, then quantised from scratch
    m2, run2, _, _ = _mmdit_setup(cfg, bf16, 2, (8, 12), 16)
    m2.apply_lora([(lora, 1.0)])
    m2.set_fp8(True)
    assert torch.equal(merged, run2())
    m.apply_lora([(lora, 0.5)])
    half = run()
    assert {k: (q.data_ptr(), s.data_ptr()) for k, (q, s) in m._fp8_w.items()} == ptrs
    assert not torch.equal(half, merged)
    m.apply_lora([])
    assert torch.equal(base, run())
    assert {k: (q.data_ptr(), s.data_ptr()) for k, (q, s) in m._fp8_w.items()} == ptrs
