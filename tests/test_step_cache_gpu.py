"""GPU checks of the opt-in first-block step cache: its two kernels, bit-identity with the cache off at threshold 0,
fixed skip patterns against the fp32 oracle replaying the same decisions (tests/step_cache_ref.py), the engine's
per-step change against the oracle's, the resets, graphs, and FP8 with the cache on."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
bf16, fp16 = torch.bfloat16, torch.float16


@pytest.fixture(scope="module")
def kc():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    from tests import kernel_checks

    kernel_checks._setup()
    return kernel_checks


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("dtype", [bf16, fp16])
@pytest.mark.parametrize("nseq,rows,h,x_seq,ldx", [(1, 4096, 3072, 4096, 3072), (8, 4096, 1536, 4096, 1536),
                                                   (3, 37, 128, 37, 128), (2, 1, 8, 1, 8),
                                                   (2, 300, 256, 377, 264), (5, 253, 520, 300, 520)])
def test_residual_delta(kc, dtype, nseq, rows, h, x_seq, ldx):
    """sums within 1e-5 of fp64, r bit-exact, two launches bit-identical; ragged row counts, strided rows and
    sequences that start past the previous one's end (x_seq > rows, as the image rows of FLUX's joint sequence)"""
    from diffusionkit_b200 import ops

    g = torch.Generator(device=DEV).manual_seed(rows + h)
    xbuf = (torch.randn((nseq * x_seq, ldx), generator=g, device=DEV) * 2.0).to(dtype)
    x = xbuf if ldx == h else xbuf[:, 8:8 + h]                # a row stride wider than h, 16-byte aligned
    base = (torch.randn((nseq * rows, h), generator=g, device=DEV)).to(dtype)
    prev = torch.randn((nseq * rows, h), generator=g, device=DEV) * 0.5
    r = torch.empty((nseq * rows, h), dtype=torch.float32, device=DEV)
    sums = ops.residual_delta(x, base, nseq, rows, x_seq_rows=x_seq, r_out=r, prev=prev)
    sums2 = ops.residual_delta(x, base, nseq, rows, x_seq_rows=x_seq, prev=prev)
    want_r, want = kc.ref_residual_delta(x, base, nseq, rows, x_seq, rows, prev)
    assert torch.equal(r, want_r)
    assert torch.equal(sums, sums2)
    err = ((sums.double() - want) / want).abs().max()
    assert float(err) <= 1e-5, float(err)
    r2 = torch.zeros_like(r)
    assert ops.residual_delta(x, base, nseq, rows, x_seq_rows=x_seq, r_out=r2) is None     # store only
    assert torch.equal(r2, r)


def test_residual_delta_zero_prev(kc):
    from diffusionkit_b200 import ops

    x = torch.ones((64, 128), dtype=bf16, device=DEV)
    sums = ops.residual_delta(x, torch.zeros_like(x), 2, 32, prev=torch.zeros((64, 128), device=DEV))
    assert sums.tolist() == [[4096.0, 0.0], [4096.0, 0.0]]


@pytest.mark.parametrize("dtype", [bf16, fp16])
@pytest.mark.parametrize("n", [8, 4096 * 1536, 1000 * 24])
def test_residual_apply_bit_exact(kc, dtype, n):
    from diffusionkit_b200 import ops

    g = torch.Generator(device=DEV).manual_seed(n)
    x = (torch.randn((n,), generator=g, device=DEV) * 3.0).to(dtype)
    r = torch.randn((n,), generator=g, device=DEV) * torch.exp2(torch.randint(-12, 4, (n,), generator=g, device=DEV))
    want = (x.float() + r).to(dtype)
    assert torch.equal(ops.residual_apply(x, r), want)
    y = x.clone()
    ops.residual_apply(y, r, out=y)                        # in place
    assert torch.equal(y, want)


def test_step_cache_error_paths(kc):
    from diffusionkit_b200 import _lib, ops

    c = ops.ctx(0)
    x = torch.zeros((64, 128), dtype=bf16, device=DEV)
    f = torch.zeros((64, 128), dtype=torch.float32, device=DEV)
    s = torch.zeros((4, 2), dtype=torch.float32, device=DEV)
    ws = torch.zeros((2048,), dtype=torch.float32, device=DEV)
    n0 = c.launches

    def delta(**over):
        a = dict(dtype=_lib.DK_BF16, x=x.data_ptr(), ldx=128, xs=32, base=x.data_ptr(), ldb=128, bs=32,
                 r=f.data_ptr(), prev=f.data_ptr(), sums=s.data_ptr(), ws=ws.data_ptr(), nseq=2, rows=32, h=128)
        a.update(over)
        rc = c.lib.dk_residual_delta(c.handle, a["dtype"], a["x"], a["ldx"], a["xs"], a["base"], a["ldb"], a["bs"],
                                     a["r"], a["prev"], a["sums"], a["ws"], a["nseq"], a["rows"], a["h"], c.stream)
        return rc, c.lib.dk_last_error().decode()

    for over, word in [(dict(x=None), "required"), (dict(base=None), "required"), (dict(rows=0), "empty"),
                       (dict(nseq=0), "empty"), (dict(h=12, ldx=12, ldb=12), "multiples of 8"), (dict(ldx=64), "ldx"),
                       (dict(xs=16), "x_seq_rows"), (dict(r=None, prev=None), "nothing to do"),
                       (dict(sums=None), "needs sums"), (dict(ws=None), "needs sums"),
                       (dict(x=x.data_ptr() + 2), "aligned"), (dict(prev=f.data_ptr() + 4), "aligned"),
                       (dict(dtype=7), "dtype")]:
        rc, msg = delta(**over)
        assert rc != 0 and "dk_residual_delta" in msg and word in msg, (over, rc, msg)

    def apply(**over):
        a = dict(dtype=_lib.DK_FP16, x=x.data_ptr(), r=f.data_ptr(), out=x.data_ptr(), n=x.numel())
        a.update(over)
        rc = c.lib.dk_residual_apply(c.handle, a["dtype"], a["x"], a["r"], a["out"], a["n"], c.stream)
        return rc, c.lib.dk_last_error().decode()

    for over, word in [(dict(r=None), "required"), (dict(out=None), "required"), (dict(n=12), "multiple of 8"),
                       (dict(n=0), "multiple of 8"), (dict(out=x.data_ptr() + 2), "aligned"),
                       (dict(r=f.data_ptr() + 8), "aligned"), (dict(dtype=-1), "dtype")]:
        rc, msg = apply(**over)
        assert rc != 0 and "dk_residual_apply" in msg and word in msg, (over, rc, msg)
    rc = c.lib.dk_residual_apply(None, _lib.DK_BF16, x.data_ptr(), f.data_ptr(), x.data_ptr(), 8, c.stream)
    assert rc != 0 and "null ctx" in c.lib.dk_last_error().decode()
    assert c.launches == n0


# ------------------------------------------------------------------------------------------------ pipelines
CASES = {  # kind: (config factory name, dtype, steps, cfg weight, shift, text length, pipeline, model version)
    "flux": ("tiny_flux_config", bf16, 6, 0.0, 1.0, 16, "FluxPipeline", "argmaxinc/mlx-FLUX.1-schnell"),
    "sd3": ("tiny_sd3_config", fp16, 6, 5.0, 3.0, 24, "DiffusionPipeline", "argmaxinc/mlx-stable-diffusion-3-medium"),
    "sd35": ("tiny_sd35_config", fp16, 6, 5.0, 3.0, 24, "DiffusionPipeline",
             "argmaxinc/mlx-stable-diffusion-3.5-large"),
}
LAT = (8, 12)
SEEDS = [11, 12]


def _pipe(kind, decoder=False):
    import diffusionkit_b200 as dk
    from diffusionkit_b200 import config
    from diffusionkit_b200.config import VAEDecoderConfig
    from diffusionkit_b200.weights import init_params, mmdit_param_specs, vae_decoder_param_specs

    make, dtype, _, _, shift, T, cls, mv = CASES[kind]
    cfg = getattr(config, make)()
    p = init_params(mmdit_param_specs(cfg), seed=7, dtype=dtype, device=DEV)
    vp = init_params(vae_decoder_param_specs(VAEDecoderConfig()), seed=8, dtype=dtype, device=DEV) if decoder else None
    pipe = getattr(dk, cls)(w16=True, a16=True, shift=shift, model_version=mv, mmdit_config=cfg, params=p,
                            vae_params=vp, load_decoder=decoder)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
    return pipe, cfg, p, cond, pooled


def _denoise(pipe, kind, cond, pooled):
    steps, cfgw = CASES[kind][2], CASES[kind][3]
    lat, _ = pipe.denoise_latents(cond, pooled, num_steps=steps, cfg_weight=cfgw, latent_size=LAT, seed=SEEDS)
    torch.cuda.synchronize()
    return lat.clone()


def _oracle(kind, cfg, p, cond, pooled, decisions):
    """the fp32 oracle loop over the whole batch, replaying `decisions` -> (final latents, its (rel, skipped) log)"""
    from oracle import sampler_ref as sr
    from tests.oracle_bridge import ref_config
    from tests.step_cache_ref import SplitMMDiTRef, StepCacheRef

    _, dtype, steps, cfgw, shift, _, _, _ = CASES[kind]
    sampler = sr.FluxSamplerRef(shift) if kind == "flux" else sr.ModelSamplingDiscreteFlowRef(shift)
    sig = sr.get_sigmas(sampler, steps)
    H, W = LAT
    x0 = torch.cat([sampler.noise_scaling(float(sig[0]), sr.get_noise(s, H, W), sr.get_empty_latent(H, W))
                    for s in SEEDS])
    model = StepCacheRef(SplitMMDiTRef(ref_config(cfg), {k: v.float().cpu() for k, v in p.items()}),
                         decisions=decisions)
    x = sr.sample_euler(model, model.cache_modulation_params, x0, sig, cond.float(), pooled.float(), cfgw, dtype)
    return sr.process_out(x, "flux" if kind == "flux" else "sd3"), model.log


@pytest.mark.parametrize("graphs", ["1", "0"])
@pytest.mark.parametrize("kind", ["flux", "sd3"])
def test_threshold_zero_is_bit_identical_to_off(kc, monkeypatch, kind, graphs):
    monkeypatch.setenv("DK_CUDA_GRAPHS", graphs)
    pipe, _, _, cond, pooled = _pipe(kind)
    assert pipe.mmdit.use_cuda_graphs == (graphs == "1") and pipe.step_cache is None
    off = _denoise(pipe, kind, cond, pooled)
    pipe.set_step_cache(0.0)
    assert pipe.step_cache == (0.0, None)
    on = _denoise(pipe, kind, cond, pooled)
    log = pipe.mmdit.step_cache_log
    assert torch.equal(on, off)
    assert [s for _, s in log] == [False] * CASES[kind][2] and log[0][0] is None
    assert all(r is not None and math.isfinite(r) for r, _ in log[1:])
    pipe.set_step_cache(None)
    assert pipe.step_cache is None and pipe.mmdit.step_cache_log == []
    assert torch.equal(_denoise(pipe, kind, cond, pooled), off)


def _pattern(cap, steps):
    out, run = [], 0
    for i in range(steps):
        skip = i > 0 and (cap is None or run < cap)
        run = run + 1 if skip else 0
        out.append(skip)
    return out


@pytest.mark.parametrize("kind", ["flux", "sd3", "sd35"])
def test_fixed_patterns_match_the_oracle(kc, kind):
    """threshold inf: every forward after the first skips up to the cap, so the pattern is known in advance"""
    from tests.model_checks import rel_l2

    pipe, cfg, p, cond, pooled = _pipe(kind)
    steps = CASES[kind][2]
    for cap in (None, 1, 2):
        pipe.set_step_cache(math.inf, cap)
        got = _denoise(pipe, kind, cond, pooled)
        skips = [s for _, s in pipe.mmdit.step_cache_log]
        assert skips == _pattern(cap, steps), (cap, skips)
        want, _ = _oracle(kind, cfg, p, cond, pooled, skips)
        r = rel_l2(got, want)
        print(f"{kind} cap={cap} pattern={''.join('S' if s else 'F' for s in skips)} final latent rel_l2={r:.3e}")
        assert r <= 5e-2, f"{kind} cap={cap} final latent rel_l2 {r:.3e}"


# Engine rel (16-bit activations) against the oracle's (fp32) along the same decisions: measured at most 1.2e-3 (FLUX)
# and 2.6e-4 (SD3 with CFG) on an H100, DESIGN.md §10; the bound is four times the larger.
REL_BOUND = 5e-3


@pytest.mark.parametrize("kind", ["flux", "sd3"])
def test_intermediate_threshold_against_the_oracle(kc, kind):
    from tests.model_checks import rel_l2

    pipe, cfg, p, cond, pooled = _pipe(kind)
    pipe.set_step_cache(0.0)
    _denoise(pipe, kind, cond, pooled)
    # just above the second step's change, which is the same whatever the threshold: that step skips, and the steps
    # after it, measured against the first step's residual, fall on either side
    threshold = 1.05 * pipe.mmdit.step_cache_log[1][0]
    pipe.set_step_cache(threshold)
    got = _denoise(pipe, kind, cond, pooled)
    log = pipe.mmdit.step_cache_log
    want, olog = _oracle(kind, cfg, p, cond, pooled, [s for _, s in log])
    diffs = [abs(e - o) for (e, _), (o, _) in zip(log[1:], olog[1:])]
    print(f"{kind} threshold={threshold:.4f} engine rel={[round(r, 4) for r, _ in log[1:]]} "
          f"oracle rel={[round(r, 4) for r, _ in olog[1:]]} max |diff|={max(diffs):.2e} "
          f"final latent rel_l2={rel_l2(got, want):.3e}")
    assert any(s for _, s in log) and not all(s for _, s in log[1:]), "the threshold did not split the steps"
    assert max(diffs) <= REL_BOUND
    for (_, skip), (orel, _) in zip(log[1:], olog[1:]):
        if abs(orel - threshold) > REL_BOUND:
            assert skip == (orel < threshold)
    assert rel_l2(got, want) <= 5e-2


def test_graphs_and_eager_agree_with_the_cache_on(kc):
    pipe, _, _, cond, pooled = _pipe("sd3")
    pipe.set_step_cache(math.inf, 1)
    graphed = _denoise(pipe, "sd3", cond, pooled)
    state = next(iter(pipe.mmdit._shapes._states.values()))
    assert {"graph.head", "graph.tail", "graph.skip", "sc"} <= set(state) and "graph" not in state
    pipe.mmdit.use_cuda_graphs = False
    assert torch.equal(_denoise(pipe, "sd3", cond, pooled), graphed)
    pipe.mmdit.use_cuda_graphs = True
    assert torch.equal(_denoise(pipe, "sd3", cond, pooled), graphed)     # replay
    pipe.mmdit._shapes.drop_graphs()
    assert not any(k.startswith("graph") for k in state) and "sc" in state
    pipe.set_step_cache(None)
    assert "sc" not in state


def test_resets(kc):
    """every trigger makes the next forward a full one"""
    from diffusionkit_b200.config import tiny_flux_config
    from diffusionkit_b200.lora import LoRA

    pipe, cfg, _, cond, pooled = _pipe("flux")
    m = pipe.mmdit
    h = cfg.hidden_size
    lora = LoRA("a", {"multimodal_transformer_blocks.1.image_transformer_block.attn.q_proj.weight":
                      (torch.randn((h, 4)) * 0.2, torch.randn((4, h)) * 0.2)})
    g = torch.Generator().manual_seed(2)
    latent = torch.randn((2, 8, 12, 16), generator=g).to(bf16).to(DEV)
    text = cond.to(DEV)
    m.set_step_cache(math.inf)

    def fwd(lat=latent, txt=text):
        m(lat, txt, timestep=752.0)
        return m.step_cache_log[-1][1]

    def restarts(trigger):
        m.cache_modulation_params(pooled.to(DEV), [752.0])
        fwd(), fwd()
        assert [s for _, s in m.step_cache_log] == [False, True]
        trigger()
        assert fwd() is False and len(m.step_cache_log) == 1
        assert fwd() is True

    restarts(lambda: m.cache_modulation_params(pooled.to(DEV), [752.0]))
    restarts(lambda: m.apply_lora([(lora, 1.0)]))
    restarts(lambda: m.apply_lora([(lora, 0.5)]))                        # a scale change keeps the graphs
    restarts(lambda: m.set_fp8(True))
    restarts(lambda: m.set_fp8(False))
    restarts(lambda: m.set_step_cache(math.inf))
    # a new shape: the first forward at it runs in full, and so does the first one back
    m.cache_modulation_params(pooled.to(DEV), [752.0])
    fwd(), fwd()
    assert fwd(lat=latent[:, :6]) is False and fwd(lat=latent[:, :6]) is True
    assert fwd() is False
    # a new batch (the modulation cache is rebuilt for it, which resets too; the shape key changes as well)
    m.cache_modulation_params(pooled[:1].to(DEV), [752.0])
    assert fwd(lat=latent[:1], txt=text[:1]) is False and fwd(lat=latent[:1], txt=text[:1]) is True
    assert tiny_flux_config().depth_multimodal >= 1


def test_generate_image_logs_and_restarts(kc):
    pipe, _, _, cond, pooled = _pipe("flux", decoder=True)
    steps = CASES["flux"][2]
    kw = dict(num_steps=steps, latent_size=LAT, seed=SEEDS[0], verbose=False, conditioning=cond[[0]],
              pooled_conditioning=pooled[[0]])
    _, log = pipe.generate_image("", **kw)
    assert "step_cache" not in log["denoising"]
    pipe.set_step_cache(math.inf, 2)
    for _ in range(2):
        _, log = pipe.generate_image("", **kw)
        sc = log["denoising"]["step_cache"]
        assert [e["skipped"] for e in sc] == _pattern(2, steps) and sc[0]["rel"] is None
        assert all(isinstance(e["rel"], float) for e in sc[1:])


def test_fp8_with_the_cache(kc):
    """FP8 composes with the cache: threshold 0 changes nothing, and a skipping run stays within the FP8 pipeline
    bound of DESIGN.md §9 against the same run in 16 bits"""
    from tests.model_checks import psnr, rel_l2

    pipe, _, _, cond, pooled = _pipe("flux", decoder=True)
    pipe.set_fp8(True)
    plain8 = _denoise(pipe, "flux", cond, pooled)
    pipe.set_step_cache(0.0)
    assert torch.equal(_denoise(pipe, "flux", cond, pooled), plain8)
    pipe.set_step_cache(math.inf, 1)
    cached8 = _denoise(pipe, "flux", cond, pooled)
    assert [s for _, s in pipe.mmdit.step_cache_log] == _pattern(1, CASES["flux"][2])
    pipe.set_fp8(False)
    cached16 = _denoise(pipe, "flux", cond, pooled)
    img8, img16 = pipe.decode_latents_to_image(cached8), pipe.decode_latents_to_image(cached16)
    ps = psnr(img16, img8)
    print(f"fp8 + cache vs 16-bit + cache: latent rel_l2={rel_l2(cached8, cached16):.3e} decoded RGB psnr={ps:.1f}")
    assert bool(torch.isfinite(cached8).all()) and ps >= 20.0
    assert not np.array_equal(cached8.cpu().numpy(), cached16.cpu().numpy())
