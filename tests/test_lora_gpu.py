"""-m gpu: LoRA adapters merged into the packed MMDiT weights with the wgmma GEMM.

A stack of two adapters (ranks 4 and 12, so the concatenated rank needs padding on the modules only one of them
covers; scales 0.7 and -1.3) on tiny FLUX (bf16) and tiny SD3 (fp16): merge precision, forward and pipeline against
the fp32 oracle on merged parameters, exact restoration, no drift, and CUDA-graph replay after a scale change."""
from dataclasses import replace

import numpy as np
import pytest
import torch

import diffusionkit_b200 as dk
from diffusionkit_b200 import ops
from diffusionkit_b200.config import FLUX_SCHNELL, VAEDecoderConfig, tiny_flux_config, tiny_sd3_config
from diffusionkit_b200.lora import load_lora
from diffusionkit_b200.mmdit import MMDiT
from diffusionkit_b200.weights import init_params, mmdit_param_specs, vae_decoder_param_specs
from oracle import sampler_ref as sr
from oracle.mmdit_ref import MMDiTRef
from tests.lora_fixtures import kohya_dict, make_factors, merge_lora, peft_dict, upstream_modules
from tests.model_checks import psnr, rel_l2
from tests.oracle_bridge import ref_config

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASES = {"flux": (tiny_flux_config, torch.bfloat16), "sd3": (tiny_sd3_config, torch.float16)}
PREFIX = {"flux": "diffusion_model.", "sd3": "model.diffusion_model."}
SCALES = (0.7, -1.3)


def _adapter_dicts(kind, cfg):
    """kohya rank-4 and PEFT rank-12 state dicts; upstream module i: i % 3 == 0 only in the first, == 2 only in the
    second, == 1 in both, and i % 7 == 3 in neither"""
    mods = sorted(upstream_modules(cfg).items())
    a = {m: s for i, (m, s) in enumerate(mods) if i % 3 != 2 and i % 7 != 3}
    b = {m: s for i, (m, s) in enumerate(mods) if i % 3 != 0 and i % 7 != 3}
    return kohya_dict(make_factors(a, 4, seed=11)), peft_dict(make_factors(b, 12, seed=12), PREFIX[kind])


def _adapters(kind, cfg):
    da, db = _adapter_dicts(kind, cfg)
    return load_lora(da, cfg, name="a"), load_lora(db, cfg, name="b")


def _weights(m):
    """every weight a LoRA can touch, as the forward currently sees it"""
    return {n: MMDiT._bound(o, a, i)[r, c].clone() for n, (o, a, i, r, c) in m.lora_weight_slots().items()}


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def _ulp(x, dtype):
    """spacing of `dtype` at |x| (x fp64)"""
    mant, tiny = (7, 2.0 ** -133) if dtype == torch.bfloat16 else (10, 2.0 ** -24)
    _, e = torch.frexp(x)
    u = torch.ldexp(torch.ones_like(x), (e - 1 - mant).to(torch.int32))
    return torch.where(x == 0, torch.full_like(x, tiny), u.clamp(min=tiny))


def _check_merged(got, base, terms, dtype):
    """got within 1 ulp of the fp64 value want = base + Σ round16(s·up) @ round16(down), plus the error bound of the
    GEMM's fp32 sum (K + 1 terms, K = padded rank).  That term only matters where base and ΔW cancel, so that |want|
    is far below |base|: the 16-bit ulp of the result is then smaller than the fp32 rounding of the operands."""
    dev = got.device
    base64 = base.to(dev, torch.float64)
    want, mag, k = base64.clone(), base64.abs(), 0
    for s, up, down in terms:
        u, d = (s * up).to(dtype).to(dev, torch.float64), down.to(dtype).to(dev, torch.float64)
        want += u @ d
        mag += u.abs() @ d.abs()
        k += up.shape[1]
    want, mag = want.reshape(got.shape), mag.reshape(got.shape)
    err = (got.to(torch.float64) - want).abs()
    ulp = _ulp(want, dtype)
    assert bool((err <= ulp + (-(-k // 8) * 8 + 1) * 2.0 ** -23 * mag).all()), "merged weight off by more than the bound"
    over = int((err > ulp).sum())
    assert over <= 1e-5 * err.numel(), f"{over} of {err.numel()} elements are more than 1 ulp off"


def _inputs(cfg, dtype, B=2, lat=(8, 12), T=16):
    gen = torch.Generator().manual_seed(5)
    latent = torch.randn((B, lat[0], lat[1], 16), generator=gen).to(dtype)
    text = torch.randn((B, T, cfg.token_level_text_embed_dim), generator=gen).to(dtype)
    pooled = torch.randn((B, cfg.pooled_text_embed_dim), generator=gen).to(dtype)
    return latent, text, pooled


@pytest.mark.parametrize("kind", ["flux", "sd3"])
def test_merge_within_one_ulp(cuda, kind):
    make_cfg, dt = CASES[kind]
    cfg = make_cfg()
    params = init_params(mmdit_param_specs(cfg), seed=7, dtype=dt, device=DEV)
    caller = {k: v.clone() for k, v in params.items()}
    m = dk.MMDiT(cfg, params)
    before = _weights(m)
    la, lb = _adapters(kind, cfg)
    m.apply_lora([(la, SCALES[0]), (lb, SCALES[1])])
    after = _weights(m)
    touched = set(la.targets) | set(lb.targets)
    assert touched < set(before) and set(la.targets) & set(lb.targets)
    for name, w in after.items():
        if name in touched:
            terms = [(s, *l.targets[name]) for l, s in zip((la, lb), SCALES) if name in l.targets]
            _check_merged(w, before[name], terms, dt)
        else:
            assert _same_bits(w, before[name]), f"untouched weight {name} changed"
    for k, v in params.items():
        assert _same_bits(v, caller[k]), f"caller's tensor {k} was written"


@pytest.mark.parametrize("kind", ["flux", "sd3"])
def test_forward_matches_oracle_on_merged_params(cuda, kind):
    make_cfg, dt = CASES[kind]
    cfg = make_cfg()
    p16 = {k: v.to(dt) for k, v in init_params(mmdit_param_specs(cfg), seed=7, dtype=torch.float32).items()}
    la, lb = _adapters(kind, cfg)
    merged = merge_lora(p16, [(la.targets, SCALES[0]), (lb.targets, SCALES[1])])
    latent, text, pooled = _inputs(cfg, dt)
    t = torch.tensor([752.0])
    outs = []
    for p in ({k: v.float() for k, v in p16.items()}, merged):
        ref = MMDiTRef(ref_config(cfg), p)
        ref.cache_modulation_params(pooled.float(), t)
        outs.append(ref(latent.float(), text.float(), t.repeat(latent.shape[0])))
    plain, want = outs
    m = dk.MMDiT(cfg, {k: v.to(DEV) for k, v in p16.items()})
    m.apply_lora([(la, SCALES[0]), (lb, SCALES[1])])
    m.cache_modulation_params(pooled.to(DEV), [752.0])
    got = m(latent.to(DEV), text.to(DEV), timestep=752.0)
    torch.cuda.synchronize()
    r, ps, effect = rel_l2(got, want), psnr(want, got), rel_l2(plain, want)
    assert r <= 2e-2 and ps >= 35.0, f"rel_l2 {r:.3e} psnr {ps:.1f}"
    assert effect >= 10 * r, f"adapter effect {effect:.3e} is not 10x the error {r:.3e}"


@pytest.mark.parametrize("kind", ["flux", "sd3"])
def test_scale_zero_unload_and_no_drift(cuda, kind):
    """through the pipeline API: scale 0 and unload restore the never-adapted weights and graph-replayed forward bit
    for bit; twenty alternating scale changes end on the bits of one application"""
    make_cfg, dt = CASES[kind]
    cfg = make_cfg()
    Pipe = dk.FluxPipeline if kind == "flux" else dk.DiffusionPipeline
    pipe = Pipe(w16=True, a16=True, mmdit_config=cfg, load_decoder=False,
                params=init_params(mmdit_param_specs(cfg), seed=7, dtype=dt, device=DEV))
    m = pipe.mmdit
    m.use_cuda_graphs = True
    latent, text, pooled = [t.to(DEV) for t in _inputs(cfg, dt)]

    def forward():
        m.cache_modulation_params(pooled, [752.0])
        return m(latent, text, timestep=752.0).clone()

    out0, w0 = forward(), _weights(m)
    da, db = _adapter_dicts(kind, cfg)
    assert pipe.load_lora_weights(da, scale=SCALES[0], adapter_name="a") == "a"
    pipe.load_lora_weights(db, scale=SCALES[1], adapter_name="b")
    assert pipe.lora_adapters == {"a": SCALES[0], "b": SCALES[1]}
    w1, out1 = _weights(m), forward()
    assert not torch.equal(out1, out0)

    pipe.set_lora_scale("a", 0.0)
    pipe.set_lora_scale("b", 0.0)
    assert all(_same_bits(w, w0[n]) for n, w in _weights(m).items())
    assert torch.equal(forward(), out0)

    for i in range(20):
        name = "a" if i % 2 == 0 else "b"
        pipe.set_lora_scale(name, SCALES[0 if name == "a" else 1] if i >= 18 else 2.0 - 0.1 * i)
    assert pipe.lora_adapters == {"a": SCALES[0], "b": SCALES[1]}
    assert all(_same_bits(w, w1[n]) for n, w in _weights(m).items())
    assert torch.equal(forward(), out1)

    pipe.unload_lora_weights("a")
    assert pipe.lora_adapters == {"b": SCALES[1]}
    pipe.unload_lora_weights()
    assert pipe.lora_adapters == {} and not m._lora_live
    assert all(_same_bits(w, w0[n]) for n, w in _weights(m).items())
    assert torch.equal(forward(), out0)
    with pytest.raises(KeyError):
        pipe.set_lora_scale("a", 1.0)


@pytest.mark.parametrize("kind", ["flux", "sd3"])
def test_scale_change_replays_the_captured_graph(cuda, kind):
    make_cfg, dt = CASES[kind]
    cfg = make_cfg()
    m = dk.MMDiT(cfg, init_params(mmdit_param_specs(cfg), seed=7, dtype=dt, device=DEV))
    m.use_cuda_graphs = True
    latent, text, pooled = [t.to(DEV) for t in _inputs(cfg, dt)]
    la, lb = _adapters(kind, cfg)
    m.apply_lora([(la, SCALES[0]), (lb, SCALES[1])])
    m.cache_modulation_params(pooled, [752.0])
    first = m(latent, text, timestep=752.0).clone()
    (state,) = m._shapes._states.values()
    graph = state["graph"]

    m.apply_lora([(la, 1.5), (lb, 0.4)])
    m.cache_modulation_params(pooled, [752.0])
    n0 = ops.launch_count()
    replayed = m(latent, text, timestep=752.0).clone()
    n1 = ops.launch_count()
    assert state["graph"] is graph, "a scale change recaptured the graph"
    assert n1 - n0 == graph[3] > 0, f"{n1 - n0} launches counted, the graph replays {graph[3]}"
    m.use_cuda_graphs = False
    eager = m(latent, text, timestep=752.0)
    torch.cuda.synchronize()
    assert torch.equal(replayed, eager)
    assert not torch.equal(replayed, first)


def _oracle_latent(kind, cfg, params, cond, pooled, steps, cfgw, shift, H, W, seed, dtype):
    sampler = sr.FluxSamplerRef(shift) if kind == "flux" else sr.ModelSamplingDiscreteFlowRef(shift)
    sig = sr.get_sigmas(sampler, steps)
    ref = MMDiTRef(ref_config(cfg), params)
    x0 = sampler.noise_scaling(float(sig[0]), sr.get_noise(seed, H, W), sr.get_empty_latent(H, W))
    x = sr.sample_euler(lambda xin, c, t: ref(xin, c, t), ref.cache_modulation_params, x0, sig, cond.float(),
                        pooled.float(), cfgw, dtype)
    return sr.process_out(x, kind)


@pytest.mark.parametrize("kind", ["flux", "sd3"])
def test_pipeline_with_adapter_file(cuda, kind, tmp_path):
    """FLUX: a kohya file, 4 steps; SD3: a PEFT file, CFG 5.0, 6 steps; the other adapter of the stack as a dict"""
    from safetensors.torch import save_file

    make_cfg, dt = CASES[kind]
    cfg = make_cfg()
    if kind == "flux":
        Pipe, steps, cfgw, shift, T = dk.FluxPipeline, 4, 0.0, 1.0, 16
    else:
        Pipe, steps, cfgw, shift, T = dk.DiffusionPipeline, 6, 5.0, 3.0, 24
    p16 = {k: v.to(dt) for k, v in init_params(mmdit_param_specs(cfg), seed=7, dtype=torch.float32).items()}
    vp16 = {k: v.to(dt) for k, v in init_params(vae_decoder_param_specs(VAEDecoderConfig()), seed=8,
                                                 dtype=torch.float32).items()}
    pipe = Pipe(w16=True, a16=True, shift=shift, mmdit_config=cfg, params={k: v.to(DEV) for k, v in p16.items()},
                vae_params={k: v.to(DEV) for k, v in vp16.items()})
    cond, pooled = pipe.synthetic_text_embeddings(n_images=1, text_len=T)
    H, W, seed = 8, 12, 11
    kw = dict(num_steps=steps, cfg_weight=cfgw, latent_size=(H, W), seed=seed, verbose=False, conditioning=cond,
              pooled_conditioning=pooled)
    image0, _ = pipe.generate_image("", **kw)

    da, db = _adapter_dicts(kind, cfg)
    file_sd, other = (da, db) if kind == "flux" else (db, da)
    path = tmp_path / f"{kind}_style.safetensors"
    save_file({k: v.contiguous() for k, v in file_sd.items()}, str(path))
    assert pipe.load_lora_weights(path, scale=SCALES[0]) == f"{kind}_style"
    pipe.load_lora_weights(other, scale=SCALES[1], adapter_name="other")
    latent, _ = pipe.denoise_latents(cond, pooled, num_steps=steps, cfg_weight=cfgw, latent_size=(H, W), seed=seed)

    lf, lo = load_lora(file_sd, cfg), load_lora(other, cfg)
    base = {k: v.float() for k, v in p16.items()}
    merged = merge_lora(base, [(lf.targets, SCALES[0]), (lo.targets, SCALES[1])])
    want = _oracle_latent(kind, cfg, merged, cond, pooled, steps, cfgw, shift, H, W, seed, dt)
    plain = _oracle_latent(kind, cfg, base, cond, pooled, steps, cfgw, shift, H, W, seed, dt)
    r = rel_l2(latent, want)
    assert r <= 5e-2, f"{kind} final latent rel_l2 {r:.3e}"
    assert rel_l2(latent, plain) > 5e-2, "the adapted latent is within tolerance of the unadapted oracle"
    image1, _ = pipe.generate_image("", **kw)
    assert not np.array_equal(np.asarray(image1), np.asarray(image0))

    pipe.unload_lora_weights()
    image2, _ = pipe.generate_image("", **kw)
    assert np.array_equal(np.asarray(image2), np.asarray(image0))


def test_full_width_linear2_rank64(cuda):
    """h = 3072: a rank-64 merge into both column windows of the single block's [Wo | W2] weight, [h, 5h]"""
    cfg = replace(FLUX_SCHNELL, depth_multimodal=1, depth_unified=1, hidden_size_override=3072)
    h, dt = cfg.hidden_size, torch.bfloat16
    m = dk.MMDiT(cfg, init_params(mmdit_param_specs(cfg), seed=3, dtype=dt, device=DEV))
    before = _weights(m)
    module = "single_blocks.0.linear2"
    lora = load_lora(peft_dict(make_factors({module: (h, 5 * h)}, 64, seed=13)), cfg)
    m.apply_lora([(lora, SCALES[0])])
    after = _weights(m)
    assert m.single[0].w_out.shape == (h, 5 * h)
    assert set(lora.targets) == {"unified_transformer_blocks.0.transformer_block.attn.o_proj.weight",
                                 "unified_transformer_blocks.0.transformer_block.mlp.fc2.weight"}
    for name, w in after.items():
        if name in lora.targets:
            assert not _same_bits(w, before[name])
            _check_merged(w, before[name], [(SCALES[0], *lora.targets[name])], dt)
        else:
            assert _same_bits(w, before[name]), name
