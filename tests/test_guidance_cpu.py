"""CPU: FLUX.1-dev's guidance embedder — parameter specs, checkpoint loader, LoRA parser, the oracle's properties
(tests/guidance_ref.py), the resolution-dependent schedule shift and the argument checks that run before GPU work."""
import inspect
import math
from dataclasses import replace

import numpy as np
import pytest
import torch

from diffusionkit_b200 import model_io
from diffusionkit_b200.config import FLUX_DEV, FLUX_SCHNELL, tiny_flux_config, tiny_sd3_config
from diffusionkit_b200.lora import load_lora, module_table
from diffusionkit_b200.mmdit import MMDiT
from diffusionkit_b200.pipeline import DEFAULT_GUIDANCE, DiffusionPipeline, FluxPipeline
from diffusionkit_b200.sampler import FluxSampler, flux_resolution_shift
from diffusionkit_b200.weights import init_params, mmdit_param_specs
from oracle.mmdit_ref import MMDiTRef
from tests.guidance_ref import GuidanceMMDiTRef, guidance_input, guidance_sinusoid
from tests.lora_fixtures import kohya_dict, make_factors, peft_dict, upstream_delta
from tests.oracle_bridge import ref_config
from tests.test_model_io_cpu import _flux_upstream

bf16 = torch.bfloat16
GUIDANCE_SPECS = ["guidance_in.mlp.layers.0.weight", "guidance_in.mlp.layers.0.bias",
                  "guidance_in.mlp.layers.2.weight", "guidance_in.mlp.layers.2.bias"]


def tiny_dev_config():
    return replace(tiny_flux_config(), guidance_embed=True)


def dev_upstream(params, cfg):
    """engine tree with a guidance embedder -> BFL FLUX.1-dev key layout"""
    sd = _flux_upstream(params, cfg)
    for layer, idx in (("in_layer", 0), ("out_layer", 2)):
        for leaf in ("weight", "bias"):
            sd[f"guidance_in.{layer}.{leaf}"] = params[f"guidance_in.mlp.layers.{idx}.{leaf}"]
    return sd


# ------------------------------------------------------------------------------------------------ parameters
@pytest.mark.parametrize("dev, schnell", [(FLUX_DEV, FLUX_SCHNELL), (tiny_dev_config(), tiny_flux_config())])
def test_specs_append_the_embedder(dev, schnell):
    s, d = mmdit_param_specs(schnell), mmdit_param_specs(dev)
    assert d[:len(s)] == s
    h, f = dev.hidden_size, dev.frequency_embed_dim
    assert d[len(s):] == [(GUIDANCE_SPECS[0], (h, f), "w"), (GUIDANCE_SPECS[1], (h,), "b"),
                          (GUIDANCE_SPECS[2], (h, h), "w"), (GUIDANCE_SPECS[3], (h,), "b")]


def test_init_params_shares_every_other_weight():
    s = init_params(mmdit_param_specs(tiny_flux_config()), seed=7, dtype=torch.float32)
    d = init_params(mmdit_param_specs(tiny_dev_config()), seed=7, dtype=torch.float32)
    assert set(d) == set(s) | set(GUIDANCE_SPECS)
    for name, t in s.items():
        assert torch.equal(d[name], t), name


def test_guidance_embed_needs_a_flux_shaped_config():
    cfg = replace(tiny_sd3_config(), guidance_embed=True)
    params = init_params(mmdit_param_specs(replace(cfg, guidance_embed=False)), seed=0, dtype=torch.float16)
    with pytest.raises(ValueError, match="FLUX-shaped"):
        MMDiT(cfg, params)


# ------------------------------------------------------------------------------------------------ checkpoint
def test_checkpoint_loader_maps_the_embedder():
    cfg = tiny_dev_config()
    params = init_params(mmdit_param_specs(cfg), seed=3, dtype=torch.float32)
    sd = dev_upstream(params, cfg)
    got = model_io.flux_checkpoint_to_params(sd, cfg.hidden_size, cfg.mlp_ratio, guidance_embed=True)
    model_io.check_against_specs(got, mmdit_param_specs(cfg))
    for name in GUIDANCE_SPECS:
        assert torch.equal(got[name], params[name]), name
    # flag off: dropped, as before (quirk Q1)
    off = model_io.flux_checkpoint_to_params(sd, cfg.hidden_size, cfg.mlp_ratio)
    assert not any(k.startswith("guidance_in") for k in off)
    model_io.check_against_specs(off, mmdit_param_specs(tiny_flux_config()))


@pytest.mark.parametrize("missing", ["guidance_in.out_layer.bias", "guidance_in.in_layer.weight"])
def test_checkpoint_loader_names_a_missing_key(missing):
    cfg = tiny_dev_config()
    sd = dev_upstream(init_params(mmdit_param_specs(cfg), seed=3, dtype=torch.float32), cfg)
    del sd[missing]
    with pytest.raises(ValueError, match=missing.replace(".", r"\.")):
        model_io.flux_checkpoint_to_params(sd, cfg.hidden_size, cfg.mlp_ratio, guidance_embed=True)
    sd["guidance_in.mystery.weight"] = torch.zeros(2)
    with pytest.raises(KeyError, match="guidance_in.mystery"):
        model_io.flux_checkpoint_to_params(sd, cfg.hidden_size, cfg.mlp_ratio, guidance_embed=True)


# ------------------------------------------------------------------------------------------------ LoRA
def test_lora_guidance_keys_are_targets_with_the_embedder():
    cfg = tiny_dev_config()
    h, f = cfg.hidden_size, cfg.frequency_embed_dim
    assert set(module_table(cfg)) == set(module_table(tiny_flux_config())) | {"guidance_in.in_layer",
                                                                              "guidance_in.out_layer"}
    factors = make_factors({"guidance_in.in_layer": (h, f), "guidance_in.out_layer": (h, h)}, rank=3, seed=5)
    want = upstream_delta(factors)
    names = {"guidance_in.in_layer.weight": "guidance_in.mlp.layers.0.weight",
             "guidance_in.out_layer.weight": "guidance_in.mlp.layers.2.weight"}
    kohya = load_lora(kohya_dict(factors), cfg)
    assert kohya.skipped == [] and set(kohya.targets) == set(names.values())
    for up_name, name in names.items():
        up, down = kohya.targets[name]
        torch.testing.assert_close(up @ down, want[up_name], rtol=1e-5, atol=1e-6)
    for prefix in ("", "diffusion_model."):
        peft = load_lora(peft_dict(factors, prefix), cfg)
        assert peft.skipped == [] and set(peft.targets) == set(kohya.targets)
        for name, (up, down) in kohya.targets.items():
            assert torch.equal(peft.targets[name][0], up) and torch.equal(peft.targets[name][1], down)
    # the same adapter on a model without the embedder: skipped and reported, as before
    plain = load_lora(peft_dict(factors, "diffusion_model."), tiny_flux_config())
    assert plain.targets == {} and len(plain.skipped) == 6


# ------------------------------------------------------------------------------------------------ oracle
def _oracle_case(cfg, params, B=2, T=8, lat=(4, 6), seed=1):
    g = torch.Generator().manual_seed(seed)
    latent = torch.randn((B, lat[0], lat[1], 16), generator=g)
    text = torch.randn((B, T, cfg.token_level_text_embed_dim), generator=g)
    pooled = torch.randn((B, cfg.pooled_text_embed_dim), generator=g)
    return latent, text, pooled, torch.tensor([752.0, 500.0])


def test_oracle_zero_embedder_is_the_plain_oracle():
    cfg = tiny_dev_config()
    p = init_params(mmdit_param_specs(cfg), seed=7, dtype=torch.float32)
    p["guidance_in.mlp.layers.2.weight"].zero_()
    p["guidance_in.mlp.layers.2.bias"].zero_()
    latent, text, pooled, ts = _oracle_case(cfg, p)
    plain, dev = MMDiTRef(ref_config(cfg), p), GuidanceMMDiTRef(ref_config(cfg), p)
    plain.cache_modulation_params(pooled, ts)
    dev.cache_modulation_params(pooled, ts, [3.5, 5.0])
    for t in ts:
        tt = t.reshape(1).repeat(2)
        assert torch.equal(dev(latent, text, tt), plain(latent, text, tt))
    # and a non-zero embedder changes it
    p2 = init_params(mmdit_param_specs(cfg), seed=7, dtype=torch.float32)
    live = GuidanceMMDiTRef(ref_config(cfg), p2)
    live.cache_modulation_params(pooled, ts, [3.5, 5.0])
    tt = ts[:1].repeat(2)
    assert not torch.equal(live(latent, text, tt), plain(latent, text, tt))


def test_oracle_guidance_vector_is_the_formula():
    """W2 · SiLU(W0 · sinusoid(v) + b0) + b2 in numpy fp64, the sinusoid from v = 3504 and 4992 with fp64 angles"""
    cfg = tiny_dev_config()
    p = init_params(mmdit_param_specs(cfg), seed=7, dtype=torch.float32)
    ref = GuidanceMMDiTRef(ref_config(cfg), p)
    got = ref.guidance_vector([3.5, 5.0]).numpy()
    v = np.array([3504.0, 4992.0])
    k = np.arange(128, dtype=np.float64)
    ang = v[:, None] * np.exp(-np.log(10000.0) * k / 128)[None, :]
    s = np.concatenate([np.cos(ang), np.sin(ang)], axis=1)
    s_or = guidance_sinusoid(guidance_input([3.5, 5.0], bf16), 256, 10000, bf16).numpy()
    # fp32 angles near 5000 are off by up to ~5e-4 rad; bf16 rounding of a value <= 1 by up to 2^-9
    assert np.abs(s_or - s).max() <= 3e-3
    w0, b0, w2, b2 = [p[n].double().numpy() for n in GUIDANCE_SPECS]
    z = s @ w0.T + b0
    want = (z / (1.0 + np.exp(-z))) @ w2.T + b2
    err = np.linalg.norm(got - want) / np.linalg.norm(want)
    assert err <= 1e-2, err
    # against the oracle's own (rounded) sinusoid the MLP agrees to fp32 accuracy
    z = s_or.astype(np.float64) @ w0.T + b0
    exact = (z / (1.0 + np.exp(-z))) @ w2.T + b2
    assert np.abs(got - exact).max() <= 1e-5 * np.abs(exact).max()


def test_guidance_input_rounding():
    v = guidance_input([3.5, 1.0, 4.0, 5.0, 3.3], bf16)
    # bf16 steps are 16 wide in [2048, 4096) and 32 wide in [4096, 8192): 3500 -> 3504, 5000 -> 4992
    assert v.tolist()[:4] == [3504.0, 1000.0, 4000.0, 4992.0]
    assert v.tolist()[4] == float(torch.tensor(float(torch.tensor(3.3).to(bf16)) * 1000).to(bf16))


def test_product_sinusoid_equals_the_oracle():
    m = object.__new__(MMDiT)
    m.config, m.dtype = FLUX_DEV, bf16
    g = [0.0, 1.0, 3.5, 5.0, 10.0, 2.7]
    got = m.guidance_embedding(g)
    assert got.dtype == bf16 and got.shape == (6, 256)
    assert torch.equal(got.float(), guidance_sinusoid(guidance_input(g, bf16), 256, 10000, bf16))


# ------------------------------------------------------------------------------------------------ schedule shift
@pytest.mark.parametrize("size, mu", [((32, 32), 0.5), ((64, 64), 0.63), ((128, 128), 1.15)])
def test_flux_resolution_shift_values(size, mu):
    assert flux_resolution_shift(size) == pytest.approx(math.exp(mu), rel=1e-12)


def test_flux_resolution_shift_at_1024():
    assert round(flux_resolution_shift((128, 128)), 4) == 3.1582
    assert flux_resolution_shift((64, 64), base_shift=0.0, max_shift=0.0) == 1.0
    with pytest.raises(ValueError):
        flux_resolution_shift((0, 64))


@pytest.mark.parametrize("n", [4, 28, 50])
@pytest.mark.parametrize("size", [(32, 32), (64, 64), (128, 128), (96, 160)])
def test_get_sigmas_with_the_shift_is_bfl_time_shift(n, size):
    shift = flux_resolution_shift(size)
    sig = object.__new__(FluxPipeline).get_sigmas(FluxSampler(shift=shift), n)
    t = np.linspace(1.0, 0.0, n + 1)
    with np.errstate(divide="ignore"):
        want = np.where(t > 0, shift / (shift + 1.0 / t - 1.0), 0.0)
    assert len(sig) == n + 1
    assert np.abs(sig.astype(np.float64) - want).max() <= 1e-6


# ------------------------------------------------------------------------------------------------ arguments
def _pipe_shell(cfg):
    """a pipeline object with only its config: enough for the checks that run before any GPU work"""
    p = object.__new__(FluxPipeline)
    p.config = cfg
    return p


def test_guidance_values():
    dev = _pipe_shell(tiny_dev_config())
    assert dev._guidance_values(None, 2) == [DEFAULT_GUIDANCE] * 2 == [3.5, 3.5]
    assert dev._guidance_values(4, 3) == [4.0, 4.0, 4.0]
    assert dev._guidance_values(np.float32(2.5), 1) == [2.5]
    assert dev._guidance_values([1.0, 5.0], 2) == [1.0, 5.0]
    assert dev._guidance_values(torch.tensor([1.0, 5.0]), 2) == [1.0, 5.0]
    for bad, n in (([1.0], 2), ([1.0, 2.0, 3.0], 2), (float("nan"), 1), ([1.0, float("inf")], 2)):
        with pytest.raises(ValueError):
            dev._guidance_values(bad, n)
    schnell = _pipe_shell(tiny_flux_config())
    assert schnell._guidance_values(None, 2) is None
    with pytest.raises(ValueError, match="no guidance embedder"):
        schnell._guidance_values(3.5, 1)


def test_public_methods_check_guidance_first():
    """the checks run before anything touches the models or the device (the shell has neither)"""
    dev, schnell = _pipe_shell(tiny_dev_config()), _pipe_shell(tiny_flux_config())
    cond, pooled = torch.zeros(2, 4, 8), torch.zeros(2, 8)
    with pytest.raises(ValueError):
        dev.denoise_latents(cond, pooled, seed=[1, 2], guidance=[3.5])
    with pytest.raises(ValueError):
        dev.generate_image("", seed=[1, 2], guidance=[3.5, float("nan")], conditioning=cond, pooled_conditioning=pooled)
    with pytest.raises(ValueError):
        schnell.denoise_latents(cond, pooled, seed=1, guidance=3.5)
    with pytest.raises(ValueError):
        schnell.generate_image("", seed=1, guidance=3.5, conditioning=cond, pooled_conditioning=pooled)


def test_mmdit_checks_guidance_first():
    m = object.__new__(MMDiT)
    m.config = tiny_dev_config()
    pooled = torch.zeros(3, 64)
    with pytest.raises(ValueError, match="guidance embedder"):
        m.cache_modulation_params(pooled, [1000.0])
    with pytest.raises(ValueError, match="3 conditioning rows"):
        m.cache_modulation_params(pooled, [1000.0], [3.5, 3.5])
    with pytest.raises(ValueError, match="finite"):
        m.cache_modulation_params(pooled, [1000.0], [3.5, float("nan"), 1.0])
    m.config = tiny_flux_config()
    with pytest.raises(ValueError, match="no guidance embedder"):
        m.cache_modulation_params(pooled, [1000.0], [3.5] * 3)


def test_only_flux_takes_guidance():
    for name in ("denoise_latents", "generate_image"):
        assert "guidance" in inspect.signature(getattr(FluxPipeline, name)).parameters
        assert "guidance" not in inspect.signature(getattr(DiffusionPipeline, name)).parameters
        assert inspect.signature(getattr(FluxPipeline, name)).parameters["guidance"].kind == inspect.Parameter.KEYWORD_ONLY
