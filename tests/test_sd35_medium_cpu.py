"""CPU: SD3.5 Medium (MMDiT-X) and skip-layer guidance — the preset, parameter specs, checkpoint loader, LoRA table,
FP8 coverage, config and SLG validation, and the properties that pin the oracle (tests/sd35_medium_ref.py)."""
import inspect
import math
import re
from dataclasses import replace

import numpy as np
import pytest
import torch

from diffusionkit_b200 import model_io
from diffusionkit_b200.config import (MODEL_CONFIGS, SD3_2b, SD3_8b, SD35_MEDIUM, T5_MAX_LENGTH, tiny_flux_config,
                                      tiny_sd3_config, tiny_sd35_config, tiny_sd35_medium_config)
from diffusionkit_b200.lora import load_lora, module_table
from diffusionkit_b200.mmdit import MMDiT, fp8_covered_linears
from diffusionkit_b200.pipeline import MMDIT_CKPT, DiffusionPipeline, FluxPipeline, _check_slg
from diffusionkit_b200.sampler import SkipLayerGuidance, check_skip_layer_guidance, skip_layer_guidance_steps
from diffusionkit_b200.weights import init_params, mmdit_param_specs, param_count
from oracle import sampler_ref as sr
from oracle.mmdit_ref import MMDiTRef
from tests import solver_ref
from tests.lora_fixtures import kohya_dict, make_factors, peft_dict, upstream_delta
from tests.oracle_bridge import ref_config
from tests.sd35_medium_ref import MMDiTXRef, sample, slg_denoiser, slg_window

MEDIUM = "stabilityai/stable-diffusion-3.5-medium"
IMG = "multimodal_transformer_blocks.{}.image_transformer_block"


def xref(cfg, params, act_dtype=None):
    return MMDiTXRef(ref_config(cfg), params, act_dtype, x_layers=cfg.x_block_self_attn_layers,
                     k_bias=cfg.attn_k_bias)


def medium_upstream(params, cfg, prefix="model.diffusion_model.", vae=True):
    """engine tree -> Stability's SD3 / SD3.5 single-file layout (concatenated qkv, attn2, ln_q / ln_k)"""
    h = cfg.hidden_size
    sd = {}
    for i in range(cfg.depth_multimodal):
        for b_up, s_us in (("x_block", "image_transformer_block"), ("context_block", "text_transformer_block")):
            b = f"multimodal_transformer_blocks.{i}.{s_us}"
            u = f"{prefix}joint_blocks.{i}.{b_up}"
            attns = [("attn", "qk_norm")] + ([("attn2", "qk_norm2")] if f"{b}.attn2.q_proj.weight" in params else [])
            for attn, norm in attns:
                sd[f"{u}.{attn}.qkv.weight"] = torch.cat([params[f"{b}.{attn}.{n}_proj.weight"] for n in "qkv"], 0)
                sd[f"{u}.{attn}.qkv.bias"] = torch.cat([params[f"{b}.{attn}.q_proj.bias"],
                                                        params.get(f"{b}.{attn}.k_proj.bias", torch.zeros(h)),
                                                        params[f"{b}.{attn}.v_proj.bias"]])
                if f"{b}.{norm}.q_norm.weight" in params:
                    sd[f"{u}.{attn}.ln_q.weight"] = params[f"{b}.{norm}.q_norm.weight"]
                    sd[f"{u}.{attn}.ln_k.weight"] = params[f"{b}.{norm}.k_norm.weight"]
                if f"{b}.{attn}.o_proj.weight" in params:
                    for leaf in ("weight", "bias"):
                        sd[f"{u}.{attn}.proj.{leaf}"] = params[f"{b}.{attn}.o_proj.{leaf}"]
            for leaf in ("weight", "bias"):
                sd[f"{u}.adaLN_modulation.1.{leaf}"] = params[f"{b}.adaLN_modulation.layers.1.{leaf}"]
                if f"{b}.mlp.fc1.{leaf}" in params:
                    sd[f"{u}.mlp.fc1.{leaf}"] = params[f"{b}.mlp.fc1.{leaf}"]
                    sd[f"{u}.mlp.fc2.{leaf}"] = params[f"{b}.mlp.fc2.{leaf}"]
    sd[prefix + "pos_embed"] = params["x_pos_embedder.pos_embed.weight"][None]
    sd[prefix + "x_embedder.proj.weight"] = params["x_embedder.proj.weight"].permute(0, 3, 1, 2).contiguous()
    sd[prefix + "x_embedder.proj.bias"] = params["x_embedder.proj.bias"]
    for leaf in ("weight", "bias"):
        sd[prefix + f"context_embedder.{leaf}"] = params[f"context_embedder.{leaf}"]
        sd[prefix + f"final_layer.linear.{leaf}"] = params[f"final_layer.linear.{leaf}"]
        sd[prefix + f"final_layer.adaLN_modulation.1.{leaf}"] = params[f"final_layer.adaLN_modulation.layers.1.{leaf}"]
        for emb in ("y_embedder", "t_embedder"):
            for idx in (0, 2):
                sd[prefix + f"{emb}.mlp.{idx}.{leaf}"] = params[f"{emb}.mlp.layers.{idx}.{leaf}"]
    if vae:
        sd["first_stage_model.decoder.conv_in.bias"] = torch.zeros(3)
        sd["first_stage_model.encoder.conv_in.bias"] = torch.zeros(3)
    return sd


# ------------------------------------------------------------------------------------------------ preset, specs
def test_preset():
    c = SD35_MEDIUM
    assert (c.hidden_size, c.num_heads, c.head_dim, c.depth_multimodal, c.depth_unified) == (1536, 24, 64, 24, 0)
    assert c.use_qk_norm and c.attn_k_bias and c.x_block_self_attn_layers == tuple(range(13))
    assert c.max_latent_resolution == 384 and c.dtype == torch.float16
    assert MODEL_CONFIGS[MEDIUM] is SD35_MEDIUM and MMDIT_CKPT[MEDIUM] == MEDIUM and T5_MAX_LENGTH[MEDIUM] == 512
    for old in (SD3_2b, SD3_8b, tiny_sd3_config(), tiny_flux_config()):
        assert old.x_block_self_attn_layers == () and not old.attn_k_bias
    t = tiny_sd35_medium_config()
    assert (t.hidden_size, t.num_heads, t.depth_multimodal, t.x_block_self_attn_layers, t.max_latent_resolution) == (
        128, 2, 3, (0, 1), 24)


def test_specs_append_attn2_and_k_bias():
    cfg = tiny_sd35_medium_config()
    base = mmdit_param_specs(replace(cfg, x_block_self_attn_layers=(), attn_k_bias=False))
    got = mmdit_param_specs(cfg)
    h, d = cfg.hidden_size, cfg.head_dim
    # the existing specs keep their place; only the x-layers' adaLN grows to 9h
    for (n0, s0, k0), (n1, s1, k1) in zip(base, got):
        assert n0 == n1 and k0 == k1
        x_ada = any(n0 == f"{IMG.format(i)}.adaLN_modulation.layers.1.{leaf}" for i in (0, 1)
                    for leaf in ("weight", "bias"))
        assert s1 == ((9 * h,) + s0[1:] if x_ada else s0), n0
    want = []
    for i in (0, 1):
        p = IMG.format(i)
        for n in "qkvo":
            want.append((f"{p}.attn2.{n}_proj.weight", (h, h), "w"))
            want.append((f"{p}.attn2.{n}_proj.bias", (h,), "b"))
        want += [(f"{p}.qk_norm2.q_norm.weight", (d,), "g"), (f"{p}.qk_norm2.k_norm.weight", (d,), "g")]
    for i in range(3):
        for s in ("image", "text"):
            want.append((f"multimodal_transformer_blocks.{i}.{s}_transformer_block.attn.k_proj.bias", (h,), "b"))
    assert got[len(base):] == want
    # without the k bias the attn2 k projection has none either (quirk Q3)
    no_kb = [n for n, _, _ in mmdit_param_specs(replace(cfg, attn_k_bias=False))]
    assert not any(n.endswith("k_proj.bias") for n in no_kb) and f"{IMG.format(0)}.attn2.q_proj.bias" in no_kb


def test_parameter_delta_against_sd3_medium():
    c, h, d = SD35_MEDIUM, 1536, 64
    base = replace(SD3_2b, use_qk_norm=True)
    per_x = 4 * h * h + 4 * h + 2 * d + 3 * h * h + 3 * h       # attn2 q/k/v/o, its norms, 3 more adaLN chunks
    delta = 13 * per_x + 2 * 24 * h + (384 ** 2 - 192 ** 2) * h  # + every stream's k bias + the larger position table
    assert param_count(mmdit_param_specs(c)) - param_count(mmdit_param_specs(base)) == delta
    print(f"SD3.5 Medium: {param_count(mmdit_param_specs(c)) / 1e9:.3f} B parameters")


def test_init_params_shares_the_untouched_weights():
    cfg = tiny_sd35_medium_config()
    base_cfg = replace(cfg, x_block_self_attn_layers=(), attn_k_bias=False)
    a = init_params(mmdit_param_specs(base_cfg), seed=4, dtype=torch.float32)
    b = init_params(mmdit_param_specs(cfg), seed=4, dtype=torch.float32)
    for name, t in a.items():
        if t.shape == b[name].shape:
            assert torch.equal(t, b[name]), name


# ------------------------------------------------------------------------------------------------ checkpoint
@pytest.mark.parametrize("vae", [False, True])
def test_checkpoint_roundtrip(vae):
    cfg = tiny_sd35_medium_config()
    specs = mmdit_param_specs(cfg)
    params = init_params(specs, seed=6, dtype=torch.float32)
    got = model_io.sd3_checkpoint_to_params(medium_upstream(params, cfg, vae=vae), k_bias=True)
    model_io.check_against_specs(got, specs)
    for name, t in params.items():
        assert torch.equal(got[name], t), name


def test_missing_attn2_key_is_named():
    cfg = tiny_sd35_medium_config()
    sd = medium_upstream(init_params(mmdit_param_specs(cfg), seed=6, dtype=torch.float32), cfg)
    del sd["model.diffusion_model.joint_blocks.1.x_block.attn2.proj.bias"]
    got = model_io.sd3_checkpoint_to_params(sd, k_bias=True)
    with pytest.raises(ValueError, match=re.escape(f"{IMG.format(1)}.attn2.o_proj.bias")):
        model_io.check_against_specs(got, mmdit_param_specs(cfg))


def test_wrong_family_files_are_refused():
    med = tiny_sd35_medium_config()
    large = replace(tiny_sd35_config(depth=3), upcast_multimodal_blocks=None)
    sd3 = tiny_sd3_config()
    med_sd = medium_upstream(init_params(mmdit_param_specs(med), seed=1, dtype=torch.float32), med)
    for cfg in (large, sd3):
        # a Medium file under the older presets: unexpected attn2 keys and 9h-row adaLN weights
        with pytest.raises(ValueError, match="unexpected"):
            model_io.check_against_specs(model_io.sd3_checkpoint_to_params(med_sd, k_bias=cfg.attn_k_bias),
                                         mmdit_param_specs(cfg))
        # an older file under the Medium preset: attn2 (and k biases) missing
        old_sd = medium_upstream(init_params(mmdit_param_specs(cfg), seed=1, dtype=torch.float32), cfg)
        with pytest.raises(ValueError, match="missing"):
            model_io.check_against_specs(model_io.sd3_checkpoint_to_params(old_sd, k_bias=True),
                                         mmdit_param_specs(med))


def test_loader_drops_the_k_bias_unless_asked():
    cfg = tiny_sd35_medium_config()
    sd = medium_upstream(init_params(mmdit_param_specs(cfg), seed=2, dtype=torch.float32), cfg)
    off = model_io.sd3_checkpoint_to_params(sd)
    assert not any(k.endswith("k_proj.bias") for k in off)
    on = model_io.sd3_checkpoint_to_params(sd, k_bias=True)
    assert f"{IMG.format(0)}.attn2.k_proj.bias" in on and f"{IMG.format(2)}.attn.k_proj.bias" in on


# ------------------------------------------------------------------------------------------------ LoRA, FP8
def test_lora_table_maps_attn2():
    cfg = tiny_sd35_medium_config()
    plain = module_table(replace(cfg, x_block_self_attn_layers=()))
    table = module_table(cfg)
    new = {f"joint_blocks.{i}.x_block.attn2.{m}" for i in (0, 1) for m in ("qkv", "proj")}
    assert set(table) == set(plain) | new
    h = cfg.hidden_size
    factors = make_factors({f"joint_blocks.0.x_block.attn2.qkv": (3 * h, h),
                            f"joint_blocks.1.x_block.attn2.proj": (h, h)}, rank=4, seed=3)
    want = upstream_delta(factors)
    kohya = load_lora(kohya_dict(factors), cfg)
    p0, p1 = IMG.format(0), IMG.format(1)
    assert kohya.skipped == [] and set(kohya.targets) == {f"{p0}.attn2.{n}_proj.weight" for n in "qkv"} | {
        f"{p1}.attn2.o_proj.weight"}
    qkv = torch.cat([kohya.targets[f"{p0}.attn2.{n}_proj.weight"][0] @ kohya.targets[f"{p0}.attn2.{n}_proj.weight"][1]
                     for n in "qkv"])
    torch.testing.assert_close(qkv, want["joint_blocks.0.x_block.attn2.qkv.weight"], rtol=1e-5, atol=1e-6)
    for prefix in ("", "model.diffusion_model."):
        peft = load_lora(peft_dict(factors, prefix), cfg)
        assert set(peft.targets) == set(kohya.targets)
    # a model without MMDiT-X has no such module
    with pytest.raises(KeyError, match="attn2"):
        load_lora(peft_dict(factors), replace(cfg, x_block_self_attn_layers=()))


def test_fp8_covers_attn2():
    cfg = tiny_sd35_medium_config()
    plain = fp8_covered_linears(replace(cfg, x_block_self_attn_layers=()))
    got = fp8_covered_linears(cfg)
    assert got[:len(plain)] == plain
    assert got[len(plain):] == [f"{IMG.format(i)}.attn2.{n}_proj" for i in (0, 1) for n in "qkvo"]


# ------------------------------------------------------------------------------------------------ validation
@pytest.mark.parametrize("bad, match", [
    (dict(depth_unified=2), "SD3-shaped"),
    (dict(x_block_self_attn_layers=(0, 3)), "distinct"),
    (dict(x_block_self_attn_layers=(1, 1)), "distinct"),
    (dict(x_block_self_attn_layers=(-1,)), "distinct"),
    (dict(use_qk_norm=False), "use_qk_norm"),
])
def test_config_validation(bad, match):
    cfg = replace(tiny_sd35_medium_config(), **bad)
    with pytest.raises(ValueError, match=match):
        MMDiT(cfg, {"x": torch.zeros(1, dtype=torch.float16)})


@pytest.mark.parametrize("slg, cfgw, match", [
    (SkipLayerGuidance(), 0.0, "CFG"),
    (SkipLayerGuidance(), -1.0, "CFG"),
    (SkipLayerGuidance(layers=()), 4.5, "layers"),
    (SkipLayerGuidance(layers=(7, 7)), 4.5, "layers"),
    (SkipLayerGuidance(layers=(24,)), 4.5, "layers"),
    (SkipLayerGuidance(layers=(-1,)), 4.5, "layers"),
    (SkipLayerGuidance(start=0.2, end=0.2), 4.5, "window"),
    (SkipLayerGuidance(start=-0.1), 4.5, "window"),
    (SkipLayerGuidance(end=1.5), 4.5, "window"),
    (SkipLayerGuidance(scale=float("nan")), 4.5, "finite"),
    (SkipLayerGuidance(scale=float("inf")), 4.5, "finite"),
    ((7, 8, 9), 4.5, "SkipLayerGuidance"),
])
def test_slg_validation(slg, cfgw, match):
    with pytest.raises(ValueError, match=match):
        check_skip_layer_guidance(slg, cfgw, 24)


def test_slg_refused_on_flux_and_accepted_otherwise():
    with pytest.raises(ValueError, match="SD3-family"):
        _check_slg(SkipLayerGuidance(layers=(1,)), 4.5, tiny_flux_config())
    _check_slg(None, 0.0, tiny_flux_config())
    _check_slg(SkipLayerGuidance(), 4.5, SD35_MEDIUM)
    _check_slg(SkipLayerGuidance(layers=(0, 1, 2)), 4.5, tiny_sd3_config())


def test_slg_api():
    s = SkipLayerGuidance()
    assert (s.scale, s.layers, s.start, s.end) == (2.5, (7, 8, 9), 0.01, 0.20)
    with pytest.raises(Exception):
        s.scale = 1.0                                            # frozen
    for cls in (DiffusionPipeline,):
        for fn in (cls.denoise_latents, cls.generate_image):
            p = inspect.signature(fn).parameters["slg"]
            assert p.kind == inspect.Parameter.KEYWORD_ONLY and p.default is None
    for fn in (FluxPipeline.denoise_latents, FluxPipeline.generate_image):
        assert "slg" not in inspect.signature(fn).parameters


def test_slg_window():
    s = SkipLayerGuidance()
    assert skip_layer_guidance_steps(s, 40) == list(range(1, 8)) == slg_window(40, 0.01, 0.20)
    assert skip_layer_guidance_steps(s, 28) == list(range(1, 6)) == slg_window(28, 0.01, 0.20)
    for n in (1, 2, 4, 6, 9, 17, 50):
        for start, end in ((0.0, 1.0), (0.1, 0.6), (0.01, 0.2)):
            assert skip_layer_guidance_steps(SkipLayerGuidance(start=start, end=end), n) == slg_window(n, start, end)


# ------------------------------------------------------------------------------------------------ oracle pins
def _case(cfg, seed=1, B=2, T=8, lat=(4, 6)):
    g = torch.Generator().manual_seed(seed)
    latent = torch.randn((B, lat[0], lat[1], 16), generator=g)
    text = torch.randn((B, T, cfg.token_level_text_embed_dim), generator=g)
    pooled = torch.randn((B, cfg.pooled_text_embed_dim), generator=g)
    return latent, text, pooled, torch.tensor([701.0])


def _run(ref, case, **kw):
    latent, text, pooled, t = case
    ref.cache_modulation_params(pooled, t)
    return ref(latent, text, t.repeat(latent.shape[0]), **kw)


@pytest.mark.parametrize("act_dtype", [None, torch.float16])
def test_zero_attn2_is_the_plain_oracle(act_dtype):
    """zero attn2 output and zero k biases: MMDiTRef on the same other weights and the 6h-row adaLN slice, on an
    SD3.5-large-shaped tiny config"""
    plain_cfg = replace(tiny_sd35_config(depth=3), upcast_multimodal_blocks=None)
    cfg = replace(plain_cfg, x_block_self_attn_layers=(0, 2), attn_k_bias=True)
    p = init_params(mmdit_param_specs(cfg), seed=3, dtype=torch.float32)
    for i in (0, 2):
        p[f"{IMG.format(i)}.attn2.o_proj.weight"].zero_()
        p[f"{IMG.format(i)}.attn2.o_proj.bias"].zero_()
    for k in p:
        if k.endswith("k_proj.bias"):
            p[k].zero_()
    plain = {k: v for k, v in p.items() if k in {n for n, _, _ in mmdit_param_specs(plain_cfg)}}
    for i in (0, 2):
        for leaf in ("weight", "bias"):
            name = f"{IMG.format(i)}.adaLN_modulation.layers.1.{leaf}"
            plain[name] = p[name][:6 * cfg.hidden_size]
    case = _case(cfg)
    got = _run(xref(cfg, p, act_dtype), case)
    want = _run(MMDiTRef(ref_config(plain_cfg), plain, act_dtype), case)
    assert torch.equal(got, want)


def _np_x_forward(ref, case, order):
    """fp64 numpy transcription of a depth-1 MMDiT-X forward (Stability's pre_attention_x / post_attention_x), with
    the modulation vectors and the embedders' outputs of the oracle as inputs; order = chunk indices of
    (msa, mlp, msa2)"""
    P = {k: v.double().numpy() for k, v in ref.p.items()}
    cfg = ref.cfg
    latent, text, pooled, t = case
    ref.cache_modulation_params(pooled, t)
    mods = {k: v.double().numpy() for k, v in ref._mod[float(t[0])].items()}
    h, H, d = cfg.hidden_size, cfg.num_heads, cfg.hidden_size // cfg.num_heads
    B, Hl, Wl, C = latent.shape
    hp, wp = Hl // 2, Wl // 2
    N = hp * wp

    def lin(x, name, bias=True):
        y = x @ P[name + ".weight"].reshape(P[name + ".weight"].shape[0], -1).T
        return y + P[name + ".bias"] if bias and name + ".bias" in P else y

    def ln(x):
        mu = x.mean(-1, keepdims=True)
        return (x - mu) / np.sqrt(((x - mu) ** 2).mean(-1, keepdims=True) + 1e-6)

    def rms(x, w):
        return x / np.sqrt((x * x).mean(-1, keepdims=True) + 1e-6) * w

    def attention(q, k, v):
        s = np.einsum("bhqd,bhkd->bhqk", q, k) / math.sqrt(d)
        s = np.exp(s - s.max(-1, keepdims=True))
        return np.einsum("bhqk,bhkd->bhqd", s / s.sum(-1, keepdims=True), v)

    def heads(x):
        return x.reshape(B, -1, H, d).transpose(0, 2, 1, 3)

    def qkv(x, attn, norm):
        q, k, v = (heads(lin(x, f"{attn}.{n}_proj")) for n in "qkv")
        return rms(q, P[norm + ".q_norm.weight"]), rms(k, P[norm + ".k_norm.weight"]), v

    rows = latent.double().numpy().reshape(B, hp, 2, wp, 2, C).transpose(0, 1, 3, 2, 4, 5).reshape(B, N, -1)
    m = cfg.max_latent_resolution
    pos = P["x_pos_embedder.pos_embed.weight"].reshape(m, m, h)[(m - hp) // 2:(m - hp) // 2 + hp,
                                                              (m - wp) // 2:(m - wp) // 2 + wp].reshape(1, N, h)
    x = lin(rows, "x_embedder.proj") + pos
    c = lin(text.double().numpy(), "context_embedder")
    ib, tb = IMG.format(0), "multimodal_transformer_blocks.0.text_transformer_block"
    ch = [mods[ib][:, None, j * h:(j + 1) * h] for j in range(9)]
    msa, mlp, msa2 = (ch[3 * o:3 * o + 3] for o in order)
    cm = [mods[tb][:, None, j * h:(j + 1) * h] for j in range(2)]
    # pre_attention_x: one LayerNorm, two modulations
    n = ln(x)
    qi, ki, vi = qkv(n * (1 + msa[1]) + msa[0], ib + ".attn", ib + ".qk_norm")
    q2, k2, v2 = qkv(n * (1 + msa2[1]) + msa2[0], ib + ".attn2", ib + ".qk_norm2")
    qt, kt, vt = qkv(ln(c) * (1 + cm[1]) + cm[0], tb + ".attn", tb + ".qk_norm")
    o = attention(np.concatenate([qi, qt], 2), np.concatenate([ki, kt], 2), np.concatenate([vi, vt], 2))
    o = o.transpose(0, 2, 1, 3).reshape(B, -1, h)[:, :N]
    o2 = attention(q2, k2, v2).transpose(0, 2, 1, 3).reshape(B, N, h)
    # post_attention_x
    x = x + msa[2] * lin(o, ib + ".attn.o_proj") + msa2[2] * lin(o2, ib + ".attn2.o_proj")
    hid = lin(ln(x) * (1 + mlp[1]) + mlp[0], ib + ".mlp.fc1")
    hid = 0.5 * hid * (1 + np.vectorize(math.erf)(hid / math.sqrt(2)))
    x = x + mlp[2] * lin(hid, ib + ".mlp.fc2")
    f = mods["final_layer"][:, None]
    y = lin(ln(x) * (1 + f[..., h:]) + f[..., :h], "final_layer.linear")
    return y.reshape(B, hp, wp, 2, 2, C).transpose(0, 5, 1, 3, 2, 4).reshape(B, C, Hl, Wl).transpose(0, 2, 3, 1)


def test_one_x_block_matches_stabilitys_formulas():
    cfg = replace(tiny_sd35_medium_config(), depth_multimodal=1, x_block_self_attn_layers=(0,))
    p = init_params(mmdit_param_specs(cfg), seed=5, dtype=torch.float32)
    ref = xref(cfg, p)
    case = _case(cfg, seed=2)
    got = _run(ref, case).double().numpy()
    want = _np_x_forward(ref, case, (0, 1, 2))
    err = np.linalg.norm(got - want) / np.linalg.norm(want)
    swapped = _np_x_forward(ref, case, (0, 2, 1))                # msa2 and mlp chunks exchanged
    sep = np.linalg.norm(swapped - want) / np.linalg.norm(want)
    print(f"x-block vs fp64: {err:.2e}; swapped chunks: {sep:.2e}")
    assert err <= 1e-5 and sep >= 1e-2


def test_attn2_of_block_0_ignores_the_text():
    cfg = tiny_sd35_medium_config()
    p = init_params(mmdit_param_specs(cfg), seed=8, dtype=torch.float32)
    for name in ("attn.o_proj.weight", "attn.o_proj.bias"):
        p[f"{IMG.format(0)}.{name}"].zero_()                     # the joint attention no longer reaches the image
    cfg1 = replace(cfg, depth_multimodal=1, x_block_self_attn_layers=(0,))
    p1 = {k: v for k, v in p.items() if k in {n for n, _, _ in mmdit_param_specs(cfg1)} or "blocks.0." in k}
    p1["multimodal_transformer_blocks.0.text_transformer_block.adaLN_modulation.layers.1.weight"] = \
        p["multimodal_transformer_blocks.0.text_transformer_block.adaLN_modulation.layers.1.weight"][:2 * 128]
    p1["multimodal_transformer_blocks.0.text_transformer_block.adaLN_modulation.layers.1.bias"] = \
        p["multimodal_transformer_blocks.0.text_transformer_block.adaLN_modulation.layers.1.bias"][:2 * 128]
    latent, text, pooled, t = _case(cfg1, seed=3)
    other = torch.randn_like(text)
    ref = xref(cfg1, p1)
    a = _run(ref, (latent, text, pooled, t))
    b = _run(ref, (latent, other, pooled, t))
    assert torch.equal(a, b)
    p1[f"{IMG.format(0)}.attn2.o_proj.bias"] = torch.zeros_like(p1[f"{IMG.format(0)}.attn2.o_proj.bias"])
    p1[f"{IMG.format(0)}.attn2.o_proj.weight"] = torch.zeros_like(p1[f"{IMG.format(0)}.attn2.o_proj.weight"])
    assert not torch.equal(_run(xref(cfg1, p1), (latent, text, pooled, t)), a)   # attn2 does reach the output


def test_k_bias_changes_the_output():
    cfg = tiny_sd35_medium_config()
    p = init_params(mmdit_param_specs(cfg), seed=9, dtype=torch.float32)
    case = _case(cfg)
    a = _run(xref(cfg, p), case)
    dropped = _run(MMDiTXRef(ref_config(cfg), p, None, cfg.x_block_self_attn_layers, k_bias=False), case)
    r = (a - dropped).norm() / a.norm()
    print(f"k bias on vs dropped: rel_l2 {r:.2e}")
    assert r >= 1e-3


def _sched(n):
    return sr.get_sigmas(sr.ModelSamplingDiscreteFlowRef(3.0), n)


@pytest.mark.parametrize("solver", ["euler", "heun", "dpmpp_2m"])
def test_slg_off_is_the_cfg_oracle(solver):
    """scale 0, and layers=(), give the CFG oracles exactly"""
    cfg = tiny_sd35_medium_config()
    p = init_params(mmdit_param_specs(cfg), seed=4, dtype=torch.float32)
    ref = xref(cfg, p, torch.float16)
    sig = _sched(5)
    g = torch.Generator().manual_seed(7)
    x0 = torch.randn((1, 4, 6, 16), generator=g)
    cond = torch.randn((2, 8, cfg.token_level_text_embed_dim), generator=g)
    pooled = torch.randn((2, cfg.pooled_text_embed_dim), generator=g)
    base = {"euler": sr.sample_euler, "heun": solver_ref.sample_heun, "dpmpp_2m": solver_ref.sample_dpmpp_2m}[solver]
    want = base(lambda xin, c, t: ref(xin, c, t), ref.cache_modulation_params, x0, sig, cond, pooled, 4.5,
                torch.float16)
    for scale, layers in ((0.0, (1,)), (2.5, ())):
        got = sample(solver, ref, x0, sig, cond, pooled, 4.5, torch.float16, scale=scale, layers=layers, start=0.0,
                     end=1.0)
        assert torch.equal(got, want), (scale, layers)
    on = sample(solver, ref, x0, sig, cond, pooled, 4.5, torch.float16, scale=2.5, layers=(1,), start=0.0, end=1.0)
    assert not torch.equal(on, want)


def test_slg_mix_matches_fp64():
    cfg = tiny_sd35_medium_config()
    p = init_params(mmdit_param_specs(cfg), seed=10, dtype=torch.float32)
    ref = xref(cfg, p)
    case = _case(cfg, B=2)
    latent, text, pooled, t = case
    x = latent[:1]
    ref.cache_modulation_params(pooled, t)
    sigma, w, s = 0.71, 4.5, 2.5
    got = slg_denoiser(ref, x, text, t[0], sigma, w, lambda v: v, s, (1,), True)
    o2 = ref(torch.cat([x, x]), text, t.repeat(2)).double()
    osk = ref(x, text[:1], t.repeat(1), skip_layers=(1,)).double()
    xd = x.double()
    d_pos, d_neg, d_skip = xd - o2[:1] * sigma, xd - o2[1:] * sigma, xd - osk * sigma
    want = d_neg + w * (d_pos - d_neg) + s * (d_pos - d_skip)
    assert ((got.double() - want).norm() / want.norm()) <= 1e-6
    assert not torch.equal(osk, o2[:1])                          # the skip forward differs from the positive one
