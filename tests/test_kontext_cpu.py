"""CPU: FLUX.1 Kontext (DESIGN.md §14) — the ids-driven oracle's properties (tests/kontext_ref.py), the engine's RoPE
table against BFL's id layout, the preset, and the pipeline's argument checks that run before any GPU work."""
import inspect
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from diffusionkit_b200 import model_io
from diffusionkit_b200.config import FLUX_DEV, MODEL_CONFIGS, T5_MAX_LENGTH, tiny_flux_config, tiny_sd3_config
from diffusionkit_b200.mmdit import MMDiT
from diffusionkit_b200.pipeline import MMDIT_CKPT, DiffusionPipeline, FluxPipeline
from diffusionkit_b200.weights import init_params, mmdit_param_specs
from oracle.mmdit_ref import MMDiTRef
from tests.guidance_ref import GuidanceMMDiTRef
from tests.kontext_ref import KontextMMDiTRef, kontext_ids, patch_rows, rope_from_ids, sharpen
from tests.oracle_bridge import ref_config
from tests.test_guidance_cpu import dev_upstream, tiny_dev_config

KONTEXT = "black-forest-labs/FLUX.1-Kontext-dev"
T = 8


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def _case(cfg, B=1, lat=(8, 8), ref=(8, 12), seed=5):
    params = init_params(mmdit_param_specs(cfg), seed=7, dtype=torch.float32)
    g = torch.Generator().manual_seed(seed)
    latent = torch.randn((B, *lat, 16), generator=g)
    reference = torch.randn((B, *ref, 16), generator=g)
    text = torch.randn((B, T, cfg.token_level_text_embed_dim), generator=g)
    pooled = torch.randn((B, cfg.pooled_text_embed_dim), generator=g)
    return params, latent, reference, text, pooled, torch.tensor([752.0])


def _kontext(cfg, params, pooled, t, guidance):
    ref = KontextMMDiTRef(ref_config(cfg), params)
    ref.cache_modulation_params(pooled, t, guidance)
    return ref


# ------------------------------------------------------------------------------------------------ oracle properties
@pytest.mark.parametrize("dev", [False, True])
def test_no_reference_tokens_is_the_parent_oracle(dev):
    cfg = tiny_dev_config() if dev else tiny_flux_config()
    params, latent, _, text, pooled, t = _case(cfg, B=2)
    guidance = [2.5, 5.0] if dev else None
    parent = GuidanceMMDiTRef(ref_config(cfg), params) if dev else MMDiTRef(ref_config(cfg), params)
    if dev:
        parent.cache_modulation_params(pooled, t, guidance)
    else:
        parent.cache_modulation_params(pooled, t)
    want = parent(latent, text, t.repeat(2))
    got = _kontext(cfg, params, pooled, t, guidance)(latent, text, t.repeat(2))
    assert torch.equal(got, want)


def test_position_enters_only_through_the_ids():
    """[text | reference | target] with the ids carried along gives the target outputs up to fp32 reassociation"""
    cfg = tiny_dev_config()
    params, latent, reference, text, pooled, t = _case(cfg, B=1, lat=(8, 8), ref=(8, 12))
    ref = _kontext(cfg, params, pooled, t, [3.5])
    rows_x, rows_r = patch_rows(latent), patch_rows(reference)
    Nx, Nr = rows_x.shape[1], rows_r.shape[1]
    ids = kontext_ids(T, 4, 4, (4, 6))
    want = ref.forward_tokens(text, torch.cat([rows_x, rows_r], 1), ids, t, torch.arange(Nx))
    perm_ids = torch.cat([ids[:T], ids[T + Nx:], ids[T:T + Nx]])
    got = ref.forward_tokens(text, torch.cat([rows_r, rows_x], 1), perm_ids, t, Nr + torch.arange(Nx))
    r = _rel(got, want)
    print(f"permuted sequence: rel_l2 {r:.2e}")
    assert r <= 1e-5, r
    # without the ids the order matters: the same permutation with the unpermuted ids is far off
    wrong = ref.forward_tokens(text, torch.cat([rows_r, rows_x], 1), ids, t, Nr + torch.arange(Nx))
    assert _rel(wrong, want) > 1e-2


def _bfl_kontext_ids(T, h, w, hr, wr):
    """numpy transcription of BFL's prepare_kontext / diffusers' _prepare_latent_image_ids for latent (not packed)
    sizes h x w (target) and hr x wr (reference): text ids zero, image ids (0, r, c), reference ids (1, r, c)"""
    def latent_image_ids(hh, ww):
        ids = np.zeros((hh // 2, ww // 2, 3), dtype=np.float32)
        ids[..., 1] = ids[..., 1] + np.arange(hh // 2)[:, None]
        ids[..., 2] = ids[..., 2] + np.arange(ww // 2)[None, :]
        return ids.reshape(-1, 3)

    txt_ids = np.zeros((T, 3), dtype=np.float32)
    img_ids = latent_image_ids(h, w)
    cond_ids = latent_image_ids(hr, wr)
    cond_ids[..., 0] = 1
    return np.concatenate([txt_ids, img_ids, cond_ids])


def test_ids_are_bfl_prepare_kontext():
    """target 16 x 16 latent, reference 16 x 32: the oracle's ids and the engine's RoPE table both follow BFL"""
    want = _bfl_kontext_ids(T, 16, 16, 16, 32)
    ids = kontext_ids(T, 8, 8, (8, 16))
    assert np.array_equal(ids.numpy(), want)
    cfg = tiny_flux_config()
    stub = SimpleNamespace(config=cfg, d=cfg.head_dim, device=torch.device("cpu"))
    table = MMDiT._rope_table(stub, {}, T, 8, 8, (8, 16))
    assert torch.equal(table, rope_from_ids(torch.from_numpy(want), cfg.rope_axes_dim))
    # without a reference the table is the parent oracle's
    from oracle.mmdit_ref import rope_table

    assert torch.equal(MMDiT._rope_table(stub, {}, T, 8, 8), rope_table(T, 8, 8, cfg.rope_axes_dim))


def test_the_reference_and_its_axis0_id_matter():
    """with the reference, without it, and with its axis-0 id 0 instead of 1: three outputs far apart, so that the
    GPU bounds (rel-L2 <= 2e-2) tell them apart.  The GPU tests use the same sharpened weights."""
    cfg = tiny_dev_config()
    params, latent, reference, text, pooled, t = _case(cfg, B=1, lat=(8, 8), ref=(8, 8))
    ref = _kontext(cfg, sharpen(params), pooled, t, [3.5])
    with_ref = ref(latent, text, t, reference=reference)
    without = ref(latent, text, t)
    axis0 = ref(latent, text, t, reference=reference, ref_axis0=0.0)
    gaps = {"with vs without": _rel(without, with_ref), "with vs axis0=0": _rel(axis0, with_ref),
            "without vs axis0=0": _rel(axis0, without)}
    print("oracle gaps (rel_l2):", {k: f"{v:.3f}" for k, v in gaps.items()})
    for name, gap in gaps.items():
        assert gap >= 4 * 2e-2, (name, gap)


# ------------------------------------------------------------------------------------------------ preset and loader
def test_kontext_preset():
    assert MODEL_CONFIGS[KONTEXT] is FLUX_DEV and MMDIT_CKPT[KONTEXT] == KONTEXT and T5_MAX_LENGTH[KONTEXT] == 512


def test_a_checkpoint_with_other_keys_fails_naming_the_key():
    """the released Kontext file is taken to have FLUX.1-dev's keys; a file that does not must fail loudly"""
    cfg = tiny_dev_config()
    params = init_params(mmdit_param_specs(cfg), seed=3, dtype=torch.float32)
    sd = dev_upstream(params, cfg)
    got = model_io.flux_checkpoint_to_params(sd, cfg.hidden_size, cfg.mlp_ratio, guidance_embed=True)
    model_io.check_against_specs(got, mmdit_param_specs(cfg))
    missing = dict(sd)
    del missing["final_layer.linear.weight"]
    with pytest.raises(ValueError, match="final_layer.linear.weight"):
        model_io.check_against_specs(
            model_io.flux_checkpoint_to_params(missing, cfg.hidden_size, cfg.mlp_ratio, guidance_embed=True),
            mmdit_param_specs(cfg))
    extra = dict(sd, **{"double_blocks.0.img_attn.extra.weight": sd["final_layer.linear.weight"]})
    with pytest.raises(KeyError, match="double_blocks.0.img_attn.extra.weight"):
        model_io.flux_checkpoint_to_params(extra, cfg.hidden_size, cfg.mlp_ratio, guidance_embed=True)


# ------------------------------------------------------------------------------------------------ pipeline arguments
def test_only_flux_pipelines_take_a_reference():
    for name in ("generate_image", "denoise_latents"):
        flux = inspect.signature(getattr(FluxPipeline, name)).parameters
        sd3 = inspect.signature(getattr(DiffusionPipeline, name)).parameters
        for arg in ("reference_image", "reference_latents"):
            assert flux[arg].kind == inspect.Parameter.KEYWORD_ONLY and flux[arg].default is None
            assert arg not in sd3


def _pipe_stub(cfg):
    """a FluxPipeline without its models: enough for the host-side argument checks"""
    pipe = object.__new__(FluxPipeline)
    pipe.config = cfg
    return pipe


def test_reference_argument_checks():
    pipe = _pipe_stub(FLUX_DEV)
    lat = torch.zeros((1, 8, 12, 16))
    rgb = np.zeros((128, 192, 3), dtype=np.uint8)
    assert pipe._reference_input(None, None, 2) is None
    r, size = pipe._reference_input(None, lat, 2)
    assert r is lat and size == (8, 12)
    assert pipe._reference_input(None, torch.zeros((2, 8, 12, 16)), 2)[1] == (8, 12)
    arr, size = pipe._reference_input(rgb, None, 1)
    assert arr.shape == (128, 192, 3) and size == (16, 24)
    arr, size = pipe._reference_input(np.zeros((100, 150, 3), dtype=np.uint8), None, 1)   # sides cut to 64
    assert arr.shape == (64, 128, 3) and size == (8, 16)
    bad = [
        dict(reference_image=rgb, reference_latents=lat),                       # both
        dict(reference_latents=torch.zeros((1, 7, 12, 16))),                    # odd height
        dict(reference_latents=torch.zeros((1, 8, 13, 16))),                    # odd width
        dict(reference_latents=torch.zeros((3, 8, 12, 16))),                    # batch neither 1 nor B
        dict(reference_latents=torch.zeros((1, 8, 12, 16), dtype=torch.bfloat16)),  # not fp32
        dict(reference_latents=torch.zeros((1, 8, 12, 4))),                     # not 16 channels
        dict(reference_latents=torch.zeros((8, 12, 16))),                       # not NHWC
        dict(reference_image=np.zeros((128, 128), dtype=np.uint8)),             # greyscale array
        dict(reference_image=np.zeros((128, 128, 1), dtype=np.uint8)),
    ]
    from PIL import Image

    bad.append(dict(reference_image=Image.new("L", (128, 128))))                  # greyscale image
    for kw in bad:
        with pytest.raises(ValueError):
            pipe._reference_input(kw.get("reference_image"), kw.get("reference_latents"), 2)
    with pytest.raises(ValueError, match="FLUX-shaped"):
        _pipe_stub(tiny_sd3_config())._reference_input(None, lat, 1)
