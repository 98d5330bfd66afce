"""CPU: FLUX.1 Fill [dev] (DESIGN.md §18) — the einops packing against the index formula, the masked
pre-normalisation, the config / specs / checkpoint loader and its refusals, the argument checks that run before GPU
work, an all-zeros mask, and the column split of an x-embedder LoRA."""
from dataclasses import replace

import numpy as np
import pytest
import torch

from diffusionkit_b200 import fill, model_io
from diffusionkit_b200.config import (FLUX_DEV, FLUX_FILL_DEV, MODEL_CONFIGS, T5_MAX_LENGTH, tiny_flux_config)
from diffusionkit_b200.lora import load_lora
from diffusionkit_b200.pipeline import DEFAULT_GUIDANCE, MMDIT_CKPT, DiffusionPipeline, FluxPipeline
from diffusionkit_b200.weights import init_params, mmdit_param_specs
from tests import fill_ref
from tests.kontext_ref import patch_rows
from tests.lora_fixtures import kohya_dict, make_factors, upstream_modules
from tests.test_guidance_cpu import dev_upstream

FILL = "black-forest-labs/FLUX.1-Fill-dev"


def tiny_fill_config():
    return replace(tiny_flux_config(), guidance_embed=True, x_embedder_cond_channels=320)


def _mask(H, W, seed=0, p=0.3):
    return (np.random.RandomState(seed).rand(H, W) < p).astype(np.uint8)


# ------------------------------------------------------------------------------------------------ packing
@pytest.mark.parametrize("H, W", [(16, 16), (64, 128), (48, 32)])
def test_einops_mask_packing_is_the_index_formula(H, W):
    m = _mask(H, W, seed=H + W)
    got = fill_ref.bfl_pack_mask(m)
    assert got.shape == (1, (H // 16) * (W // 16), 256)
    assert np.array_equal(got[0].numpy(), fill_ref.loop_mask_channels(m))


def test_latent_packing_is_the_target_packing():
    lat = torch.randn((2, 8, 12, 16), generator=torch.Generator().manual_seed(1))
    assert torch.equal(fill_ref.bfl_pack_latent(lat), patch_rows(lat))


def test_masked_prenormalisation_is_bfls_formula():
    rng = np.random.RandomState(3)
    src = rng.randint(0, 256, (32, 48, 4), dtype=np.uint8)
    m = _mask(32, 48, seed=4)
    got = fill_ref.ref_image_pre_masked(torch.from_numpy(src)[None], torch.from_numpy(m), torch.float32, cpad=8)
    want = fill_ref.bfl_img_cond(src, m)
    assert torch.equal(got[..., :3], want)                          # == : BFL's -0.0 equals the kernel's +0
    assert not bool(got[..., 3:].any())
    assert not bool(torch.signbit(got[0][torch.from_numpy(m) != 0]).any()), "masked pixels are +0"
    kept = torch.from_numpy(m) == 0
    plain = fill_ref.ref_image_pre_masked(torch.from_numpy(src)[None], torch.zeros(32, 48, dtype=torch.uint8),
                                          torch.bfloat16)
    assert torch.equal(fill_ref.ref_image_pre_masked(torch.from_numpy(src)[None], torch.from_numpy(m),
                                                     torch.bfloat16)[0][kept], plain[0][kept])


# ------------------------------------------------------------------------------------------------ config and loader
def test_config_and_specs():
    assert FLUX_FILL_DEV == replace(FLUX_DEV, x_embedder_cond_channels=320)
    assert MODEL_CONFIGS[FILL] is FLUX_FILL_DEV and T5_MAX_LENGTH[FILL] == 512 and MMDIT_CKPT[FILL] == FILL
    assert all(c.x_embedder_cond_channels == 0 for k, c in MODEL_CONFIGS.items() if k != FILL)
    plain, filled = mmdit_param_specs(FLUX_DEV), mmdit_param_specs(FLUX_FILL_DEV)
    assert len(plain) == len(filled)
    for a, b in zip(plain, filled):
        if a[0] == "x_embedder.proj.weight":
            assert a[1] == (3072, 1, 1, 64) and b[1] == (3072, 1, 1, 384)
        else:
            assert a == b
    assert fill.COND_CHANNELS == 320 and fill.DEFAULT_GUIDANCE == 30.0


def test_loader_takes_the_fill_layout_and_refuses_mismatches():
    cfg, dev = tiny_fill_config(), replace(tiny_flux_config(), guidance_embed=True)
    params = init_params(mmdit_param_specs(cfg), seed=5, dtype=torch.float32)
    sd = dev_upstream(params, cfg)
    assert tuple(sd["img_in.weight"].shape) == (cfg.hidden_size, 384)
    got = model_io.flux_checkpoint_to_params(sd, cfg.hidden_size, cfg.mlp_ratio, guidance_embed=True,
                                             cond_channels=320)
    model_io.check_against_specs(got, mmdit_param_specs(cfg))
    assert torch.equal(got["x_embedder.proj.weight"], params["x_embedder.proj.weight"])
    with pytest.raises(ValueError, match="img_in.weight.*plain FLUX"):
        model_io.flux_checkpoint_to_params(sd, cfg.hidden_size, cfg.mlp_ratio, guidance_embed=True)
    plain_sd = dev_upstream(init_params(mmdit_param_specs(dev), seed=5, dtype=torch.float32), dev)
    with pytest.raises(ValueError, match="img_in.weight.*FLUX.1 Fill"):
        model_io.flux_checkpoint_to_params(plain_sd, cfg.hidden_size, cfg.mlp_ratio, guidance_embed=True,
                                           cond_channels=320)


# ------------------------------------------------------------------------------------------------ argument checks
def _stub(cls, cfg):
    """a pipeline object with only its config: the checks below run before any model or GPU work"""
    p = object.__new__(cls)
    p.config = cfg
    return p


def test_argument_errors_before_gpu_work():
    flux = _stub(FluxPipeline, tiny_fill_config())
    img, m = np.zeros((64, 64, 3), np.uint8), np.zeros((64, 64), np.uint8)
    for kw, msg in [(dict(image_path=img, mask_image=None), "needs image_path and mask_image"),
                    (dict(image_path=None, mask_image=m), "needs image_path and mask_image"),
                    (dict(image_path=img, mask_image=m, reference_latents=torch.zeros(1, 8, 8, 16)), "Kontext"),
                    (dict(image_path=img, mask_image=m, reference_image=img), "Kontext")]:
        kw.setdefault("reference_image", None)
        kw.setdefault("reference_latents", None)
        with pytest.raises(ValueError, match=msg):
            flux._check_fill(**kw)
    flux._check_fill(img, m, None, None)
    with pytest.raises(ValueError, match="FluxPipeline only"):
        _stub(DiffusionPipeline, tiny_fill_config())._check_fill(img, m, None, None)
    # other models: nothing to check, and mask_image keeps its §17 meaning
    _stub(FluxPipeline, replace(tiny_flux_config(), guidance_embed=True))._check_fill(None, m, None, None)


def test_default_guidance_is_30_on_fill_only():
    assert _stub(FluxPipeline, tiny_fill_config())._guidance_values(None, 2) == [30.0, 30.0]
    dev = _stub(FluxPipeline, replace(tiny_flux_config(), guidance_embed=True))
    assert dev._guidance_values(None, 1) == [DEFAULT_GUIDANCE] == [3.5]
    assert _stub(FluxPipeline, tiny_fill_config())._guidance_values([2.0, 4.0], 2) == [2.0, 4.0]


# ------------------------------------------------------------------------------------------------ oracle properties
class _TinyEncoder:
    """a deterministic stand-in for the VAE encoder: per-8x8-block means of the three channels and their squares, as
    (mean | logvar) with 16 channels each"""

    def __call__(self, x):
        B, H, W, _ = x.shape
        blk = x.reshape(B, H // 8, 8, W // 8, 8, 3).mean(dim=(2, 4))
        mean = torch.cat([blk, blk ** 2, blk.flip(-1), torch.zeros(B, H // 8, W // 8, 7)], dim=-1)
        return torch.cat([mean, torch.full_like(mean, -3.0)], dim=-1)


def test_all_zeros_mask_gives_zero_mask_channels_and_the_encoded_source():
    from tests.model_checks import _test_image

    src = _test_image(64, 96)
    zeros = np.zeros((64, 96), np.uint8)
    rows = fill_ref.oracle_cond_rows(_TinyEncoder(), src, zeros, 0.1159, 0.3611, torch.bfloat16)
    assert rows.shape == (4 * 6, 320) and not bool(rows[:, 64:].any())
    x = torch.from_numpy(src).float()[None] / 255 * 2 - 1.0
    mean = _TinyEncoder()(x)[..., :16]
    want = fill_ref.bfl_pack_latent(((mean - 0.1159) * 0.3611).to(torch.bfloat16).float())[0]
    assert torch.equal(rows[:, :64], want)
    ones = fill_ref.oracle_cond_rows(_TinyEncoder(), src, np.ones((64, 96), np.uint8), 0.1159, 0.3611, torch.bfloat16)
    assert bool((ones[:, 64:] == 1).all())


def test_lora_on_the_x_embedder_splits_by_columns():
    """a Fill model's img_in adapter has 384 down columns; merged into the packed (h, 384) weight it equals the latent
    columns and the conditioning columns merged separately"""
    cfg = tiny_fill_config()
    mods = {k: v for k, v in upstream_modules(cfg).items() if k == "img_in"}
    assert mods == {"img_in": (cfg.hidden_size, 384)}
    lora = load_lora(kohya_dict(make_factors(mods, 4, seed=2)), cfg)
    up, down = lora.targets["x_embedder.proj.weight"]
    assert tuple(down.shape) == (4, 384)
    w = init_params(mmdit_param_specs(cfg), seed=1, dtype=torch.float32)["x_embedder.proj.weight"].reshape(
        cfg.hidden_size, -1)
    merged = w + up @ down
    split = torch.cat([w[:, :64] + up @ down[:, :64], w[:, 64:] + up @ down[:, 64:]], dim=1)
    assert torch.allclose(merged, split, rtol=0, atol=1e-6)
    with pytest.raises(ValueError, match="img_in"):
        load_lora(kohya_dict(make_factors({"img_in": (cfg.hidden_size, 64)}, 4, seed=2)), cfg)
