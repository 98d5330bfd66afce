"""CPU: FLUX.1 Canny / Depth [dev] (DESIGN.md §19) — the numpy Canny of tests/control_ref.py against committed
cv2.Canny outputs (and live cv2 where it imports), BFL's round-trip table, the control image's loading, the config /
specs / checkpoint loader and its refusals, the argument checks that run before GPU work, the guidance defaults, and
the packing of the control rows against the index formula."""
import os
from dataclasses import replace

import numpy as np
import pytest
import torch

from diffusionkit_b200 import control, model_io
from diffusionkit_b200.config import (CONTROL_MODEL_CONFIGS, FLUX_CANNY_DEV, FLUX_DEPTH_DEV, FLUX_DEV, FLUX_FILL_DEV,
                                      MODEL_CONFIGS, T5_MAX_LENGTH, tiny_flux_config)
from diffusionkit_b200.pipeline import DEFAULT_GUIDANCE, MMDIT_CKPT, DiffusionPipeline, FluxPipeline
from diffusionkit_b200.weights import init_params, mmdit_param_specs
from tests import control_ref
from tests.fill_ref import bfl_pack_latent
from tests.test_guidance_cpu import dev_upstream

CANNY, DEPTH = "black-forest-labs/FLUX.1-Canny-dev", "black-forest-labs/FLUX.1-Depth-dev"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "canny_cv2.npz")


def tiny_control_config(kind: str = "canny"):
    return replace(tiny_flux_config(), guidance_embed=True, x_embedder_cond_channels=64, control=kind)


# ------------------------------------------------------------------------------------------------ Canny
def test_oracle_canny_equals_the_committed_cv2_outputs():
    g = np.load(GOLDEN)
    n = sum(1 for k in g.files if k.endswith("_edges"))
    assert n >= 6
    for i in range(n):
        img, (low, high), want = g[f"case{i}_img"], g[f"case{i}_thr"], g[f"case{i}_edges"]
        got = control_ref.canny(img, int(low), int(high))
        assert got.dtype == np.uint8 and np.array_equal(got, want), (i, int((got != want).sum()))


def test_oracle_canny_equals_live_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(7)
    bad = 0
    for t in range(24):
        H, W = (int(v) for v in rng.integers(16, 120, 2))
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        if t % 3:
            img = cv2.GaussianBlur(img, (0, 0), float(rng.uniform(0.7, 3.0)))
        low = int(rng.integers(10, 80))
        high = low + int(rng.integers(0, 200))
        bad += int((cv2.Canny(img, low, high) != control_ref.canny(img, low, high)).sum())
        grey = np.ascontiguousarray(img[..., 1])
        bad += int((cv2.Canny(grey, low, high) != control_ref.canny(grey, low, high)).sum())
    s = control_ref.spiral(150, 130)
    bad += int((cv2.Canny(s, 50, 200) != control_ref.canny(s)).sum())
    assert bad == 0


def test_spiral_is_connected_by_hysteresis_only():
    s = control_ref.spiral(96, 96)
    strong_only = int((control_ref.canny(s, 200, 200) > 0).sum())
    full = int((control_ref.canny(s) > 0).sum())
    assert 0 < strong_only and full > 2 * strong_only


def test_roundtrip_table_is_bfls_fp32_expression():
    literal = np.array([int(((torch.tensor(float(v)) / 127.5 - 1.0) + 1.0) * 127.5) for v in range(256)], np.uint8)
    want = np.array([v - 1 if 1 <= v <= 63 else v for v in range(256)], dtype=np.uint8)
    assert np.array_equal(literal, want)
    assert np.array_equal(control.ROUNDTRIP, want) and np.array_equal(control_ref.roundtrip_table(), want)
    assert control.ROUNDTRIP.dtype == np.uint8


def test_canny_control_image_goes_to_the_vae_as_minus_one_and_one():
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (32, 48, 3), dtype=np.uint8)
    c = control_ref.canny_control(img)
    assert c.shape == (32, 48, 3) and set(np.unique(c)) <= {0, 255}
    assert np.array_equal(c[..., 0], c[..., 2])
    x = torch.from_numpy(c).float() / 255 * 2 - 1.0
    assert set(torch.unique(x).tolist()) <= {-1.0, 1.0}


# ------------------------------------------------------------------------------------------------ control image
def test_control_image_loading():
    from PIL import Image

    rng = np.random.default_rng(4)
    rgb = rng.integers(0, 256, (40, 70, 3), dtype=np.uint8)
    got = control.load_control_image(rgb, (64, 32))
    want = np.asarray(Image.fromarray(rgb).resize((64, 32), Image.LANCZOS))
    assert got.shape == (32, 64, 3) and np.array_equal(got, want)
    grey = rng.integers(0, 256, (32, 64), dtype=np.uint8)
    g = control.load_control_image(grey, (64, 32))
    assert np.array_equal(g, np.repeat(grey[..., None], 3, axis=2))
    assert np.array_equal(control.load_control_image(grey[..., None], (64, 32)), g)
    rgba = np.concatenate([rgb, np.full((40, 70, 1), 9, np.uint8)], axis=2)
    assert np.array_equal(control.load_control_image(rgba, (70, 40)), rgb)
    assert np.array_equal(control.load_control_image(Image.fromarray(rgb), (70, 40)), rgb)
    for bad in (rgb.astype(np.float32), rng.integers(0, 256, (4, 4, 2), dtype=np.uint8), 3.0):
        with pytest.raises(ValueError, match="control_image"):
            control.load_control_image(bad, (64, 32))
    with pytest.raises(ValueError, match="could not be read"):
        control.load_control_image("/nonexistent/control.png", (64, 32))


# ------------------------------------------------------------------------------------------------ config and loader
def test_config_and_specs():
    assert FLUX_CANNY_DEV == replace(FLUX_DEV, x_embedder_cond_channels=64, control="canny")
    assert FLUX_DEPTH_DEV == replace(FLUX_DEV, x_embedder_cond_channels=64, control="depth")
    assert CONTROL_MODEL_CONFIGS == {CANNY: FLUX_CANNY_DEV, DEPTH: FLUX_DEPTH_DEV}
    for mv in (CANNY, DEPTH):
        assert T5_MAX_LENGTH[mv] == 512 and MMDIT_CKPT[mv] == mv and mv not in MODEL_CONFIGS
    assert all(c.control is None for c in MODEL_CONFIGS.values()) and FLUX_FILL_DEV.control is None
    plain, ctl = mmdit_param_specs(FLUX_DEV), mmdit_param_specs(FLUX_CANNY_DEV)
    assert len(plain) == len(ctl)
    for a, b in zip(plain, ctl):
        if a[0] == "x_embedder.proj.weight":
            assert a[1] == (3072, 1, 1, 64) and b[1] == (3072, 1, 1, 128)
        else:
            assert a == b
    assert control.DEFAULT_GUIDANCE == {"canny": 30.0, "depth": 10.0} and control.DEFAULT_THRESHOLDS == (50, 200)


def test_loader_takes_the_control_layout_and_refuses_mismatches():
    cfg, dev = tiny_control_config(), replace(tiny_flux_config(), guidance_embed=True)
    params = init_params(mmdit_param_specs(cfg), seed=5, dtype=torch.float32)
    sd = dev_upstream(params, cfg)
    assert tuple(sd["img_in.weight"].shape) == (cfg.hidden_size, 128)
    got = model_io.flux_checkpoint_to_params(sd, cfg.hidden_size, cfg.mlp_ratio, guidance_embed=True, cond_channels=64)
    model_io.check_against_specs(got, mmdit_param_specs(cfg))
    assert torch.equal(got["x_embedder.proj.weight"], params["x_embedder.proj.weight"])
    with pytest.raises(ValueError, match="img_in.weight.*128 input columns.*plain FLUX"):
        model_io.flux_checkpoint_to_params(sd, cfg.hidden_size, cfg.mlp_ratio, guidance_embed=True)
    plain_sd = dev_upstream(init_params(mmdit_param_specs(dev), seed=5, dtype=torch.float32), dev)
    with pytest.raises(ValueError, match="img_in.weight.*64 input columns.*Canny / Depth config takes 128"):
        model_io.flux_checkpoint_to_params(plain_sd, cfg.hidden_size, cfg.mlp_ratio, guidance_embed=True,
                                           cond_channels=64)


# ------------------------------------------------------------------------------------------------ argument checks
def _stub(cls, cfg):
    """a pipeline object with only its config: the checks below run before any model or GPU work"""
    p = object.__new__(cls)
    p.config = cfg
    return p


def test_argument_errors_before_gpu_work():
    img = np.zeros((64, 64, 3), np.uint8)
    canny = _stub(FluxPipeline, tiny_control_config("canny"))
    depth = _stub(FluxPipeline, tiny_control_config("depth"))
    dflt = control.DEFAULT_THRESHOLDS
    for pipe, kw, msg in [
            (canny, dict(control_image=None), "Canny needs control_image"),
            (depth, dict(control_image=None), "Depth needs control_image"),
            (canny, dict(control_image=img, reference_image=img), "Kontext"),
            (depth, dict(control_image=img, reference_latents=torch.zeros(1, 8, 8, 16)), "Kontext"),
            (canny, dict(control_image=img, canny_thresholds=(200, 50)), "0 <= low <= high"),
            (canny, dict(control_image=img, canny_thresholds=(-1, 50)), "0 <= low <= high"),
            (canny, dict(control_image=img, canny_thresholds=(50.5, 200)), "integers"),
            (canny, dict(control_image=img, canny_thresholds=50), r"\(low, high\)"),
            (depth, dict(control_image=img, canny_thresholds=None), "Canny model only"),
            (_stub(FluxPipeline, replace(tiny_control_config(), x_embedder_cond_channels=320)),
             dict(control_image=img), "64 conditioning channels"),
            (_stub(FluxPipeline, replace(tiny_control_config(), control="pose")), dict(control_image=img),
             "config.control"),
            (_stub(DiffusionPipeline, tiny_control_config()), dict(control_image=img), "FluxPipeline only"),
            (_stub(FluxPipeline, replace(tiny_flux_config(), guidance_embed=True)), dict(control_image=img),
             "has none"),
            (_stub(FluxPipeline, FLUX_FILL_DEV), dict(control_image=img), "has none"),
            (_stub(FluxPipeline, tiny_flux_config()), dict(canny_thresholds=(10, 20)), "Canny model only")]:
        kw = {"control_image": None, "canny_thresholds": dflt, "reference_image": None, "reference_latents": None,
              **kw}
        with pytest.raises(ValueError, match=msg):
            pipe._check_control(**kw)
    assert canny._check_control(img, dflt, None, None) == (50, 200)
    assert canny._check_control(img, (0, 0), None, None) == (0, 0)
    assert canny._check_control(img, None, None, None) is None
    assert depth._check_control(img, dflt, None, None) is None
    assert _stub(FluxPipeline, tiny_flux_config())._check_control(None, dflt, None, None) is None
    # a control model's Fill check has nothing to say, and the control check runs in denoise_latents before any GPU
    # work: an unreadable control image, and a missing one, raise from a pipeline that has no model or device
    canny._check_fill(None, None, None, None)
    with pytest.raises(ValueError, match="could not be read"):
        canny.denoise_latents(None, None, control_image="/nonexistent/control.png")
    with pytest.raises(ValueError, match="needs control_image"):
        canny.generate_image("", verbose=False)
    with pytest.raises(ValueError, match="has none"):
        _stub(FluxPipeline, tiny_flux_config()).denoise_latents(None, None, control_image=img)


def test_guidance_defaults():
    assert _stub(FluxPipeline, tiny_control_config("canny"))._guidance_values(None, 2) == [30.0, 30.0]
    assert _stub(FluxPipeline, tiny_control_config("depth"))._guidance_values(None, 1) == [10.0]
    assert _stub(FluxPipeline, tiny_control_config("depth"))._guidance_values(4.0, 1) == [4.0]
    assert _stub(FluxPipeline, replace(tiny_flux_config(), guidance_embed=True,
                                       x_embedder_cond_channels=320))._guidance_values(None, 1) == [30.0]
    assert _stub(FluxPipeline, replace(tiny_flux_config(), guidance_embed=True))._guidance_values(None, 1) == \
        [DEFAULT_GUIDANCE] == [3.5]


# ------------------------------------------------------------------------------------------------ packing
@pytest.mark.parametrize("H, W", [(2, 2), (8, 16), (12, 6)])
def test_control_rows_packing_is_the_index_formula(H, W):
    lat = torch.randn((1, H, W, 16), generator=torch.Generator().manual_seed(H * W))
    got = bfl_pack_latent(lat)[0].numpy()
    assert got.shape == ((H // 2) * (W // 2), 64)
    assert np.array_equal(got, control_ref.loop_pack(lat[0].numpy()))
