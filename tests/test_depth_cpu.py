"""CPU checks of FLUX.1 Depth's depth estimator (DESIGN.md §20): the fp32 oracle on the engine's packed tree against
transformers' DepthAnythingForDepthEstimation, the folds and the ConvTranspose / stride-2 geometry in fp64, every tap
table against torch.nn.functional.interpolate, the preprocessing against the DPT image processor and PIL, the config
reader, the loader's refusals and the pipeline's argument errors."""
from dataclasses import replace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from diffusionkit_b200 import DkError, FluxPipeline, DiffusionPipeline, control, depth, model_io
from diffusionkit_b200.config import DEPTH_ANYTHING_LARGE, FLUX_FILL_DEV, tiny_depth_anything_config
from tests.depth_ref import DepthAnythingRef, unfold_slabs

LARGE4 = replace(DEPTH_ANYTHING_LARGE, num_hidden_layers=4, out_indices=(1, 2, 3, 4))


def hf_model(cfg, seed=3):
    """transformers' DepthAnythingForDepthEstimation of cfg with the repo initialiser's conditioned weights, and its
    state_dict (mask_token and the unused residual unit included, as a real checkpoint holds them)"""
    transformers = pytest.importorskip("transformers")
    from diffusionkit_b200.weights import init_params

    bc = transformers.Dinov2Config(hidden_size=cfg.hidden_size, num_hidden_layers=cfg.num_hidden_layers,
                                   num_attention_heads=cfg.num_attention_heads,
                                   mlp_ratio=cfg.intermediate_size // cfg.hidden_size, image_size=cfg.image_size,
                                   patch_size=cfg.patch_size, out_indices=list(cfg.out_indices),
                                   reshape_hidden_states=False)
    hc = transformers.DepthAnythingConfig(backbone_config=bc, neck_hidden_sizes=list(cfg.neck_hidden_sizes),
                                          reassemble_factors=list(cfg.reassemble_factors),
                                          fusion_hidden_size=cfg.fusion_hidden_size,
                                          head_hidden_size=cfg.head_hidden_size, reassemble_hidden_size=cfg.hidden_size)
    torch.manual_seed(seed)
    m = transformers.DepthAnythingForDepthEstimation(hc).eval()
    sd = dict(m.state_dict())
    sd.update(init_params(depth.depth_param_specs(cfg), seed=seed, dtype=torch.float32))
    depth.condition_depth_params(sd, cfg)
    m.load_state_dict(sd)
    return m, sd


def processor_pixels(img_u8: np.ndarray) -> torch.Tensor:
    x = torch.from_numpy(img_u8).float() / 255
    x = (x - torch.tensor(depth.IMAGENET_MEAN)) / torch.tensor(depth.IMAGENET_STD)
    return x.permute(2, 0, 1)[None]


@pytest.mark.parametrize("cfg, size", [(tiny_depth_anything_config(), (518, 518)),
                                       (tiny_depth_anything_config(), (518, 686)),
                                       (LARGE4, (518, 518))], ids=["tiny-518", "tiny-518x686", "large-width-4-layers"])
def test_oracle_equals_transformers(cfg, size):
    m, sd = hf_model(cfg)
    cfg_engine = cfg
    params = model_io.depth_anything_checkpoint_to_params(sd, cfg_engine)
    img = np.random.default_rng(1).integers(0, 256, (*size, 3), dtype=np.uint8)
    with torch.no_grad():
        want = m(pixel_values=processor_pixels(img)).predicted_depth[0]
        got = DepthAnythingRef(params, cfg_engine)(torch.from_numpy(img))
    r = float((got - want).norm() / want.norm())
    print(f"{cfg.hidden_size} wide {size}: rel_l2 {r:.2e}, depth {float(want.min()):.1f} .. {float(want.max()):.1f}")
    assert r <= 1e-5
    # the conditioned weights give a real spread: BFL's depth / 127.5 - 1 spans a good part of [-1, 1]
    v = want / 127.5 - 1
    assert float(v.max() - v.min()) > 0.5 and float(want.std()) > 10.0


# ------------------------------------------------------------------------------------------------ fp64 identities
def test_folds_in_fp64():
    g = torch.Generator().manual_seed(0)
    D, K = 16, 24
    W, b, lam = (torch.randn(D, K, generator=g, dtype=torch.float64), torch.randn(D, generator=g, dtype=torch.float64),
                 torch.randn(D, generator=g, dtype=torch.float64))
    x = torch.randn(5, K, generator=g, dtype=torch.float64)
    w2, b2 = depth.fold_layer_scale(W, b, lam)
    assert torch.allclose(lam * (x @ W.T + b), x @ w2.T + b2, rtol=1e-12, atol=1e-12)
    Wp, bp = torch.randn(D, 3, 14, 14, generator=g, dtype=torch.float64), torch.randn(D, generator=g, dtype=torch.float64)
    u8 = torch.randint(0, 256, (2, 3, 28, 42), generator=g).double()
    mu = torch.tensor(depth.IMAGENET_MEAN, dtype=torch.float64)[None, :, None, None]
    sd = torch.tensor(depth.IMAGENET_STD, dtype=torch.float64)[None, :, None, None]
    want = F.conv2d((u8 / 255 - mu) / sd, Wp, bp, stride=14)
    w2, b2 = depth.fold_imagenet(Wp, bp)
    got = F.conv2d(u8 / 255 * 2 - 1, w2, b2, stride=14)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-10)


@pytest.mark.parametrize("s, gh, gw", [(4, 3, 5), (2, 37, 37), (2, 37, 49)])
def test_conv_transpose_row_map_in_fp64(s, gh, gw):
    """the s GEMMs of the engine: slab di maps input row y * gw + x to output row y * s gw + di gw + x of the (s gh s gw,
    s O)-shaped view (rows_per_batch gw, out_batch_rows s gw, out_row_off di gw, ldc s O)"""
    g = torch.Generator().manual_seed(s)
    I, O = 8, 6
    W, b = torch.randn(I, O, s, s, generator=g, dtype=torch.float64), torch.randn(O, generator=g, dtype=torch.float64)
    x = torch.randn(1, I, gh, gw, generator=g, dtype=torch.float64)
    want = F.conv_transpose2d(x, W, b, stride=s)[0].permute(1, 2, 0)          # (s gh, s gw, O)
    slabs, brep = depth.conv_transpose_slabs(W, b)
    assert torch.equal(unfold_slabs(slabs), W)
    A = x[0].permute(1, 2, 0).reshape(gh * gw, I)
    out = torch.full((s * gh * gw, s * O), float("nan"), dtype=torch.float64)
    for di in range(s):
        res = A @ slabs[di].T + brep                                           # (gh gw, s O)
        for m in range(gh * gw):
            out[(m // gw) * s * gw + di * gw + m % gw] = res[m]
    assert torch.allclose(out.reshape(s * gh, s * gw, O), want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("H, W", [(37, 37), (37, 49), (8, 8), (5, 7)])
def test_stride2_pad1_geometry_in_fp64(H, W):
    """output (ceil(H/2), ceil(W/2)); output (y, x) reads rows 2y - 1 .. 2y + 1 and columns 2x - 1 .. 2x + 1, zero
    outside, which is what the TMA tap coordinates y0 * 2 + dy - 1 of dk_conv3x3_s2_p1 load"""
    g = torch.Generator().manual_seed(H * W)
    x = torch.randn(1, 4, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(3, 4, 3, 3, generator=g, dtype=torch.float64)
    want = F.conv2d(x, w, stride=2, padding=1)
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    assert want.shape[2:] == (Ho, Wo)
    got = torch.zeros(1, 3, Ho, Wo, dtype=torch.float64)
    for y in range(Ho):
        for xx in range(Wo):
            for dy in range(3):
                for dx in range(3):
                    iy, ix = 2 * y + dy - 1, 2 * xx + dx - 1
                    if 0 <= iy < H and 0 <= ix < W:
                        got[0, :, y, xx] += w[:, :, dy, dx] @ x[0, :, iy, ix]
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)


def _apply(first, wts, x, axis_len):
    M = torch.zeros((len(first), axis_len), dtype=torch.float64)
    for o, (i0, ws) in enumerate(zip(first, wts)):
        for t, w in enumerate(ws):
            assert 0 <= i0 + t < axis_len
            M[o, i0 + t] += w
    return M


@pytest.mark.parametrize("kind, n_in, n_out", [
    ("bilinear_ac", 19, 37), ("bilinear_ac", 148, 296), ("bilinear_ac", 296, 518), ("bilinear_ac", 37, 74),
    ("bilinear", 19, 37), ("bilinear", 37, 74), ("bilinear", 74, 37), ("bicubic", 37, 18), ("bicubic", 37, 49),
    ("bicubic", 37, 74), ("bicubic_aa", 518, 1024), ("bicubic_aa", 686, 1024), ("bicubic_aa", 1024, 518),
    ("bicubic_aa", 37, 64), ("bicubic_aa", 252, 64), ("bicubic_aa", 518, 768)])
def test_tap_tables_equal_interpolate(kind, n_in, n_out):
    first, wts = depth.TAPS[kind](n_in, n_out)
    M = _apply(first, wts, None, n_in)
    x = torch.randn(1, 1, 3, n_in, dtype=torch.float64, generator=torch.Generator().manual_seed(n_in))
    mode = {"bilinear": "bilinear", "bilinear_ac": "bilinear", "bicubic": "bicubic", "bicubic_aa": "bicubic"}[kind]
    kw = dict(align_corners=kind == "bilinear_ac") if kind != "bicubic_aa" else dict(align_corners=False,
                                                                                      antialias=True)
    want = F.interpolate(x, size=(3, n_out), mode=mode, **kw)[0, 0]
    got = x[0, 0] @ M.T
    assert torch.allclose(got, want, rtol=1e-10, atol=1e-10), float((got - want).abs().max())


# ------------------------------------------------------------------------------------------------ preprocessing
@pytest.mark.parametrize("h, w", [(1024, 1024), (768, 1024), (1024, 768), (512, 1536), (64, 128), (333, 517),
                                  (1080, 1920)])
def test_network_size_equals_the_dpt_processor(h, w):
    transformers = pytest.importorskip("transformers")
    from transformers.models.dpt.image_processing_dpt import get_resize_output_image_size

    img = torch.zeros((3, h, w))                                 # channels first, as the processor passes it
    want = get_resize_output_image_size(img, output_size=(518, 518), keep_aspect_ratio=True, multiple=14)
    assert depth.network_size(h, w) == (want.height, want.width)
    assert transformers is not None
    if (h, w) == (1024, 1024):
        assert depth.network_size(h, w) == (518, 518)
    if (h, w) == (768, 1024):
        assert depth.network_size(h, w) == (518, 686)


def test_network_input_equals_pil_and_the_processor():
    from PIL import Image

    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, (300, 410, 3), dtype=np.uint8)
    got = depth.network_input(img)
    h, w = depth.network_size(300, 410)
    want = np.asarray(Image.fromarray(control.ROUNDTRIP[img]).resize((w, h), Image.BICUBIC))
    assert got.shape == (h, w, 3) and np.array_equal(got, want)
    transformers = pytest.importorskip("transformers")
    try:
        proc = transformers.DPTImageProcessorPil(size={"height": 518, "width": 518}, keep_aspect_ratio=True,
                                              ensure_multiple_of=14, do_pad=False, resample=Image.BICUBIC,
                                              image_mean=list(depth.IMAGENET_MEAN), image_std=list(depth.IMAGENET_STD))
        pix = proc(Image.fromarray(control.ROUNDTRIP[img]), return_tensors="pt")["pixel_values"][0]
    except (AttributeError, ImportError) as e:                # a transformers without the PIL processor
        pytest.skip(f"DPTImageProcessorPil unavailable: {e}")
    assert tuple(pix.shape[1:]) == (h, w)
    mine = processor_pixels(got)[0]
    assert float((mine - pix).abs().max()) < 1e-5


# ------------------------------------------------------------------------------------------------ config and loader
def test_depth_anything_config_from_json():
    cj = {"backbone_config": {"hidden_size": 1024, "num_attention_heads": 16, "num_hidden_layers": 24,
                              "mlp_ratio": 4, "patch_size": 14, "image_size": 518, "layer_norm_eps": 1e-6,
                              "out_indices": [21, 22, 23, 24], "model_type": "dinov2"},
          "neck_hidden_sizes": [256, 512, 1024, 1024], "reassemble_factors": [4, 2, 1, 0.5],
          "fusion_hidden_size": 256, "head_hidden_size": 32, "depth_estimation_type": "relative",
          "reassemble_hidden_size": 1024, "model_type": "depth_anything"}
    assert model_io.depth_anything_config(cj) == DEPTH_ANYTHING_LARGE
    cj["backbone_config"].pop("out_indices")
    cj["backbone_config"]["out_features"] = ["stage9", "stage10", "stage11", "stage12"]
    assert model_io.depth_anything_config(cj).out_indices == (9, 10, 11, 12)


def test_loader_refusals():
    cfg = tiny_depth_anything_config()
    sd = {n: torch.zeros(s) for n, s, _ in depth.depth_param_specs(cfg)}
    sd["backbone.embeddings.mask_token"] = torch.zeros(1, cfg.hidden_size)
    for u in (1, 2):
        sd[f"neck.fusion_stage.layers.0.residual_layer1.convolution{u}.weight"] = torch.zeros(128, 128, 3, 3)
    params = model_io.depth_anything_checkpoint_to_params(sd, cfg)
    assert {k: tuple(v.shape) for k, v in params.items()} == depth.engine_depth_shapes(cfg)
    bad = dict(sd)
    del bad["head.conv3.bias"]
    with pytest.raises(ValueError, match="missing head.conv3.bias"):
        model_io.depth_anything_checkpoint_to_params(bad, cfg)
    bad = dict(sd, **{"head.extra": torch.zeros(1)})
    with pytest.raises(ValueError, match="unexpected keys.*head.extra"):
        model_io.depth_anything_checkpoint_to_params(bad, cfg)
    bad = dict(sd, **{"neck.convs.0.weight": torch.zeros(128, 64, 1, 1)})
    with pytest.raises(ValueError, match="neck.convs.0.weight has shape"):
        model_io.depth_anything_checkpoint_to_params(bad, cfg)
    for c, msg in [(replace(cfg, depth_estimation_type="metric"), "relative"),
                   (replace(cfg, num_attention_heads=4), "head dim must be 64"),
                   (replace(cfg, neck_hidden_sizes=(48, 96, 192, 384)), "multiple of 64"),
                   (replace(cfg, fusion_hidden_size=64), "multiple of 64")]:
        with pytest.raises(ValueError, match=msg):
            model_io.depth_anything_checkpoint_to_params(sd, c)
    assert DEPTH_ANYTHING_LARGE.head_dim == 64
    depth.check_config(DEPTH_ANYTHING_LARGE)


# ------------------------------------------------------------------------------------------------ argument checks
def _stub(cls, cfg, **attrs):
    p = object.__new__(cls)
    p.config = cfg
    p.__dict__.update(attrs)
    return p


def test_pipeline_argument_errors_before_gpu_work():
    from tests.test_control_cpu import tiny_control_config
    from diffusionkit_b200.config import tiny_flux_config

    img = np.zeros((64, 64, 3), np.uint8)
    dflt = control.DEFAULT_THRESHOLDS
    ready = _stub(FluxPipeline, tiny_control_config("depth"), depth_estimator=object())
    for pipe, kw, exc, msg in [
            (_stub(FluxPipeline, tiny_control_config("canny"), depth_estimator=object()), {}, ValueError,
             "FLUX.1 Depth model"),
            (_stub(FluxPipeline, replace(tiny_flux_config(), guidance_embed=True)), {}, ValueError, "FLUX.1 Depth"),
            (_stub(FluxPipeline, FLUX_FILL_DEV), {}, ValueError, "FLUX.1 Depth"),
            (_stub(DiffusionPipeline, tiny_control_config("depth")), {}, ValueError, "FluxPipeline only"),
            (ready, dict(control_image=None), ValueError, "needs control_image"),
            (_stub(FluxPipeline, tiny_control_config("depth")), {}, DkError, "load_depth_estimator")]:
        kw = {"control_image": img, "canny_thresholds": dflt, "reference_image": None, "reference_latents": None,
              "estimate_depth": True, **kw}
        with pytest.raises(exc, match=msg):
            pipe._check_control(**kw)
    assert ready._check_control(img, dflt, None, None, True) is None
    # without estimate_depth nothing about the estimator is asked
    assert _stub(FluxPipeline, tiny_control_config("depth"))._check_control(img, dflt, None, None) is None
    with pytest.raises(DkError, match="load_depth_estimator"):
        _stub(FluxPipeline, tiny_control_config("depth")).estimate_depth(img)
