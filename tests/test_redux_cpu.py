"""CPU: FLUX.1 Redux image prompts (DESIGN.md §15) — the SigLIP oracle (tests/redux_ref.py) against transformers'
SiglipVisionModel through the checkpoint loader, the exactness of the head and patch-weight padding, the host resize,
tanh-GELU and the projector against their upstream definitions, and the pipeline's argument checks."""
import inspect
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from diffusionkit_b200 import model_io
from diffusionkit_b200._lib import DkError
from diffusionkit_b200.config import SIGLIP_SO400M_PATCH14_384, SiglipVisionConfig, tiny_siglip_config
from diffusionkit_b200.image_encoders import (pack_siglip_params, padded_head_dim, patch_weight_kp, redux_param_specs,
                                              siglip_param_specs)
from diffusionkit_b200.pipeline import DiffusionPipeline, FluxPipeline
from diffusionkit_b200.weights import init_params
from tests.model_checks import _test_image
from tests.redux_ref import SiglipVisionRef, gelu_tanh, redux_project, ref_image_patches

transformers = pytest.importorskip("transformers")


def _hf_model(cfg: SiglipVisionConfig, seed=0):
    """transformers' SiglipVisionModel built from a config (no download), every parameter redrawn at random"""
    hc = transformers.SiglipVisionConfig(
        hidden_size=cfg.hidden_size, num_attention_heads=cfg.num_attention_heads, num_hidden_layers=cfg.num_hidden_layers,
        intermediate_size=cfg.intermediate_size, patch_size=cfg.patch_size, image_size=cfg.image_size,
        layer_norm_eps=cfg.layer_norm_eps, hidden_act="gelu_pytorch_tanh", num_channels=3)
    m = transformers.SiglipVisionModel(hc).eval()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, t in m.named_parameters():
            if t.dim() == 1:
                t.copy_((1.0 if "norm" in name and name.endswith("weight") else 0.0) + 0.05 * torch.randn(t.shape, generator=g))
            else:
                t.copy_(torch.randn(t.shape, generator=g) / t[0].numel() ** 0.5)
    return m


def _siglip_model_file(m):
    """a SiglipModel-style state dict: the vision tower (with its pooling head) beside a text tower and the logits"""
    sd = {k if k.startswith("vision_model.") else "vision_model." + k: v for k, v in m.state_dict().items()}
    assert any(k.startswith("vision_model.head.") for k in sd)
    sd["text_model.embeddings.token_embedding.weight"] = torch.zeros(8, 4)
    sd["text_model.final_layer_norm.weight"] = torch.ones(4)
    sd["logit_scale"], sd["logit_bias"] = torch.ones(1), torch.zeros(1)
    return sd


def _hf_last_hidden(m, img_u8):
    px = img_u8.permute(0, 3, 1, 2).float() / 255 * 2 - 1.0          # the processor's (x / 255 - 0.5) / 0.5
    with torch.no_grad():
        return m(pixel_values=px).last_hidden_state


@pytest.mark.parametrize("cfg", [tiny_siglip_config(), tiny_siglip_config(image_size=100),
                                 SiglipVisionConfig(num_hidden_layers=1)],
                         ids=["tiny-98", "tiny-100-ragged", "so400m-width-1-layer"])
def test_oracle_equals_transformers_through_the_loader(cfg):
    m = _hf_model(cfg)
    params = model_io.siglip_checkpoint_to_params(_siglip_model_file(m), cfg)
    g = torch.Generator().manual_seed(3)
    img = torch.randint(0, 256, (2, cfg.image_size, cfg.image_size, 3), generator=g, dtype=torch.uint8)
    want = _hf_last_hidden(m, img)
    got = SiglipVisionRef(params, cfg)(img)
    assert got.shape == want.shape == (2, cfg.num_patches, cfg.hidden_size)
    err = float((got - want).norm() / want.norm())
    assert err <= 1e-5, err
    # a vision-only export, without the `vision_model.` prefix, loads to the same tree
    bare = model_io.siglip_checkpoint_to_params({k: v for k, v in m.state_dict().items()}, cfg)
    assert bare.keys() == params.keys() and all(torch.equal(bare[k], params[k]) for k in params)


def test_real_preset():
    c = SIGLIP_SO400M_PATCH14_384
    assert (c.hidden_size, c.num_attention_heads, c.intermediate_size, c.num_hidden_layers) == (1152, 16, 4304, 27)
    assert (c.patch_size, c.image_size, c.layer_norm_eps, c.head_dim, c.num_patches) == (14, 384, 1e-6, 72, 729)
    assert patch_weight_kp(c) == 592 and padded_head_dim(c) == 128
    assert padded_head_dim(SiglipVisionConfig(hidden_size=128, num_attention_heads=2)) == 64
    for bad in (SiglipVisionConfig(hidden_size=160, num_attention_heads=2),     # head dim 80
                SiglipVisionConfig(hidden_size=1150, num_attention_heads=16)):  # not heads x head_dim
        with pytest.raises(ValueError):
            padded_head_dim(bad)


def test_loader_names_a_missing_or_misshaped_key():
    cfg = tiny_siglip_config()
    sd = _siglip_model_file(_hf_model(cfg))
    for key in ("vision_model.encoder.layers.1.mlp.fc2.bias", "vision_model.embeddings.patch_embedding.weight"):
        bad = dict(sd)
        del bad[key]
        with pytest.raises(ValueError, match=key.replace(".", r"\.")):
            model_io.siglip_checkpoint_to_params(bad, cfg)
        bad = dict(sd)
        bad[key] = torch.zeros(3)
        with pytest.raises(ValueError, match=key.replace(".", r"\.")):
            model_io.siglip_checkpoint_to_params(bad, cfg)
    with pytest.raises(ValueError, match="unexpected"):
        model_io.siglip_checkpoint_to_params({**sd, "vision_model.encoder.layers.9.mlp.fc1.bias": torch.zeros(3)}, cfg)

    rsd = {n: torch.zeros(s) for n, s, _ in redux_param_specs(1152, 4096)}
    assert set(model_io.redux_checkpoint_to_params(rsd)) == set(rsd)
    for key in rsd:
        bad = dict(rsd)
        del bad[key]
        with pytest.raises(ValueError, match=key.replace(".", r"\.")):
            model_io.redux_checkpoint_to_params(bad)
    with pytest.raises(ValueError, match=r"redux_down\.weight"):          # a 3072-wide projector for a 4096 FLUX
        model_io.redux_checkpoint_to_params({**rsd, "redux_down.weight": torch.zeros(3072, 12288)})
    small = {n: torch.zeros(s) for n, s, _ in redux_param_specs(144, 128)}
    assert set(model_io.redux_checkpoint_to_params(small, token_level_text_embed_dim=128, siglip_hidden=144)) == set(small)


def test_padding_is_exact_in_fp64():
    """the zero-padded heads (72 -> 128) give the unpadded attention, and the permuted, K-padded patch weight gives the
    stride-14 Conv2d, to fp64 rounding"""
    cfg = SiglipVisionConfig(num_hidden_layers=1)
    D, H, d, dp = cfg.hidden_size, cfg.num_attention_heads, cfg.head_dim, padded_head_dim(cfg)
    up = init_params(siglip_param_specs(cfg), seed=2, dtype=torch.float64)
    for k in up:
        if k.endswith("bias"):
            up[k] = up[k] * 10                                           # biases that matter
    packed = pack_siglip_params(up, cfg)
    g = torch.Generator().manual_seed(1)
    x = torch.randn((2, 50, D), generator=g, dtype=torch.float64)
    a = "encoder.layers.0.self_attn."

    def heads(t, dd):
        return t.reshape(2, 50, H, dd).transpose(1, 2)

    q, k, v = (heads(x @ up[a + n + "_proj.weight"].t() + up[a + n + "_proj.bias"], d) for n in "qkv")
    o = (torch.softmax(q @ k.transpose(-1, -2) * d ** -0.5, -1) @ v).transpose(1, 2).reshape(2, 50, D)
    want = o @ up[a + "out_proj.weight"].t()
    qkv = x @ packed[a + "qkv_proj.weight"].t() + packed[a + "qkv_proj.bias"]
    qp, kp_, vp = (heads(t, dp) for t in qkv.split(H * dp, dim=-1))
    op = (torch.softmax(qp @ kp_.transpose(-1, -2) * d ** -0.5, -1) @ vp).transpose(1, 2).reshape(2, 50, H * dp)
    got = op @ packed[a + "out_proj.weight"].t()
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())

    img = torch.randint(0, 256, (2, 384, 384, 3), generator=g, dtype=torch.uint8)
    w = up["embeddings.patch_embedding.weight"]
    x = (img.permute(0, 3, 1, 2).float() / 255 * 2 - 1.0).double()          # the fp32 normalisation the kernel rounds
    conv = F.conv2d(x, w, stride=14)                                          # (2, D, 27, 27)
    want = conv.permute(0, 2, 3, 1).reshape(-1, D)
    got = ref_image_patches(img, torch.float32, 14, patch_weight_kp(cfg)).double() @ packed["embeddings.patch_embedding.weight"].t()
    assert got.shape == (2 * 729, D)
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())


def _host_pipe(image_size=384):
    """a FluxPipeline shell with just what the host-side Redux checks read (no GPU)"""
    p = object.__new__(FluxPipeline)
    p.siglip = SimpleNamespace(config=SiglipVisionConfig(image_size=image_size))
    p.redux = object()
    return p


def test_host_resize_is_pil_bicubic_and_matches_the_processor():
    from PIL import Image

    pipe = _host_pipe()
    src = _test_image(300, 500, seed=4)
    got = pipe._redux_image_u8(src)
    want = np.asarray(Image.fromarray(src).resize((384, 384), Image.BICUBIC, reducing_gap=None))
    assert got.shape == (384, 384, 3) and got.dtype == np.uint8 and np.array_equal(got, want)
    assert np.array_equal(pipe._redux_image_u8(Image.fromarray(src)), want)
    grey = pipe._redux_image_u8(src[:, :, 0])                                   # greyscale and RGBA are converted
    assert grey.shape == (384, 384, 3) and np.array_equal(grey[..., 0], grey[..., 2])
    rgba = np.concatenate([src, np.full(src.shape[:2] + (1,), 255, np.uint8)], axis=2)
    assert np.array_equal(pipe._redux_image_u8(rgba), want)
    # the installed processor resizes with another bicubic implementation: one 8-bit level apart on a fraction of a
    # percent of the values of a downscaled photo-like image (upscaling also shows a few values two levels apart)
    proc = transformers.SiglipImageProcessor(size={"height": 384, "width": 384})
    big = _test_image(1024, 768, seed=2)
    px = proc(images=Image.fromarray(big), return_tensors="pt")["pixel_values"][0].permute(1, 2, 0).float()
    d = (px - torch.from_numpy(pipe._redux_image_u8(big)).float() / 255 * 2 + 1.0).abs()
    assert float(d.max()) <= 1 / 127.5 + 1e-6 and float((d > 1e-6).float().mean()) <= 0.01
    for bad in (np.zeros((8, 8, 2), np.uint8), np.zeros((8, 8, 3), np.float32)):
        with pytest.raises(ValueError):
            pipe._redux_image_u8(bad)


def test_tanh_gelu_and_projector_match_their_definitions():
    from transformers.activations import ACT2FN

    x = torch.linspace(-12, 12, 100001)
    want = F.gelu(x, approximate="tanh")
    assert float((gelu_tanh(x) - want).abs().max()) <= 1e-6
    assert float((ACT2FN["gelu_pytorch_tanh"](x) - want).abs().max()) <= 1e-6
    from diffusionkit_b200._lib import ACT_GELU_TANH, ACT_SILU
    from tests import kernel_checks as kc
    from tests.redux_ref import with_gelu_tanh

    g = torch.Generator().manual_seed(2)
    A, W, b = torch.randn(40, 24, generator=g), torch.randn(32, 24, generator=g), torch.randn(32, generator=g)
    ref = with_gelu_tanh(kc.ref_gemm)
    assert torch.allclose(ref(A, W, b, ACT_GELU_TANH), F.gelu(A @ W.t() + b, approximate="tanh"), atol=1e-5)
    assert torch.equal(ref(A, W, b, ACT_SILU), kc.ref_gemm(A, W, b, ACT_SILU))

    class ReduxImageEncoder(torch.nn.Module):              # BFL flux/modules/image_embedders.py, written out
        def __init__(self, redux_dim: int = 1152, txt_in_features: int = 4096):
            super().__init__()
            self.redux_up = torch.nn.Linear(redux_dim, txt_in_features * 3)
            self.redux_down = torch.nn.Linear(txt_in_features * 3, txt_in_features)

        def forward(self, sigclip_embeds):
            return self.redux_down(F.silu(self.redux_up(sigclip_embeds)))

    torch.manual_seed(0)
    bfl = ReduxImageEncoder(144, 128)
    x = torch.randn(2, 49, 144)
    with torch.no_grad():
        want = bfl(x)
    got = redux_project(dict(bfl.state_dict()), x)
    assert float((got - want).norm() / want.norm()) <= 1e-6


def test_argument_checks_come_before_any_gpu_work():
    pipe = _host_pipe()
    img = np.zeros((64, 64, 3), np.uint8)
    assert pipe._redux_input(None, 0.0, 2) is None
    with pytest.raises(ValueError, match="cfg_weight"):
        pipe._redux_input(img, 1.5, 1)
    with pytest.raises(ValueError, match="one per seed"):
        pipe._redux_input([img, img, img], 0.0, 2)
    with pytest.raises(ValueError, match="one per seed"):
        pipe._redux_input([img], 0.0, 2)
    assert len(pipe._redux_input(img, 0.0, 3)) == 1 and len(pipe._redux_input([img, img], 0.0, 2)) == 2
    bare = object.__new__(FluxPipeline)
    with pytest.raises(DkError, match="load_redux"):
        bare._redux_input(img, 0.0, 1)
    with pytest.raises(DkError, match="load_redux"):
        bare.encode_redux(img)
    for fn in (FluxPipeline.generate_image, FluxPipeline.denoise_latents):
        assert inspect.signature(fn).parameters["redux_image"].kind is inspect.Parameter.KEYWORD_ONLY
    for fn in (DiffusionPipeline.generate_image, DiffusionPipeline.denoise_latents):
        assert "redux_image" not in inspect.signature(fn).parameters
