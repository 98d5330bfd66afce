"""FP8 linears, the parts that need no GPU: the reference quantiser's known answers, the fake-quantised oracle, and
which linears each model family covers."""
import torch

from diffusionkit_b200.config import MODEL_CONFIGS, tiny_flux_config, tiny_sd3_config, tiny_sd35_config
from diffusionkit_b200.mmdit import fp8_covered_linears
from diffusionkit_b200.weights import init_params, mmdit_param_specs
from oracle.mmdit_ref import MMDiTRef
from tests.fp8_ref import FakeQuantMMDiTRef, fake_quantize_rows, quantize_rows_e4m3
from tests.oracle_bridge import ref_config


def test_zero_row_has_scale_one():
    q, s = quantize_rows_e4m3(torch.zeros(2, 16))
    assert s.tolist() == [1.0, 1.0] and float(q.abs().max()) == 0.0


def test_power_of_two_maximum_is_exact():
    for k in (-9, 0, 7):
        x = torch.tensor([[448.0 * 2.0 ** k, -224.0 * 2.0 ** k, 2.0 ** k, 0.0]])
        q, s = quantize_rows_e4m3(x)
        assert float(s) == 2.0 ** k
        assert q.tolist() == [[448.0, -224.0, 1.0, 0.0]]


def test_subnormals_round_to_nearest_even():
    # with scale 1 (maximum 448) the e4m3 subnormals are multiples of 2^-9; ties go to the even multiple
    u = 2.0 ** -9
    x = torch.tensor([[448.0, 0.5 * u, 1.5 * u, 2.5 * u, 0.49 * u, -3.2 * u, 7.0 * u, 8.0 * u]])
    q, s = quantize_rows_e4m3(x)
    assert float(s) == 1.0
    assert q[0, 1:].tolist() == [0.0, 2 * u, 2 * u, 0.0, -3 * u, 7 * u, 8 * u]


def test_saturation_is_finite():
    # the division can land a hair above 448; satfinite keeps it at 448 and never makes a NaN
    x = torch.tensor([[3.0000002, -3.0, 1e-3], [65504.0, -65504.0, 1.0]])
    q, s = quantize_rows_e4m3(x)
    assert bool(torch.isfinite(q).all()) and float(q.abs().max()) == 448.0
    assert q[:, 0].tolist() == [448.0, 448.0] and q[:, 1].tolist() == [-448.0, -448.0]
    back = fake_quantize_rows(x)
    assert float((back - x).abs()[:, :2].max()) <= 1e-3 * 65504.0


def test_quantisation_error_is_within_half_an_ulp():
    g = torch.Generator().manual_seed(0)
    x = torch.randn((33, 256), generator=g)
    q, s = quantize_rows_e4m3(x)
    y = x / s[:, None]
    ulp = torch.maximum(torch.floor(torch.log2(y.abs().clamp_min(2.0 ** -6))), torch.tensor(-6.0)).exp2() * 2.0 ** -3
    assert bool(((q - y).abs() <= 0.5 * ulp * (1 + 1e-6)).all())


def _tiny_case(cfg, covered):
    p = {k: v.float() for k, v in init_params(mmdit_param_specs(cfg), seed=7, dtype=torch.bfloat16).items()}
    g = torch.Generator().manual_seed(5)
    latent = torch.randn((1, 4, 4, 16), generator=g)
    text = torch.randn((1, 8, cfg.token_level_text_embed_dim), generator=g)
    pooled = torch.randn((1, cfg.pooled_text_embed_dim), generator=g)
    t = torch.tensor([752.0])
    outs = []
    for ref in (MMDiTRef(ref_config(cfg), p), FakeQuantMMDiTRef(ref_config(cfg), p, covered)):
        ref.cache_modulation_params(pooled, t)
        outs.append(ref(latent, text, t))
    return outs


def test_no_covered_linear_leaves_the_oracle_bit_identical():
    for cfg in (tiny_flux_config(), tiny_sd3_config()):
        plain, hooked = _tiny_case(cfg, [])
        assert torch.equal(plain, hooked)


def test_fake_quantised_oracle_moves_but_stays_close():
    for cfg in (tiny_flux_config(), tiny_sd3_config(), tiny_sd35_config()):
        plain, fq = _tiny_case(cfg, fp8_covered_linears(cfg))
        err = float((fq - plain).norm() / plain.norm())
        assert 0.0 < err < 0.2, err


def test_covered_linears_per_model_family():
    flux = MODEL_CONFIGS["argmaxinc/mlx-FLUX.1-schnell"]
    names = fp8_covered_linears(flux)
    assert len(names) == len(set(names)) == flux.depth_multimodal * 2 * 6 + flux.depth_unified * 6
    assert "unified_transformer_blocks.0.transformer_block.mlp.fc2" in names
    for cfg in (MODEL_CONFIGS["argmaxinc/mlx-stable-diffusion-3-medium"], tiny_sd3_config(), tiny_sd35_config()):
        names = fp8_covered_linears(cfg)
        d = cfg.depth_multimodal
        # the last text stream has no post-attention linears (skip_post)
        assert len(names) == d * 12 - 3
        last_txt = f"multimodal_transformer_blocks.{d - 1}.text_transformer_block"
        assert last_txt + ".attn.q_proj" in names and last_txt + ".attn.o_proj" not in names
        assert last_txt + ".mlp.fc1" not in names
    for names in (fp8_covered_linears(flux), fp8_covered_linears(tiny_sd3_config())):
        assert not any(("embedder" in n) or ("adaLN" in n) or ("final_layer" in n) for n in names)
