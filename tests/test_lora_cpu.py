"""CPU: LoRA adapter parsing — kohya and PEFT encodings, the split of fused upstream modules onto reference-named
weights (pinned to the checkpoint loader), skipped and rejected keys."""
import pytest
import torch

from diffusionkit_b200 import model_io
from diffusionkit_b200.config import tiny_flux_config, tiny_sd3_config
from diffusionkit_b200.lora import load_lora, module_table
from diffusionkit_b200.weights import mmdit_param_specs
from tests.lora_fixtures import kohya_dict, make_factors, peft_dict, upstream_delta, upstream_modules

CONFIGS = {"flux": tiny_flux_config, "sd3": tiny_sd3_config}
PREFIX = {"flux": "diffusion_model.", "sd3": "model.diffusion_model."}


def _to_params(kind, cfg, sd):
    if kind == "flux":
        return model_io.flux_checkpoint_to_params(sd, cfg.hidden_size, cfg.mlp_ratio)
    return model_io.sd3_checkpoint_to_params(sd)


@pytest.mark.parametrize("kind", ["flux", "sd3"])
def test_targets_match_checkpoint_loader(kind):
    """ΔW of every upstream module pushed through the checkpoint loader equals up @ down of the adapter's targets"""
    cfg = CONFIGS[kind]()
    modules = upstream_modules(cfg)
    assert set(modules) == set(module_table(cfg))                       # every upstream Linear / conv is adaptable
    factors = make_factors(modules, rank=5, seed=1)
    want = _to_params(kind, cfg, upstream_delta(factors))
    shapes = {n: s for n, s, _ in mmdit_param_specs(cfg)}
    lora = load_lora(kohya_dict(factors), cfg)
    assert set(lora.targets) == set(want)
    assert lora.skipped == []
    for name, (up, down) in lora.targets.items():
        got = (up @ down).reshape(shapes[name])
        assert got.dtype == torch.float32
        torch.testing.assert_close(got, want[name], rtol=1e-5, atol=1e-6, msg=name)
    assert any(".attn.k_proj.weight" in n for n in lora.targets)       # k keeps its share of qkv / linear1


@pytest.mark.parametrize("kind", ["flux", "sd3"])
def test_kohya_and_peft_give_identical_targets(kind):
    cfg = CONFIGS[kind]()
    factors = make_factors(upstream_modules(cfg), rank=3, seed=2)
    ref = load_lora(kohya_dict(factors), cfg).targets
    for prefix in ("", PREFIX["flux"], PREFIX["sd3"]):
        got = load_lora(peft_dict(factors, prefix), cfg).targets
        assert set(got) == set(ref)
        for name in ref:
            assert torch.equal(got[name][0], ref[name][0]) and torch.equal(got[name][1], ref[name][1]), name
    # without an alpha, alpha = rank: the same as kohya with alpha = rank
    plain = make_factors(upstream_modules(cfg), rank=3, seed=2, alphas=False)
    a, b = load_lora(kohya_dict(plain), cfg).targets, load_lora(peft_dict(plain), cfg).targets
    for name in a:
        assert torch.equal(a[name][0], b[name][0]) and torch.equal(a[name][1], b[name][1]), name


def test_alpha_scales_the_up_factor():
    cfg = tiny_flux_config()
    m = "double_blocks.0.img_attn.proj"
    up, down = torch.randn(cfg.hidden_size, 4), torch.randn(4, cfg.hidden_size)
    one = load_lora({f"{m}.lora_A.weight": down, f"{m}.lora_B.weight": up}, cfg).targets
    two = load_lora({f"{m}.lora_A.weight": down, f"{m}.lora_B.weight": up, f"{m}.alpha": torch.tensor(8.0)}, cfg).targets
    name = "multimodal_transformer_blocks.0.image_transformer_block.attn.o_proj.weight"
    assert torch.equal(one[name][0], up) and torch.equal(two[name][0], up * 2.0)


def test_skipped_keys_are_reported():
    cfg = tiny_flux_config()
    m = "double_blocks.1.txt_mlp.0"
    sd = peft_dict(make_factors({m: (4 * cfg.hidden_size, cfg.hidden_size)}, rank=2, seed=3), "diffusion_model.")
    extra = ["lora_te1_text_model_encoder_layers_0_mlp_fc1.lora_down.weight",
             "text_encoder.text_model.encoder.layers.0.mlp.fc1.lora_A.weight",
             "lora_unet_guidance_in_in_layer.lora_down.weight",
             "diffusion_model.guidance_in.out_layer.lora_B.weight"]
    for k in extra:
        sd[k] = torch.zeros(2, 2)
    lora = load_lora(sd, cfg, name="style")
    assert sorted(lora.skipped) == sorted(extra)
    assert lora.name == "style"
    assert set(lora.targets) == {"multimodal_transformer_blocks.1.text_transformer_block.mlp.fc1.weight"}


def test_unknown_misshaped_and_lycoris_keys_raise():
    cfg, h = tiny_flux_config(), tiny_flux_config().hidden_size
    ok = {"lora_unet_single_blocks_0_linear2.lora_down.weight": torch.zeros(4, 5 * h),
          "lora_unet_single_blocks_0_linear2.lora_up.weight": torch.zeros(h, 4)}
    assert set(load_lora(ok, cfg).targets) == {"unified_transformer_blocks.0.transformer_block.attn.o_proj.weight",
                                               "unified_transformer_blocks.0.transformer_block.mlp.fc2.weight"}
    for bad in ("transformer.transformer_blocks.0.attn.to_q.lora_A.weight",        # diffusers naming
                "lora_unet_double_blocks_0_img_attn_mystery.lora_down.weight",
                "lora_unet_double_blocks_9_img_attn_qkv.lora_down.weight",         # block the model does not have
                "joint_blocks.0.x_block.attn.qkv.lora_A.weight",                  # SD3 module in a FLUX adapter
                "diffusion_model.double_blocks.0.img_attn.qkv.weight"):
        with pytest.raises(KeyError, match=bad.replace(".", r"\.")):
            load_lora({**ok, bad: torch.zeros(4, h)}, cfg)
    wrong = dict(ok)
    wrong["lora_unet_single_blocks_0_linear2.lora_down.weight"] = torch.zeros(4, 4 * h)
    with pytest.raises(ValueError, match="linear2"):
        load_lora(wrong, cfg)
    wrong = dict(ok)
    wrong["lora_unet_single_blocks_0_linear2.lora_up.weight"] = torch.zeros(h, 3)   # rank differs from down's
    with pytest.raises(ValueError):
        load_lora(wrong, cfg)
    half = {"lora_unet_single_blocks_0_linear2.lora_down.weight": torch.zeros(4, 5 * h)}
    with pytest.raises(ValueError, match="up"):
        load_lora(half, cfg)
    for k in ("lora_unet_double_blocks_0_img_attn_qkv.hada_w1_a", "lora_unet_double_blocks_0_img_attn_qkv.lokr_w1",
              "lora_unet_double_blocks_0_img_attn_qkv.dora_scale"):
        with pytest.raises(ValueError, match="LyCORIS"):
            load_lora({**ok, k: torch.zeros(4, h)}, cfg)
    # an SD3 model has no FLUX modules and vice versa
    with pytest.raises(KeyError):
        load_lora(ok, tiny_sd3_config())


def test_safetensors_roundtrip(tmp_path):
    from safetensors.torch import save_file

    cfg = tiny_sd3_config()
    factors = make_factors(upstream_modules(cfg), rank=4, seed=4)
    sd = {k: v.to(torch.bfloat16).contiguous() for k, v in kohya_dict(factors).items()}
    path = tmp_path / "my_style.safetensors"
    save_file(sd, str(path))
    from_file = load_lora(path, cfg)
    from_dict = load_lora(sd, cfg)
    assert from_file.name == "my_style" and from_dict.name == "adapter"
    assert set(from_file.targets) == set(from_dict.targets)
    for name, (up, down) in from_dict.targets.items():
        assert torch.equal(from_file.targets[name][0], up) and torch.equal(from_file.targets[name][1], down)
