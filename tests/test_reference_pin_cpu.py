"""CPU: the oracle pinned against the REFERENCE'S OWN code.

argmaxinc/DiffusionKit ships a PyTorch twin of its SD3 MMDiT and VAE decoder (python/src/diffusionkit/torch/mmdit.py,
vae.py — the sources of its Core ML conversion).  Unlike the MLX path they can execute in this container once the four
generic argmaxtools layers they import are supplied (tests/golden/reference_shims.py).  tests/golden/
make_reference_golden.py ran them on the deterministic synthetic weights and committed inputs + outputs
(reference_torch_*.npz); here the oracle has to reproduce those outputs.  The two documented differences between the
twins are switched on the oracle side: tanh GELU (torch/mmdit.py:242 vs mlx/mmdit.py:421) and GroupNorm eps 1e-6
(torch/vae.py:20 vs the MLX default 1e-5).

When the reference checkout is present the reference modules are also re-run live, so a stale fixture cannot hide a
drift; the other comparisons with reference code use outputs stored by tests/golden/reference_values.py.
"""
import os

import numpy as np
import pytest
import torch

from diffusionkit_b200.weights import init_params, mmdit_param_specs, vae_decoder_param_specs
from oracle.mmdit_ref import MMDiTRef
from oracle.vae_ref import VAEDecoderRef
from tests.golden import make_reference_golden as mk
from tests.golden import reference_shims as rs
from tests.golden.reference_values import recorded
from tests.oracle_bridge import ref_config

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
AVAILABLE = rs.reference_available()


def _oracle_mmdit(latent, text, pooled, timestep):
    cfg = mk.pin_mmdit_config()
    params = init_params(mmdit_param_specs(cfg), seed=mk.MMDIT_SEED, dtype=torch.float32)
    rc = ref_config(cfg)
    rc.gelu_tanh = True
    ref = MMDiTRef(rc, params, act_dtype=None)
    ref.cache_modulation_params(pooled, timestep[:1])
    return ref(latent, text, timestep)


def _oracle_vae(z):
    cfg = mk.pin_vae_config()
    params = init_params(vae_decoder_param_specs(cfg), seed=mk.VAE_SEED, dtype=torch.float32)
    dec = VAEDecoderRef(params, None, cfg.block_out_channels, cfg.layers_per_block)
    dec.gn_eps = 1e-6
    return dec(z)


def test_oracle_mmdit_matches_reference_torch_module():
    g = np.load(os.path.join(GOLD, "reference_torch_mmdit.npz"))
    latent, text, pooled, timestep = [torch.from_numpy(g[k]) for k in ("latent", "text", "pooled", "timestep")]
    got = _oracle_mmdit(latent, text, pooled, timestep)
    want = torch.from_numpy(g["out"])
    assert got.shape == want.shape == (2, 12, 8, 16)
    assert torch.allclose(got, want, atol=2e-4, rtol=1e-4), float((got - want).abs().max())
    # the pin is sensitive to exactly the things a restatement gets wrong: activation flavour ...
    cfg = mk.pin_mmdit_config()
    params = init_params(mmdit_param_specs(cfg), seed=mk.MMDIT_SEED, dtype=torch.float32)
    erf = MMDiTRef(ref_config(cfg), params, act_dtype=None)
    erf.cache_modulation_params(pooled, timestep[:1])
    assert not torch.allclose(erf(latent, text, timestep), want, atol=2e-4, rtol=1e-4)


def test_oracle_vae_decoder_matches_reference_torch_module():
    g = np.load(os.path.join(GOLD, "reference_torch_vae_decoder.npz"))
    z, want = torch.from_numpy(g["latent"]), torch.from_numpy(g["out"])
    got = _oracle_vae(z)
    assert got.shape == want.shape == (1, 48, 32, 3)
    assert torch.allclose(got, want, atol=2e-4, rtol=1e-4), float((got - want).abs().max())


def test_fixtures_are_what_the_reference_produces_today():
    """the stored inputs are what the generator produces today; with the reference checkout present, the stored outputs
    are also what the reference modules produce today"""
    latent, text, pooled, timestep, z = mk.make_inputs()
    g = np.load(os.path.join(GOLD, "reference_torch_mmdit.npz"))
    gv = np.load(os.path.join(GOLD, "reference_torch_vae_decoder.npz"))
    assert np.array_equal(g["latent"], latent.numpy()) and np.array_equal(gv["latent"], z.numpy())
    if AVAILABLE:
        y = mk.run_reference_mmdit(latent, text, pooled, timestep)
        assert np.allclose(y.numpy(), g["out"], atol=1e-6)
        img = mk.run_reference_vae(z)
        assert np.allclose(img.numpy(), gv["out"], atol=1e-6)


def test_checkpoint_loaders_match_the_reference_loaders():
    """SURVEY.md §8 row f1 pinned by reference code: an upstream-layout (Stability SD3 / LDM) checkpoint goes through the
    REFERENCE's own key adjustments (torch/mmdit.py:424-497, torch/model_io.py:90-122) into the reference modules with
    strict=True, and through diffusionkit_b200.model_io into the oracle — same outputs."""
    from diffusionkit_b200 import model_io
    from tests.test_model_io_cpu import _sd3_upstream, _vae_upstream

    latent, text, pooled, timestep, z = mk.make_inputs()

    # ---- SD3 MMDiT
    cfg = mk.pin_mmdit_config()
    params = init_params(mmdit_param_specs(cfg), seed=31, dtype=torch.float32)
    upstream = _sd3_upstream(params, cfg)
    for k in list(upstream):                        # a real checkpoint has a k bias; both loaders must drop it
        if k.endswith("attn.qkv.bias"):
            upstream[k] = upstream[k] + 0.3
    # ---- VAE decoder
    vcfg = mk.pin_vae_config()
    vparams = init_params(vae_decoder_param_specs(vcfg), seed=32, dtype=torch.float32)
    vup = _vae_upstream(vparams, prefix="first_stage_model.decoder.")

    def reference():
        m, v, mio = rs.load_reference_module("mmdit"), rs.load_reference_module("vae"), rs.load_reference_module("model_io")
        # the reference loader's own prefix rule (torch/model_io.py:67-71): drop "model.diffusion_model", skip the VAE
        stripped = {".".join(k.rsplit(".")[2:]): t for k, t in upstream.items()
                    if all(s not in k for s in ["encoder", "decoder"])}
        ref_sd = m.mmdit_state_dict_adjustments(stripped)
        rcfg = m.MMDiTConfig(depth=cfg.depth_multimodal, max_latent_resolution=cfg.max_latent_resolution,
                             pooled_text_embed_dim=cfg.pooled_text_embed_dim,
                             token_level_text_embed_dim=cfg.token_level_text_embed_dim)
        net = m.MMDiT(rcfg).eval()
        net.load_state_dict(ref_sd, strict=True)
        with torch.no_grad():
            (want,) = net(latent.permute(0, 3, 1, 2).contiguous(), text.permute(0, 2, 1)[:, :, None, :].contiguous(),
                          pooled[:, :, None, None], timestep)
        boc = vcfg.block_out_channels
        vnet = v.VAEDecoder(v.VAEDecoderConfig(resolution=z.shape[1] * 8, base_channels=boc[0],
                                               channel_multipliers=[c // boc[0] for c in boc],
                                               num_res_blocks=vcfg.layers_per_block - 1)).eval()
        vnet.load_state_dict(mio.vae_decoder_state_dict_adjustments(dict(vup)), strict=True)
        with torch.no_grad():
            vwant = vnet(z.permute(0, 3, 1, 2).contiguous()).permute(0, 2, 3, 1)
        return {"mmdit": want.permute(0, 2, 3, 1), "vae": vwant}

    want = recorded("torch_checkpoint_loaders", reference, AVAILABLE)
    mine = model_io.sd3_checkpoint_to_params(upstream)
    model_io.check_against_specs(mine, mmdit_param_specs(cfg))
    rc = ref_config(cfg)
    rc.gelu_tanh = True
    ref = MMDiTRef(rc, mine, act_dtype=None)
    ref.cache_modulation_params(pooled, timestep[:1])
    want.close("mmdit", ref(latent, text, timestep), atol=2e-4, rtol=1e-4)

    vmine = model_io.vae_decoder_checkpoint_to_params(vup)
    model_io.check_against_specs(vmine, vae_decoder_param_specs(vcfg))
    dec = VAEDecoderRef(vmine, None, vcfg.block_out_channels, vcfg.layers_per_block)
    dec.gn_eps = 1e-6
    want.close("vae", dec(z), atol=2e-4, rtol=1e-4)


def test_psnr_metric_is_the_reference_metric():
    """the parity metric itself (tests use oracle.sampler_ref.compute_psnr): reference diffusionkit/utils.py:70-82"""
    import importlib.util

    from oracle.sampler_ref import compute_psnr

    rng = np.random.RandomState(0)
    a = rng.randn(3, 8, 8).astype(np.float32)
    b = a + 0.01 * rng.randn(3, 8, 8).astype(np.float32)
    c = a + 0.3 * rng.randn(3, 8, 8).astype(np.float32)

    def reference():
        rs.install()
        path = os.path.join(os.path.dirname(rs.REFERENCE_TORCH_DIR), "utils.py")
        spec = importlib.util.spec_from_file_location("_reference_utils", path)
        utils = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(utils)
        return {"psnr_ab": np.array(float(utils.compute_psnr(a, b))), "psnr_ac": np.array(float(utils.compute_psnr(a, c)))}

    want = recorded("torch_psnr", reference, AVAILABLE)
    assert abs(compute_psnr(a, b) - float(want["psnr_ab"])) < 1e-3
    assert abs(compute_psnr(a, c) - float(want["psnr_ac"])) < 1e-3
