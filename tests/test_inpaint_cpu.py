"""CPU checks of masked inpainting (DESIGN.md §17): the mask preparation for every input form against plain loops
(tests/inpaint_ref.py), its argument errors, and properties of the masked oracle solvers: an all-ones mask is img2img,
an all-zeros mask ends at the source, and every solver ends at the source wherever the mask keeps it."""
import math

import numpy as np
import pytest
import torch
from PIL import Image

from diffusionkit_b200 import inpaint
from tests import inpaint_ref as ir


def _gray(H, W, seed=0):
    rng = np.random.RandomState(seed)
    g = np.zeros((H, W), dtype=np.uint8)
    g[H // 4:H // 2, W // 3:2 * W // 3] = 255
    g[:, W - 5] = rng.randint(100, 256, H).astype(np.uint8)          # a noisy column around the threshold
    return g


def _forms(gray, tmp_path):
    """the same mask as a path (L, RGB, RGBA files), a PIL image (L, RGB, RGBA) and arrays (H, W), (H, W, 1|3|4)"""
    rgb = np.repeat(gray[:, :, None], 3, axis=2)
    rgba = np.concatenate([rgb, np.full(gray.shape + (1,), 77, np.uint8)], axis=2)
    out = {"array_hw": gray, "array_hw1": gray[:, :, None], "array_rgb": rgb, "array_rgba": rgba}
    for mode, arr in (("L", gray), ("RGB", rgb), ("RGBA", rgba)):
        im = Image.fromarray(arr, mode)
        out[f"pil_{mode}"] = im
        p = tmp_path / f"mask_{mode}.png"
        im.save(p)
        out[f"path_{mode}"] = str(p)
    return out


@pytest.mark.parametrize("size", [(128, 192), (130, 200)])           # (H, W): a multiple of 64, and one to resize
def test_mask_preparation_matches_plain_loops(tmp_path, size):
    H, W = size
    gray = _gray(H, W)
    want_px, want_lat = ir.ref_prepare(Image.fromarray(gray, "L"), (W, H))
    assert want_px.shape == (H - H % 64, W - W % 64)
    for name, m in _forms(gray, tmp_path).items():
        got = inpaint.prepare_mask(m, (W, H))
        assert got.pixels.dtype == np.uint8 and got.latent.dtype == np.uint8, name
        assert np.array_equal(got.pixels, want_px), name
        assert np.array_equal(got.latent, want_lat), name
        assert got.masked_fraction == float(want_lat.mean())


def test_a_one_pixel_stroke_marks_its_latent():
    g = np.zeros((64, 128), dtype=np.uint8)
    g[37, :] = 255                                                    # one row of pixels
    g[:, 101] = 200                                                   # one column
    g[5, 5] = 128                                                     # one pixel, exactly at the threshold
    m = inpaint.prepare_mask(g, (128, 64))
    want = np.zeros((8, 16), dtype=np.uint8)
    want[37 // 8, :] = 1
    want[:, 101 // 8] = 1
    want[0, 0] = 1
    assert np.array_equal(m.latent, want) and np.array_equal(m.latent, ir.ref_latent_mask(m.pixels))
    assert int(m.pixels.sum()) == 128 + 64 - 1 + 1
    assert inpaint.prepare_mask(np.full((64, 64), 127, np.uint8), (64, 64)).latent.sum() == 0


def test_latent_mask_against_the_loop():
    rng = np.random.RandomState(3)
    for p in (0.002, 0.05, 0.5):
        px = (rng.rand(64, 192) < p).astype(np.uint8)
        assert np.array_equal(inpaint.latent_mask(px), ir.ref_latent_mask(px))


def test_mask_errors(tmp_path):
    g = np.zeros((64, 64), dtype=np.uint8)
    with pytest.raises(ValueError, match="same size"):
        inpaint.prepare_mask(g, (128, 64))
    with pytest.raises(ValueError, match="uint8"):
        inpaint.prepare_mask(g.astype(np.float32), (64, 64))
    with pytest.raises(ValueError, match="uint8"):
        inpaint.prepare_mask(np.zeros((64, 64, 2), np.uint8), (64, 64))
    with pytest.raises(ValueError, match="uint8"):
        inpaint.prepare_mask(np.zeros((2, 64, 64, 1), np.uint8), (64, 64))
    with pytest.raises(ValueError, match="cannot be read"):
        inpaint.prepare_mask(str(tmp_path / "missing.png"), (64, 64))
    bad = tmp_path / "bad.png"
    bad.write_bytes(b"not an image")
    with pytest.raises(ValueError, match="cannot be read"):
        inpaint.prepare_mask(str(bad), (64, 64))
    with pytest.raises(ValueError, match="path, a PIL image or a uint8 array"):
        inpaint.prepare_mask([[0]], (64, 64))
    with pytest.raises(ValueError, match="smaller than 64x64"):
        inpaint.prepare_mask(np.zeros((32, 80), np.uint8), (80, 32))


def test_pipeline_refuses_bad_masks_before_any_gpu_work(tmp_path):
    """DiffusionPipeline._inpaint_input runs on the host alone (self is not used): the checks need no device"""
    from diffusionkit_b200.pipeline import DiffusionPipeline

    src = np.zeros((70, 130, 3), dtype=np.uint8)
    with pytest.raises(ValueError, match="needs image_path"):
        DiffusionPipeline._inpaint_input(None, None, np.zeros((64, 64), np.uint8))
    with pytest.raises(ValueError, match="same size"):
        DiffusionPipeline._inpaint_input(None, src, np.zeros((64, 128), np.uint8))   # the resized size is not enough
    source, m = DiffusionPipeline._inpaint_input(None, src, np.full((70, 130), 255, np.uint8))
    assert source.shape == (64, 128, 3) and m.latent.shape == (8, 16) and m.masked_fraction == 1.0
    assert DiffusionPipeline._inpaint_input(None, source, m) == (source, m)


# ------------------------------------------------------------------------------------------------ oracle properties
class _Toy:
    """a smooth stand-in denoiser: D = tanh(x) * 0.7 + 0.1 sin(3 sigma), so every solver step moves every element"""

    def __call__(self, x, k, i, sig):
        return torch.tanh(x) * 0.7 + 0.1 * math.sin(3.0 * float(sig[k]))


def _case(seed=0, H=4, W=6):
    g = torch.Generator().manual_seed(seed)
    eps = torch.randn((1, H, W, 16), generator=g)
    x0 = torch.randn((1, H, W, 16), generator=g)
    mask = torch.zeros((H, W), dtype=torch.uint8)
    mask[1:3, 2:5] = 1
    return eps, x0, mask


def _run(solver, sig, eps, x0, mask):
    toy = _Toy()
    x = float(sig[0]) * eps + (1.0 - float(sig[0])) * x0                # img2img's start
    return ir.sample(solver, lambda xx, k, i: toy(xx, k, i, sig), x, sig, eps, x0, mask, seed=5, eta=1.0)


def _sigmas(trim=0, n=6):
    from oracle import sampler_ref as sr

    return sr.get_sigmas(sr.FluxSamplerRef(1.0), n)[trim:]


@pytest.mark.parametrize("solver", ir.SOLVERS)
@pytest.mark.parametrize("trim", [0, 2])
def test_unmasked_latents_end_at_the_source(solver, trim):
    sig = _sigmas(trim)
    eps, x0, mask = _case()
    x = _run(solver, sig, eps, x0, mask)
    keep = (mask == 0)[None, :, :, None].expand_as(x)
    assert torch.equal(x[keep], x0[keep])
    assert not torch.equal(x[~keep], x0[~keep])
    zeros = _run(solver, sig, eps, x0, torch.zeros_like(mask))
    assert torch.equal(zeros, x0)


@pytest.mark.parametrize("solver", ir.SOLVERS)
def test_an_all_ones_mask_is_img2img(solver):
    """the blend never touches a repainted position: the masked loop with nothing kept is the plain img2img loop of
    the existing oracles"""
    from oracle import sampler_ref as sr
    from tests import sde_ref, solver_ref

    sig = _sigmas(1)
    eps, x0, mask = _case(1)
    got = _run(solver, sig, eps, x0, torch.ones_like(mask))
    toy = _Toy()
    sigl = [float(v) for v in sig]
    x = float(sig[0]) * eps + (1.0 - float(sig[0])) * x0

    # the existing oracle loops over a model whose "output" makes calculate_denoised return the toy D
    def mmdit_call(xin, c, t):
        k = int(np.argmin([abs(s * 1000.0 - float(t[0])) for s in sigl]))
        return (xin - toy(xin, k, k, sigl)) / sigl[k]

    args = (mmdit_call, lambda p, t: None, x, sig, None, None, 0.0, None)
    if solver in ("euler_ancestral", "dpmpp_2m_sde"):
        want = getattr(sde_ref, "sample_" + solver)(*args, seed=5, eta=1.0)
    else:
        want = {"euler": sr.sample_euler, "heun": solver_ref.sample_heun,
                "dpmpp_2m": solver_ref.sample_dpmpp_2m}[solver](*args)
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-4)


def test_ref_blend_and_paste():
    eps, x0, mask = _case(2)
    x = torch.randn_like(eps)
    got = ir.ref_blend(x, eps, x0, mask, 0.25, 0.75)
    keep = (mask == 0)[None, :, :, None].expand_as(x)
    assert torch.equal(got[~keep], x.double()[~keep])
    assert torch.allclose(got[keep], (0.25 * eps.double() + 0.75 * x0.double())[keep])
    img = torch.randint(0, 256, (2, 8, 8, 3), dtype=torch.uint8)
    src = torch.randint(0, 256, (8, 8, 3), dtype=torch.uint8)
    pm = torch.zeros((8, 8), dtype=torch.uint8)
    pm[2:5, 1:7] = 1
    out = ir.ref_paste(img, src, pm)
    for b in range(2):
        for i in range(8):
            for j in range(8):
                assert torch.equal(out[b, i, j], img[b, i, j] if pm[i, j] else src[i, j])
