"""GPU checks of FLUX.1 Canny / Depth [dev] (DESIGN.md §19): dk_canny bit for bit against the numpy Canny of
tests/control_ref.py (and the committed cv2 outputs) and its argument errors; tiny Canny and Depth pipelines against
the oracle under a launch census of their own; that the control image matters; a full-width forward under the census;
the per-step launches equal to FLUX.1-dev's; and the invariants (reruns, CUDA graphs, LoRA, the step cache, FP8,
§17's mask, Redux), with no control work on other models."""
import os
from dataclasses import replace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
bf16 = torch.bfloat16
SEEDS = [11, 12]
STEPS = 4
T = 16
HP, WP = 64, 128                       # the source image; latent 8 x 16, 4 x 8 tokens
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "canny_cv2.npz")


@pytest.fixture(scope="module")
def kc():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    from tests import kernel_checks

    kernel_checks._setup()
    return kernel_checks


def _cfg(kind="canny"):
    from tests.test_control_cpu import tiny_control_config

    return tiny_control_config(kind)


def _source():
    from tests.model_checks import _test_image

    return _test_image(HP, WP)


def _control_image(kind, flip=False):
    """a control image of another size than the target (the pipeline resizes it): blurred blocks and a ring for
    Canny, a grey ramp with a bump for Depth"""
    from scipy import ndimage

    rng = np.random.default_rng(5)
    H, W = 50, 90
    if kind == "canny":
        img = np.kron(rng.integers(0, 256, (5, 9, 3)), np.ones((10, 10, 1))).astype(np.float32)
        yy, xx = np.mgrid[:H, :W]
        ring = np.abs(np.hypot(yy - 25, xx - 60) - 14) < 2
        img[ring] = 255
        img = ndimage.gaussian_filter(img, (1.0, 1.0, 0)).round().astype(np.uint8)
    else:
        yy, xx = np.mgrid[:H, :W]
        img = (40 + 150 * xx / W + 60 * np.exp(-((yy - 20) ** 2 + (xx - 30) ** 2) / 150.0)).astype(np.uint8)
    return np.ascontiguousarray(img[::-1, ::-1]) if flip else img


def _weights(cfg, seed=7):
    from diffusionkit_b200.weights import init_params, mmdit_param_specs
    from tests.kontext_ref import sharpen

    return {k: v.to(bf16) for k, v in sharpen(init_params(mmdit_param_specs(cfg), seed=seed,
                                                          dtype=torch.float32)).items()}


def _vae(encoder):
    from tests.test_kontext_gpu import _vae_weights

    return _vae_weights(encoder=encoder)


def _pipe(cfg, p16, vp16=None, **kw):
    from tests.test_kontext_gpu import _pipe as kpipe

    return kpipe(cfg, p16, vp16, _vae(True), **kw)


# ------------------------------------------------------------------------------------------------ kernels
def _inputs(H, W, seed):
    """name -> uint8 (H, W, 4) host image: flat, noise, blurred noise, a spiral and a grey map replicated to RGB"""
    from scipy import ndimage

    from tests.control_ref import spiral

    rng = np.random.default_rng(seed)
    noise = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
    blurred = ndimage.gaussian_filter(noise.astype(np.float32), (1.5, 1.5, 0)).round().astype(np.uint8)
    grey = ndimage.gaussian_filter(rng.integers(0, 256, (H, W)).astype(np.float32), 1.0).round().astype(np.uint8)
    s = spiral(H, W, pitch=max(7.0, min(H, W) / 40))
    return {"flat": np.full((H, W, 4), 131, np.uint8), "noise": noise, "blurred": blurred,
            "spiral": np.repeat(s[..., None], 4, axis=2), "grey": np.repeat(grey[..., None], 4, axis=2)}


@pytest.mark.parametrize("H, W", [(64, 128), (1024, 1024), (2048, 2048)])
def test_canny_bit_for_bit(kc, H, W):
    from diffusionkit_b200 import control
    from tests.control_ref import canny, roundtrip_table

    table = roundtrip_table()
    for name, img in _inputs(H, W, seed=H + W).items():
        for low, high in ([(50, 200), (20, 90)] if H < 2048 or name in ("blurred", "spiral") else [(50, 200)]):
            got = control.canny(torch.from_numpy(img).to(DEV), low, high).cpu().numpy()
            want = canny(table[img[..., :3]], low, high)
            assert np.array_equal(got, np.repeat(want[..., None], 3, axis=2)), \
                (H, W, name, low, high, int((got[..., 0] != want).sum()))
            print(f"{H}x{W} {name} ({low}, {high}): {int((want > 0).sum())} edge pixels, exact")
    if H == 64:
        # with the identity table dk_canny is cv2.Canny itself: the committed OpenCV outputs
        ident = torch.arange(256, dtype=torch.uint8, device=DEV)
        g = np.load(GOLDEN)
        for i in range(sum(1 for k in g.files if k.endswith("_edges"))):
            img = g[f"case{i}_img"]
            img3 = np.repeat(img[..., None], 3, axis=2) if img.ndim == 2 else img
            low, high = (int(v) for v in g[f"case{i}_thr"])
            got = control.canny(torch.from_numpy(np.ascontiguousarray(img3)).to(DEV), low, high, lut=ident)
            assert np.array_equal(got[..., 1].cpu().numpy(), g[f"case{i}_edges"]), i


def test_canny_argument_errors_launch_nothing(kc):
    from diffusionkit_b200 import DkError, ops
    from diffusionkit_b200._lib import ptr

    c = ops.ctx(0)
    img = torch.zeros((32, 32, 3), dtype=torch.uint8, device=DEV)
    lut = torch.arange(256, dtype=torch.uint8, device=DEV)
    out = torch.empty((32, 32, 3), dtype=torch.uint8, device=DEV)
    ws = torch.empty(10 * 32 * 32 + 16, dtype=torch.uint8, device=DEV)
    a = (ptr(img), ptr(lut), ptr(out), ptr(ws))
    n0 = c.launches
    for args, msg in [((None,) + a[1:] + (32, 32, 3, 50, 200), "required"),
                      (a[:1] + (None,) + a[2:] + (32, 32, 3, 50, 200), "required"),
                      (a[:3] + (None, 32, 32, 3, 50, 200), "required"),
                      (a[:3] + (ptr(ws[1:]), 32, 32, 3, 50, 200), "aligned"),
                      (a + (0, 32, 3, 50, 200), "positive"),
                      (a + (32, -4, 3, 50, 200), "positive"),
                      (a + (65536, 65536, 3, 50, 200), "2\\^31"),
                      (a + (32, 32, 2, 50, 200), "3 channels"),
                      (a + (32, 32, 3, 200, 50), "low <= high"),
                      (a + (32, 32, 3, -1, 50), "low <= high")]:
        with pytest.raises(DkError, match=msg):
            c.call("dk_canny", *args)
    assert c.launches == n0


# ------------------------------------------------------------------------------------------------ pipelines
def _census_wrap(monkeypatch, c):
    """tests/launch_parity's census plus control.canny and the stochastic step (tests/sde_ref)"""
    from diffusionkit_b200 import control, pipeline
    from tests import launch_parity as lp
    from tests import sde_ref
    from tests.control_ref import census_check_canny

    for name, check, writes in (("canny", census_check_canny, []),
                                ("sampler_sde_step", sde_ref.census_check, ["x", "d_prev"])):
        monkeypatch.setitem(lp.CHECKS, name, check)
        monkeypatch.setitem(lp.WRITES, name, writes)
    monkeypatch.setattr(control, "canny", c._wrap("canny", control.canny))
    monkeypatch.setattr(pipeline, "sampler_sde_step", c._wrap("sampler_sde_step", pipeline.sampler_sde_step))


def _resized(ctl, H, W):
    """the oracle's prepare_control: RGB, PIL LANCZOS to exactly (W, H)"""
    from PIL import Image

    return np.asarray(Image.fromarray(ctl).convert("RGB").resize((W, H), Image.LANCZOS))


def _oracle(cfg, p16, img, ctl, cond, pooled, sig, guidance, solver):
    """the oracle control pipeline: img2img starts and the control rows from the fp32 oracle encoder"""
    from oracle import sampler_ref as sr
    from oracle.vae_ref import VAEEncoderRef, encode_image_to_latents, read_image_array
    from tests.control_ref import oracle_control_rows
    from tests.fill_ref import FillMMDiTRef, fill_pipeline_latents
    from tests.oracle_bridge import ref_config

    enc = VAEEncoderRef({k: v.float() for k, v in _vae(True).items()})
    rows = oracle_control_rows(enc, _resized(ctl, HP, WP), cfg.control, 0.1159, 0.3611, bf16)
    image = read_image_array(torch.from_numpy(img))
    x0s = []
    for s in SEEDS:
        eps = sr.get_noise(s, HP // 8, WP // 8)
        x0 = (encode_image_to_latents(enc, image, eps) - 0.1159) * 0.3611
        x0s.append(float(sig[0]) * eps + (1.0 - float(sig[0])) * x0)
    params = {k: v.float() for k, v in p16.items()}
    return fill_pipeline_latents(lambda: FillMMDiTRef(ref_config(cfg), params), solver, sig, x0s, rows, cond, pooled,
                                 guidance, 0.0, bf16, SEEDS)


def _compare(pipe, vp16, latent, want, what):
    from oracle.vae_ref import VAEDecoderRef, decode_latents_to_image
    from tests.model_checks import psnr, rel_l2

    r = rel_l2(latent, want)
    img_want = decode_latents_to_image(VAEDecoderRef({k: v.float() for k, v in vp16.items()}), want.to(bf16).float())
    ps = psnr(img_want, pipe.decode_latents_to_image(latent))
    print(f"{what}: final latent rel_l2 {r:.3e}, decoded psnr {ps:.1f} dB")
    assert r <= 5e-2 and ps >= 30.0, f"{what}: rel_l2 {r:.3e}, psnr {ps:.1f}"
    return r


@pytest.mark.parametrize("kind", ["canny", "depth"])
@pytest.mark.parametrize("denoise", [1.0, 0.6])
def test_tiny_pipeline_against_the_oracle_under_a_census(kc, monkeypatch, kind, denoise):
    from oracle import sampler_ref as sr
    from tests import launch_parity as lp
    from tests.model_checks import rel_l2

    cfg = _cfg(kind)
    p16, vp16 = _weights(cfg), _vae(False)
    pipe = _pipe(cfg, p16, vp16)
    pipe.mmdit.use_cuda_graphs = pipe.decoder.use_cuda_graphs = False
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
    img, ctl = _source(), _control_image(kind)
    sig = sr.get_sigmas(sr.FluxSamplerRef(1.0), STEPS)[int(STEPS * (1 - denoise)):]
    guidance = [30.0, 12.0]
    c = lp.Census()
    with lp.census(c):
        _census_wrap(monkeypatch, c)
        for solver in ("euler", "dpmpp_2m", "dpmpp_2m_sde"):
            c.run = f"{kind}-{solver}-{denoise}"
            n0 = len(c.records)
            lat, it = pipe.denoise_latents(cond, pooled, num_steps=STEPS, seed=SEEDS, image_path=img, denoise=denoise,
                                           solver=solver, control_image=ctl, guidance=guidance)
            torch.cuda.synchronize()
            ops_run = [r["op"] for r in c.records[n0:]]
            assert ops_run.count("canny") == (kind == "canny")
            assert len(it) == len(sig) - 1
            want = _oracle(cfg, p16, img, ctl, cond, pooled, sig, guidance, solver)
            _compare(pipe, vp16, lat, want, f"{kind} {solver} denoise {denoise}")
            if solver == "euler":
                other = _control_image(kind, flip=True)
                moved = rel_l2(_oracle(cfg, p16, img, other, cond, pooled, sig, guidance, solver), want)
                print(f"another control image moves the oracle by rel_l2 {moved:.3e}")
                assert moved > 5e-2, "the control image must matter beyond the pipeline bound"
    print(c.table())


def test_fullwidth_forward_under_a_census(kc):
    """FLUX.1-dev's width (h = 3072), 1 double + 1 single block, a 64 x 64 latent, T = 512, B = 2 with per-image
    guidance, eager under the launch census: the K = 64 control GEMM with bias once, the K = 64 x-embedder GEMM with
    the batch-broadcast residual and no bias every forward"""
    from diffusionkit_b200 import MMDiT
    from diffusionkit_b200.config import FLUX_CANNY_DEV
    from tests import launch_parity as lp
    from tests.fill_ref import FillMMDiTRef
    from tests.oracle_bridge import ref_config
    from tests.test_kontext_gpu import _check

    cfg = replace(FLUX_CANNY_DEV, depth_multimodal=1, depth_unified=1)
    B, lat, guidance = 2, (64, 64), [30.0, 10.0]
    N = (lat[0] // 2) * (lat[1] // 2)
    p16 = _weights(cfg)
    g = torch.Generator().manual_seed(5)
    latent = torch.randn((B, *lat, 16), generator=g).to(bf16)
    text = torch.randn((B, 512, cfg.token_level_text_embed_dim), generator=g).to(bf16)
    pooled = torch.randn((B, cfg.pooled_text_embed_dim), generator=g).to(bf16)
    rows = torch.randn((N, 64), generator=g).to(bf16)
    m = MMDiT(cfg, {k: v.to(DEV) for k, v in p16.items()})
    m.use_cuda_graphs = False
    m.cache_modulation_params(pooled.to(DEV), [752.0], guidance)
    c = lp.Census()
    c.run = "canny-fullwidth"
    with lp.census(c):
        m.cache_fill_conditioning(rows.to(DEV))
        got = m(latent.to(DEV), text.to(DEV), timestep=752.0)
        torch.cuda.synchronize()
        got = got.clone()
    print(c.table())
    sigs = [r["info"] for r in c.records if r["op"] == "gemm" and r["info"]["K"] == 64]
    assert [(s["M"], s["epi"]) for s in sigs] == [(N, "bias"), (B * N, "res")], sigs
    assert sigs[1]["res_batch_rows"] == 0
    del m
    torch.cuda.empty_cache()
    ref = FillMMDiTRef(ref_config(cfg), {k: v.float() for k, v in p16.items()})
    ref.cond = rows.float()
    t = torch.tensor([752.0])
    ref.cache_modulation_params(pooled.float(), t, guidance)
    _check(got, ref(latent.float(), text.float(), t.repeat(B)), "canny full width, 64x64, T = 512, B = 2")


def test_per_step_launches_equal_flux_dev(kc):
    """a control forward launches exactly what a FLUX.1-dev forward of the same shape launches"""
    from diffusionkit_b200 import MMDiT, ops

    cfg = _cfg()
    dev = replace(cfg, x_embedder_cond_channels=0, control=None)
    g = torch.Generator().manual_seed(3)
    latent = torch.randn((2, 8, 16, 16), generator=g).to(bf16).to(DEV)
    text = torch.randn((2, T, cfg.token_level_text_embed_dim), generator=g).to(bf16).to(DEV)
    pooled = torch.randn((2, cfg.pooled_text_embed_dim), generator=g).to(bf16).to(DEV)
    counts = []
    for c in (cfg, dev):
        m = MMDiT(c, {k: v.to(DEV) for k, v in _weights(c).items()})
        m.use_cuda_graphs = False
        m.cache_modulation_params(pooled, [500.0], [3.5, 3.5])
        if c.x_embedder_cond_channels:
            m.cache_fill_conditioning(torch.zeros((32, 64), dtype=bf16, device=DEV))
        m(latent, text, timestep=500.0)
        n0 = ops.launch_count()
        m(latent, text, timestep=500.0)
        counts.append(ops.launch_count() - n0)
    assert counts[0] == counts[1], counts


# ------------------------------------------------------------------------------------------------ invariants
def test_invariants(kc):
    cfg = _cfg()
    p16, vp16 = _weights(cfg), _vae(False)
    pipe = _pipe(cfg, p16, vp16)
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
    img, ctl = _source(), _control_image("canny")
    kw = dict(num_steps=STEPS, seed=SEEDS, latent_size=(HP // 8, WP // 8), control_image=ctl)

    def run(**extra):
        lat, _ = pipe.denoise_latents(cond, pooled, **{**kw, **extra})
        torch.cuda.synchronize()
        return lat.clone()

    base = run()
    assert torch.equal(run(), base), "a rerun repeats"
    pipe.mmdit.use_cuda_graphs = False
    assert torch.equal(run(), base), "CUDA graphs equal eager"
    pipe.mmdit.use_cuda_graphs = True
    assert torch.equal(run(guidance=30.0), base), "guidance None is 30 on Canny"
    assert not torch.equal(run(canny_thresholds=(20, 90)), base), "the thresholds reach the edges"
    # an edge map computed once and passed with canny_thresholds=None is the same conditioning
    from diffusionkit_b200 import control

    edges = control.canny(torch.from_numpy(_resized(ctl, HP, WP)).to(DEV)).cpu().numpy()
    assert torch.equal(run(control_image=edges, canny_thresholds=None), base)
    # the log
    _, log = pipe.generate_image("", verbose=False, conditioning=cond, pooled_conditioning=pooled, **kw)
    c = log["denoising"]["control"]
    assert c["kind"] == "canny" and c["latent_size"] == (HP // 8, WP // 8) and c["time"] >= 0
    # LoRA on the x-embedder and the blocks: load, rescale and unload restore every bit
    from tests.lora_fixtures import kohya_dict, make_factors, upstream_modules

    name = pipe.load_lora_weights(kohya_dict(make_factors(upstream_modules(cfg), 4, seed=3)), scale=1.0)
    with_lora = run()
    assert not torch.equal(with_lora, base)
    pipe.set_lora_scale(name, 0.0)
    assert torch.equal(run(), base), "scale 0"
    pipe.set_lora_scale(name, 1.0)
    assert torch.equal(run(), with_lora), "scale back"
    pipe.unload_lora_weights(name)
    assert torch.equal(run(), base), "unloaded"
    # step cache: threshold 0 never skips and changes no bit
    pipe.set_step_cache(0.0)
    assert torch.equal(run(), base)
    pipe.set_step_cache(None)
    # FP8 decodes close to 16-bit
    from tests.model_checks import psnr

    want = pipe.decode_latents_to_image(base)
    pipe.set_fp8(True)
    got = pipe.decode_latents_to_image(run())
    pipe.set_fp8(False)
    ps = psnr(want.cpu(), got.cpu())
    print(f"fp8 vs 16-bit decoded psnr {ps:.1f} dB")
    assert ps >= 25.0
    # §17's mask on a Canny model: the unmasked pixels are the source's, bit for bit
    from tests.test_fill_gpu import _mask

    mask = _mask()
    images, log = pipe.generate_image("", verbose=False, conditioning=cond, pooled_conditioning=pooled,
                                      image_path=img, mask_image=mask, denoise=0.75, **kw)
    keep = mask < 128
    for im in images:
        assert np.array_equal(np.asarray(im)[keep], img[keep])
    assert "inpaint" in log["denoising"] and "control" in log["denoising"] and "fill" not in log["denoising"]


def test_redux_tokens_equal_conditioning(kc):
    from diffusionkit_b200.config import tiny_siglip_config

    cfg = _cfg("depth")
    pipe = _pipe(cfg, _weights(cfg))
    pipe.load_redux(siglip_config=tiny_siglip_config())
    cond, pooled = pipe.synthetic_text_embeddings(n_images=1, text_len=T)
    img = _source()
    prompt = np.roll(img, 17, axis=1)
    kw = dict(num_steps=STEPS, seed=5, image_path=img, denoise=0.8, control_image=_control_image("depth"))
    a, _ = pipe.denoise_latents(cond, pooled, redux_image=prompt, **kw)
    a = a.clone()
    tokens = pipe.encode_redux(prompt)
    b, _ = pipe.denoise_latents(torch.cat([cond.to(DEV), tokens], dim=1), pooled, **kw)
    assert torch.equal(a, b)


def test_errors_and_other_models(kc, monkeypatch):
    """argument errors launch nothing; a FLUX.1-dev model and a Fill model run no control work"""
    from diffusionkit_b200 import control, ops
    from tests.test_fill_gpu import _cfg as fill_cfg
    from tests.test_fill_gpu import _mask

    cfg = _cfg()
    pipe = _pipe(cfg, _weights(cfg))
    cond, pooled = pipe.synthetic_text_embeddings(n_images=1, text_len=T)
    img, ctl = _source(), _control_image("canny")
    n0 = ops.launch_count()
    for kw, msg in [(dict(image_path=img), "needs control_image"),
                    (dict(control_image=ctl, reference_latents=torch.zeros(1, 8, 8, 16, device=DEV)), "Kontext"),
                    (dict(control_image=ctl, canny_thresholds=(9, 3)), "low <= high"),
                    (dict(control_image=np.zeros((8, 8, 2), np.uint8)), "control_image array")]:
        with pytest.raises(ValueError, match=msg):
            pipe.denoise_latents(cond, pooled, num_steps=STEPS, seed=3, **kw)
        with pytest.raises(ValueError, match=msg):
            pipe.generate_image("", num_steps=STEPS, seed=3, verbose=False, conditioning=cond,
                                pooled_conditioning=pooled, **kw)
    assert ops.launch_count() == n0
    calls = []
    for name in ("canny", "control_rows", "load_control_image"):
        fn = getattr(control, name)
        monkeypatch.setattr(control, name, lambda *a, _fn=fn, _n=name, **k: calls.append(_n) or _fn(*a, **k))
    fcfg = fill_cfg()
    fill = _pipe(fcfg, _weights(fcfg), _vae(False))
    _, log = fill.generate_image("", num_steps=STEPS, seed=3, verbose=False, conditioning=cond,
                                 pooled_conditioning=pooled, image_path=img, mask_image=_mask())
    assert "fill" in log["denoising"] and "control" not in log["denoising"]
    dcfg = replace(cfg, x_embedder_cond_channels=0, control=None)
    dev = _pipe(dcfg, _weights(dcfg), _vae(False))
    _, log = dev.generate_image("", num_steps=STEPS, seed=3, verbose=False, conditioning=cond,
                                pooled_conditioning=pooled, latent_size=(8, 16))
    assert calls == [] and "control" not in log["denoising"]
    with pytest.raises(ValueError, match="has none"):
        dev.denoise_latents(cond, pooled, num_steps=STEPS, seed=3, control_image=ctl)
