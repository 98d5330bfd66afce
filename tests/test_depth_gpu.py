"""GPU checks of FLUX.1 Depth's depth estimator (DESIGN.md §20): dk_resample, dk_conv3x3_s2_p1, dk_depth_add_relu and
dk_depth_head against their references, with argument errors that launch nothing; the estimator against the fp32
oracle (tests/depth_ref.py) under a launch census of its own; tiny FLUX.1 Depth pipelines with estimate_depth=True
against the oracle pipeline; and the exactness the feature promises."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
bf16, fp16, f32 = torch.bfloat16, torch.float16, torch.float32
SEEDS = [11, 12]
STEPS = 4
T = 16
HP, WP = 64, 128


@pytest.fixture(scope="module")
def kc():
    if not torch.cuda.is_available():
        pytest.skip("needs an H100")
    from tests import kernel_checks

    kernel_checks._setup()
    return kernel_checks


def _rel(got, want):
    got, want = got.double().cpu(), want.double().cpu()
    return float((got - want).norm() / want.norm().clamp_min(1e-30))


# ------------------------------------------------------------------------------------------------ kernels
RESAMPLES = [("bilinear_ac", (19, 19), (37, 37), 256), ("bilinear_ac", (148, 148), (296, 296), 256),
             ("bilinear_ac", (296, 296), (518, 518), 128), ("bilinear", (37, 49), (74, 98), 64),
             ("bicubic", (37, 37), (18, 37), 1024), ("bicubic", (37, 37), (37, 49), 1024),
             ("bicubic_aa", (518, 518), (1024, 1024), 1), ("bicubic_aa", (518, 686), (768, 1024), 1),
             ("bicubic_aa", (1024, 1024), (518, 518), 1)]


@pytest.mark.parametrize("kind, src, dst, C", RESAMPLES)
@pytest.mark.parametrize("dt_in, dt_out", [(f32, f32), (bf16, bf16), (fp16, fp16), (f32, bf16)])
def test_resample_against_its_reference(kc, kind, src, dst, C, dt_in, dt_out):
    from diffusionkit_b200 import depth
    from tests.depth_ref import ref_resample

    g = torch.Generator().manual_seed(src[0] + dst[1] + C)
    x = (torch.randn((*src, C), generator=g) * 40 + 80).to(dt_in)
    ty, tx = depth.Taps.get(kind, src[0], dst[0], DEV), depth.Taps.get(kind, src[1], dst[1], DEV)
    got = depth.resample(x.to(DEV), ty, tx, dt_out)
    tables = [depth.TAPS[kind](src[0], dst[0]), depth.TAPS[kind](src[1], dst[1])]
    want = ref_resample(x, tables[0], tables[1], torch.float64)
    assert got.shape == (*dst, C) and got.dtype == dt_out
    r = _rel(got, want)
    assert r <= (2e-6 if dt_out == f32 else 3e-3), (kind, src, dst, r)
    if kind != "bilinear" and dt_in == f32:
        # the tap tables are PyTorch's interpolate
        mode = "bilinear" if kind.startswith("bilinear") else "bicubic"
        kw = dict(align_corners=kind == "bilinear_ac", antialias=kind == "bicubic_aa")
        it = F.interpolate(x.double().permute(2, 0, 1)[None], size=dst, mode=mode, **kw)[0].permute(1, 2, 0)
        assert _rel(got, it) <= (2e-6 if dt_out == f32 else 3e-3)
    if C == 1:
        rgb = depth.resample(x.to(DEV), ty, tx, dt_out, depth_rgb=True)
        ref = ref_resample(x, tables[0], tables[1], torch.float64, depth_rgb=True)
        assert rgb.shape == (*dst, 3) and _rel(rgb, ref) <= (2e-6 if dt_out == f32 else 3e-3)
        assert torch.equal(rgb[..., 0], rgb[..., 2])


@pytest.mark.parametrize("shape", [(1, 37, 37, 1024), (1, 37, 49, 1024), (2, 8, 8, 64), (1, 5, 7, 128),
                                   (1, 18, 37, 256)])
@pytest.mark.parametrize("dtype", [bf16, fp16])
def test_conv_s2p1_within_conv3x3_bound(kc, shape, dtype):
    from diffusionkit_b200 import depth
    from tests import launch_parity as lp

    B, H, W, C = shape
    x = kc._rand(shape, dtype)
    w = kc._rand((C, 3, 3, C), dtype, (9 * C) ** -0.5)
    b = kc._rand((C,), dtype, 0.5)
    got = depth.conv3x3_s2_p1(x, w, b)
    assert got.shape == (B, (H + 1) // 2, (W + 1) // 2, C)
    want = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), b.float(), stride=2,
                    padding=1).permute(0, 2, 3, 1)
    kc._assert_close(f"conv3x3_s2_p1 {shape}", got.reshape(-1, C), want.reshape(-1, C), lp.TOL16)


@pytest.mark.parametrize("dtype", [bf16, fp16])
def test_add_relu_and_head_tail_bit_for_bit(kc, dtype):
    from diffusionkit_b200 import depth
    from tests.depth_ref import ref_add_relu, ref_head_tail

    for n in ((1, 296, 296, 256), (3, 17, 64)):
        a, b = kc._rand(n, dtype, 3.0), kc._rand(n, dtype, 3.0)
        s, r = torch.empty_like(a), torch.empty_like(a)
        depth.add_relu(a, b, sum_out=s, relu_out=r)
        ws, wr = ref_add_relu(a, b)
        assert torch.equal(s, ws) and torch.equal(r, wr)
        t = depth.add_relu(a, relu_out=torch.empty_like(a))
        assert torch.equal(t, ref_add_relu(a)[1])
        c = a.clone()
        depth.add_relu(c, relu_out=c)
        assert torch.equal(c, ref_add_relu(a)[1])
    for shape, C in (((518, 518), 32), ((518, 686), 32), ((7,), 64)):
        x = kc._rand((*shape, C), dtype, 2.0)
        w = torch.randn(C, device=DEV) * 3
        got = depth.head_tail(x, w, 5.0)
        assert got.dtype == f32 and torch.equal(got, ref_head_tail(x, w, 5.0))


def test_argument_errors_launch_nothing(kc):
    from diffusionkit_b200 import DkError, ops
    from diffusionkit_b200._lib import ptr

    c = ops.ctx(0)
    x = torch.zeros((8, 8, 4), dtype=f32, device=DEV)
    o = torch.empty((16, 16, 4), dtype=f32, device=DEV)
    i0 = torch.zeros(16, dtype=torch.int32, device=DEV)
    wt = torch.zeros(32, dtype=f32, device=DEV)
    t = (ptr(i0), ptr(wt), 2, ptr(i0), ptr(wt), 2)
    xb = torch.zeros((1, 5, 5, 64), dtype=bf16, device=DEV)
    wb = torch.zeros((64, 3, 3, 64), dtype=bf16, device=DEV)
    ob = torch.empty((1, 3, 3, 64), dtype=bf16, device=DEV)
    n0 = c.launches
    for name, args, msg in [
            ("dk_resample", (3, 2, ptr(x), ptr(o), 8, 8, 4, 16, 16) + t + (0,), "input dtype"),
            ("dk_resample", (2, 7, ptr(x), ptr(o), 8, 8, 4, 16, 16) + t + (0,), "output dtype"),
            ("dk_resample", (2, 2, None, ptr(o), 8, 8, 4, 16, 16) + t + (0,), "required"),
            ("dk_resample", (2, 2, ptr(x), ptr(o), 8, 8, 4, 16, 16, None) + t[1:] + (0,), "required"),
            ("dk_resample", (2, 2, ptr(x), ptr(o), 0, 8, 4, 16, 16) + t + (0,), "empty"),
            ("dk_resample", (2, 2, ptr(x), ptr(o), 8, 8, 4, 16, 16, ptr(i0), ptr(wt), 0, ptr(i0), ptr(wt), 2, 0),
             "taps"),
            ("dk_resample", (2, 2, ptr(x), ptr(o), 8, 8, 4, 16, 16) + t + (1,), "mode"),
            ("dk_depth_add_relu", (0, ptr(xb), None, None, None, 64), "sum or relu"),
            ("dk_depth_add_relu", (5, ptr(xb), None, ptr(xb), None, 64), "dtype"),
            ("dk_depth_add_relu", (0, ptr(xb), None, ptr(xb), None, 0), "empty"),
            ("dk_depth_head", (0, ptr(xb), None, 0.0, ptr(x), 4, 32), "required"),
            ("dk_depth_head", (0, ptr(xb), ptr(wt), 0.0, ptr(x), 4, 0), "C <= 1024"),
            ("dk_conv3x3_s2_p1", (0, ptr(xb), ptr(wb[:, :, :, :48].contiguous()), None, ptr(ob), 1, 5, 5, 48, 64),
             "multiple of 64"),
            ("dk_conv3x3_s2_p1", (0, ptr(xb), ptr(wb), None, ptr(ob), 1, 0, 5, 64, 64), "empty"),
            ("dk_conv3x3_s2_p1", (4, ptr(xb), ptr(wb), None, ptr(ob), 1, 5, 5, 64, 64), "dtype")]:
        with pytest.raises(DkError, match=msg):
            c.call(name, *args)
    assert c.launches == n0


# ------------------------------------------------------------------------------------------------ the estimator
def _c_resample(L, a, s, r, census):
    from tests.depth_ref import ref_resample

    ty, tx = a["ty"], a["tx"]
    tabs = [(t.first.cpu().numpy(), t.weights.double().cpu().numpy()) for t in (ty, tx)]
    want = ref_resample(s["x"].cpu(), tabs[0], tabs[1], torch.float64, a["depth_rgb"])
    L.close("out", r.reshape(-1, r.shape[-1]).float(), want.reshape(-1, want.shape[-1]).float().to(r.device),
            2e-6 if r.dtype == f32 else 3e-3)
    L.own(r)
    L.sig.update(src=tuple(s["x"].shape), dst=tuple(r.shape), dtype=str(r.dtype)[6:], rgb=a["depth_rgb"])


def _c_add_relu(L, a, s, r, census):
    from tests.depth_ref import ref_add_relu

    ws, wr = ref_add_relu(s["a"], s["b"])
    if a["sum_out"] is not None:
        L.exact("sum", a["sum_out"], ws)
        L.own(a["sum_out"])
    if a["relu_out"] is not None:
        L.exact("relu", a["relu_out"], wr)
        L.own(a["relu_out"])
    L.sig.update(shape=tuple(s["a"].shape), add=s["b"] is not None, dtype=str(s["a"].dtype)[6:])


def _c_head_tail(L, a, s, r, census):
    from tests.depth_ref import ref_head_tail

    L.exact("depth", r, ref_head_tail(s["x"], s["w"], a["b"]))
    L.own(r)
    L.sig.update(shape=tuple(s["x"].shape), dtype=str(s["x"].dtype)[6:])


def _c_conv3x3_s2_p1(L, a, s, r, census):
    from tests import launch_parity as lp

    want = F.conv2d(s["x"].float().permute(0, 3, 1, 2), s["w"].float().permute(0, 3, 1, 2),
                    None if s["bias"] is None else s["bias"].float(), stride=2, padding=1).permute(0, 2, 3, 1)
    L.close("out", r, want, lp.TOL16, lp.BLK16)
    L.own(r)
    L.sig.update(shape=tuple(s["x"].shape), dtype=str(r.dtype)[6:])


def _c_conv3x3(L, a, s, r, census):
    """tests/launch_parity's conv3x3 check, also for the DPT neck's bias-free convolutions"""
    from tests import launch_parity as lp

    b = s["bias"] if s["bias"] is not None else torch.zeros(r.shape[-1], dtype=r.dtype, device=r.device)
    L.close("out", r, _kc_ref_conv3x3(s["x"], s["w"], b, s["res"]), lp.TOL16, lp.BLK16)
    L.own(r)


def _kc_ref_conv3x3(*args):
    from tests import kernel_checks

    return kernel_checks.ref_conv3x3(*args)


@pytest.fixture
def depth_census(kc, monkeypatch):
    """tests/launch_parity's census over the estimator: every ops launch, plus the estimator's own wrappers"""
    from diffusionkit_b200 import depth
    from tests import launch_parity as lp
    from tests.test_redux_gpu import _c_image_patches

    checks = {"resample": (_c_resample, ["out"]), "add_relu": (_c_add_relu, ["sum_out", "relu_out"]),
              "head_tail": (_c_head_tail, ["out"]), "conv3x3_s2_p1": (_c_conv3x3_s2_p1, ["out"]),
              "image_patches": (_c_image_patches, ["out"])}
    for name, (check, writes) in checks.items():
        monkeypatch.setitem(lp.CHECKS, name, check)
        monkeypatch.setitem(lp.WRITES, name, writes)
    monkeypatch.setitem(lp.CHECKS, "conv3x3", _c_conv3x3)
    c = lp.Census()
    with lp.census(c):
        for name in checks:
            monkeypatch.setattr(depth, name, c._wrap(name, getattr(depth, name)))
        yield c


def _photo(h, w, seed=0):
    from tests.model_checks import _test_image

    return _test_image(h, w, seed=seed)


@pytest.mark.parametrize("which, size", [("tiny", (518, 518)), ("tiny", (518, 686)), ("large4", (518, 518)),
                                         ("large4", (518, 686))])
def test_estimator_against_the_oracle_under_a_census(depth_census, which, size):
    from dataclasses import replace

    from diffusionkit_b200 import depth
    from diffusionkit_b200.config import DEPTH_ANYTHING_LARGE, tiny_depth_anything_config
    from tests.depth_ref import DepthAnythingRef

    cfg = (tiny_depth_anything_config() if which == "tiny"
           else replace(DEPTH_ANYTHING_LARGE, num_hidden_layers=4, out_indices=(1, 2, 3, 4)))
    params = depth.init_depth_params(cfg, seed=5)
    model = depth.DepthAnythingModel(params, cfg, dtype=bf16, device=DEV)
    img = _photo(*size)
    c = depth_census
    c.run = f"{which}-{size[0]}x{size[1]}"
    got = model(torch.from_numpy(img).to(DEV))
    torch.cuda.synchronize()
    print(c.table())
    seen = {r["op"] for r in c.records}
    assert {"image_patches", "gemm", "layernorm", "attention", "conv3x3", "conv3x3_s2_p1", "resample", "add_relu",
            "head_tail"} <= seen, seen
    want = DepthAnythingRef(params, cfg)(torch.from_numpy(img))
    r = _rel(got, want)
    print(f"{which} {size}: predicted_depth rel_l2 {r:.3e}, range {float(want.min()):.1f} .. {float(want.max()):.1f}")
    assert got.shape == want.shape and r <= 2e-2


# ------------------------------------------------------------------------------------------------ pipelines
def _depth_cfg():
    from diffusionkit_b200.config import tiny_depth_anything_config

    return tiny_depth_anything_config()


def _est_params():
    from diffusionkit_b200 import depth

    return depth.init_depth_params(_depth_cfg(), seed=9)


def _oracle(cfg, p16, img, photo, cond, pooled, sig, guidance, solver):
    """the oracle FLUX.1 Depth pipeline with the depth map estimated from the photo by the fp32 oracle estimator"""
    from oracle import sampler_ref as sr
    from oracle.vae_ref import VAEEncoderRef, encode_image_to_latents, read_image_array
    from diffusionkit_b200 import depth
    from tests.depth_ref import DepthAnythingRef, bfl_depth
    from tests.fill_ref import FillMMDiTRef, bfl_pack_latent, fill_pipeline_latents
    from tests.control_ref import _r
    from tests.oracle_bridge import ref_config
    from tests.test_control_gpu import _resized, _vae

    enc = VAEEncoderRef({k: v.float() for k, v in _vae(True).items()})
    ph = _resized(photo, HP, WP)
    pred = DepthAnythingRef(_est_params(), _depth_cfg())(torch.from_numpy(depth.network_input(ph)))
    x = (bfl_depth(pred, (HP, WP)) / 127.5 - 1).to(bf16).float()[None, :, :, None].expand(-1, -1, -1, 3)
    hidden = enc(x.contiguous())
    mean = hidden[..., :hidden.shape[-1] // 2]
    rows = bfl_pack_latent(_r((mean - 0.1159) * 0.3611, bf16))[0]
    image = read_image_array(torch.from_numpy(img))
    x0s = []
    for s in SEEDS:
        eps = sr.get_noise(s, HP // 8, WP // 8)
        x0 = (encode_image_to_latents(enc, image, eps) - 0.1159) * 0.3611
        x0s.append(float(sig[0]) * eps + (1.0 - float(sig[0])) * x0)
    params = {k: v.float() for k, v in p16.items()}
    return fill_pipeline_latents(lambda: FillMMDiTRef(ref_config(cfg), params), solver, sig, x0s, rows, cond, pooled,
                                 guidance, 0.0, bf16, SEEDS)


def _depth_pipe():
    from tests.test_control_gpu import _cfg, _pipe, _vae, _weights

    cfg = _cfg("depth")
    p16, vp16 = _weights(cfg), _vae(False)
    pipe = _pipe(cfg, p16, vp16)
    pipe.load_depth_estimator(_est_params(), config=_depth_cfg())
    return cfg, p16, vp16, pipe


@pytest.mark.parametrize("denoise", [1.0, 0.6])
def test_tiny_pipeline_with_estimate_depth_against_the_oracle(kc, denoise):
    from oracle import sampler_ref as sr
    from tests.model_checks import rel_l2
    from tests.test_control_gpu import _compare, _source

    cfg, p16, vp16, pipe = _depth_pipe()
    pipe.mmdit.use_cuda_graphs = pipe.decoder.use_cuda_graphs = False
    cond, pooled = pipe.synthetic_text_embeddings(n_images=len(SEEDS), text_len=T)
    img, photo = _source(), _photo(90, 150, seed=3)
    sig = sr.get_sigmas(sr.FluxSamplerRef(1.0), STEPS)[int(STEPS * (1 - denoise)):]
    guidance = [30.0, 12.0]
    for solver in ("euler", "dpmpp_2m", "dpmpp_2m_sde"):
        lat, it = pipe.denoise_latents(cond, pooled, num_steps=STEPS, seed=SEEDS, image_path=img, denoise=denoise,
                                       solver=solver, control_image=photo, guidance=guidance, estimate_depth=True)
        torch.cuda.synchronize()
        want = _oracle(cfg, p16, img, photo, cond, pooled, sig, guidance, solver)
        _compare(pipe, vp16, lat, want, f"depth estimate {solver} denoise {denoise}")
        if solver == "euler":
            other = _photo(90, 150, seed=17)
            moved = rel_l2(_oracle(cfg, p16, img, other, cond, pooled, sig, guidance, solver), want)
            print(f"another photo moves the oracle by rel_l2 {moved:.3e}")
            assert moved > 5e-2, "the photo must matter beyond the pipeline bound"


def test_exactness(kc):
    from diffusionkit_b200 import ops
    from tests.test_control_gpu import _cfg, _pipe, _vae, _weights

    cfg, p16, vp16, pipe = _depth_pipe()
    cond, pooled = pipe.synthetic_text_embeddings(n_images=1, text_len=T)
    photo = _photo(HP, WP, seed=4)
    kw = dict(num_steps=STEPS, seed=[5], latent_size=(HP // 8, WP // 8), control_image=photo, guidance=10.0)

    def run(p, **extra):
        n0 = ops.launch_count()
        lat, _ = p.denoise_latents(cond, pooled, **kw, **extra)
        torch.cuda.synchronize()
        return lat.clone(), ops.launch_count() - n0

    a, _ = run(pipe, estimate_depth=True)                       # the first call also captures the CUDA graphs
    b, nb = run(pipe, estimate_depth=True)
    c, nc = run(pipe, estimate_depth=True)
    assert torch.equal(a, b) and torch.equal(b, c) and nb == nc  # reruns repeat bit for bit
    pipe.mmdit.use_cuda_graphs = False
    e, _ = run(pipe, estimate_depth=True)
    pipe.mmdit.use_cuda_graphs = True
    assert torch.equal(a, e)                                    # CUDA graphs equal eager
    # the depth estimate as the control image, and estimate_depth=False on a pipeline that never loaded the estimator
    plain = _pipe(cfg, p16, vp16)
    run(pipe)
    run(plain)
    f1, n1 = run(pipe)
    f2, n2 = run(plain)
    assert torch.equal(f1, f2) and n1 == n2
    assert not torch.equal(f1, a)
    # mask_image keeps the unmasked pixels bit for bit
    src = _photo(HP, WP, seed=6)
    mask = np.zeros((HP, WP), np.uint8)
    mask[:, WP // 2:] = 255
    image, log = pipe.generate_image("", num_steps=STEPS, seed=3, image_path=src, denoise=0.8, mask_image=mask,
                                     conditioning=cond, pooled_conditioning=pooled, control_image=photo,
                                     estimate_depth=True, verbose=False)
    out = np.asarray(image)
    from PIL import Image
    keep = np.asarray(Image.fromarray(src).convert("RGB"))
    assert np.array_equal(out[:, :WP // 2], keep[:, :WP // 2])
    d = log["denoising"]["control"]["depth"]
    assert d["input_size"] == (252, 518) and d["time"] >= 0
    # other models run no estimator work
    from diffusionkit_b200 import depth

    calls = []
    orig = depth.DepthAnythingModel.__call__
    depth.DepthAnythingModel.__call__ = lambda self, *a: calls.append(1) or orig(self, *a)
    try:
        run(pipe)
        canny = _pipe(_cfg("canny"), _weights(_cfg("canny")), vp16)
        canny.denoise_latents(cond, pooled, num_steps=2, seed=[5], latent_size=(HP // 8, WP // 8),
                              control_image=photo, guidance=10.0)
    finally:
        depth.DepthAnythingModel.__call__ = orig
    assert not calls
    est = pipe.estimate_depth(photo)
    assert est.shape == (HP, WP) and est.dtype == torch.float32 and bool(torch.isfinite(est).all())
    assert _vae is not None
