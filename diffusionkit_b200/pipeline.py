"""DiffusionPipeline / FluxPipeline — the reference's Python surface (python/src/diffusionkit/mlx/__init__.py:64-788)
over the H100 engine.  Same constructor arguments, method names, defaults and return structures; the denoise loop and
the decode run entirely in the CUDA kernels of libdkb200.so.

Differences that are deliberate (documented in DESIGN.md):
  * 16-bit only (w16 = a16 = True, what the reference CLI forces, scripts/generate_images.py:117-118);
    fp32 weights/activations raise NotImplementedError.
  * nothing is downloaded (the reference pulls checkpoints, text encoders and vocabularies from the Hugging Face hub in
    its constructor): weights are the deterministic synthetic initialiser of weights.py unless a `params` dict
    (reference parameter names) or `local_ckpt=` (upstream .safetensors, model_io.py) is passed, and `encode_text` works
    once `load_text_encoders(...)` has attached CLIP / T5 weights and tokenizers built from local files — otherwise pass
    `conditioning` / `pooled_conditioning` to generate_image or call denoise_latents.
  * img2img (`image_path`, `denoise`): the VAE encoder is built on first use.
  * batch-N extension: `seed` may be a list of ints — one independent image per seed (the reference is batch 1);
    a scalar seed behaves exactly like the reference.
  * FLUX.1-dev's distilled guidance (`guidance=` of FluxPipeline.generate_image / denoise_latents) when the pipeline is
    built with mmdit_config=FLUX_DEV; the reference loads dev without its guidance embedder (quirk Q1).
  * SD3.5 Medium (model_version "stabilityai/stable-diffusion-3.5-medium") and skip-layer guidance (`slg=` of
    DiffusionPipeline.generate_image / denoise_latents, any SD3-family model under CFG), DESIGN.md §13.
  * FLUX.1 Kontext editing (model_version "black-forest-labs/FLUX.1-Kontext-dev"; `reference_image=` /
    `reference_latents=` of FluxPipeline.generate_image / denoise_latents), DESIGN.md §14.
  * FLUX.1 Redux image prompts (FluxPipeline.load_redux / encode_redux, `redux_image=` of generate_image /
    denoise_latents): SigLIP + Redux tokens appended to the T5 sequence, DESIGN.md §15.
  * stochastic samplers (solver="euler_ancestral" / "dpmpp_2m_sde", `eta=`): per-image Philox noise drawn inside the
    fused CFG + solver kernel, DESIGN.md §16.
  * masked inpainting (`mask_image=` with `image_path`), DESIGN.md §17: diffusers' masked img2img blend after every
    full solver step (after Heun's corrector), except that a latent position is repainted when ANY pixel of its 8 x 8
    block is masked (diffusers samples one pixel), and generate_image always pastes the unmasked source pixels back.
  * FLUX.1 Fill [dev] (model_version "black-forest-labs/FLUX.1-Fill-dev", FluxPipeline with `mask_image=` and
    `image_path`), DESIGN.md §18: the masked source and the mask enter the x-embedder instead of the §17 blend; the
    unmasked source pixels are still pasted back.
  * FLUX.1 Canny / Depth [dev] (model_version "black-forest-labs/FLUX.1-Canny-dev" / "-Depth-dev", FluxPipeline with
    `control_image=`), DESIGN.md §19: the control image's posterior-mean latent enters the x-embedder; a Depth model
    takes the depth map the caller gives, or with `estimate_depth=True` (after FluxPipeline.load_depth_estimator) a
    photo whose depth Depth Anything estimates on the engine's kernels, DESIGN.md §20.
"""
from __future__ import annotations

import math
import time
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import control, depth, fill, inpaint, ops
from ._lib import DkError, dtype_code, ptr
from .config import CONTROL_MODEL_CONFIGS, MODEL_CONFIGS, T5_MAX_LENGTH, MMDiTConfig, VAEDecoderConfig, VAEEncoderConfig
from .mmdit import MMDiT
from .sampler import (FluxSampler, ModelSamplingDiscreteFlow, SkipLayerGuidance, check_eta, check_skip_layer_guidance,
                      dpmpp_2m_coefficients, dpmpp_2m_sde_coefficients, euler_ancestral_coefficients,
                      skip_layer_guidance_steps)
from .vae import VAEDecoder, VAEEncoder
from .weights import init_params, mmdit_param_specs, vae_decoder_param_specs, vae_encoder_param_specs

MMDIT_CKPT = {  # reference mlx/__init__.py:37-44
    "argmaxinc/mlx-stable-diffusion-3-medium": "argmaxinc/mlx-stable-diffusion-3-medium",
    "argmaxinc/mlx-stable-diffusion-3.5-large": "argmaxinc/mlx-stable-diffusion-3.5-large",
    "argmaxinc/mlx-stable-diffusion-3.5-large-4bit-quantized": "argmaxinc/mlx-stable-diffusion-3.5-large-4bit-quantized",
    "argmaxinc/mlx-FLUX.1-schnell": "argmaxinc/mlx-FLUX.1-schnell",
    "argmaxinc/mlx-FLUX.1-schnell-4bit-quantized": "argmaxinc/mlx-FLUX.1-schnell-4bit-quantized",
    "argmaxinc/mlx-FLUX.1-dev": "argmaxinc/mlx-FLUX.1-dev",
    "stabilityai/stable-diffusion-3.5-medium": "stabilityai/stable-diffusion-3.5-medium",
    "black-forest-labs/FLUX.1-Kontext-dev": "black-forest-labs/FLUX.1-Kontext-dev",
    "black-forest-labs/FLUX.1-Fill-dev": "black-forest-labs/FLUX.1-Fill-dev",
    "black-forest-labs/FLUX.1-Canny-dev": "black-forest-labs/FLUX.1-Canny-dev",
    "black-forest-labs/FLUX.1-Depth-dev": "black-forest-labs/FLUX.1-Depth-dev",
}

# FLUX.1-dev's guidance when the caller passes none (BFL's default for the dev checkpoint)
DEFAULT_GUIDANCE = 3.5


class LatentFormat:
    """Base class for latent format conversion (reference mlx/__init__.py:722-733)"""

    def __init__(self):
        self.scale_factor = 1.0
        self.shift_factor = 0.0

    def process_in(self, latent):
        return (latent - self.shift_factor) * self.scale_factor

    def process_out(self, latent):
        return (latent / self.scale_factor) + self.shift_factor


class SD3LatentFormat(LatentFormat):
    def __init__(self):
        super().__init__()
        self.scale_factor = 1.5305
        self.shift_factor = 0.0609


class FluxLatentFormat(LatentFormat):
    def __init__(self):
        super().__init__()
        self.scale_factor = 0.3611
        self.shift_factor = 0.1159


def _bytes2gigabytes(n: int) -> float:
    return n / 1024 ** 3


class CFGDenoiser:
    """Helper for applying CFG scaling to diffusion outputs (reference mlx/__init__.py:674-719).
    x_t is the fp32 sampler state on the device; one call = prepare (cast / CFG doubling) + MMDiT forward; the
    denoised estimate and the Euler update are fused in dk_sampler_step (see sample_euler)."""

    def __init__(self, model: "DiffusionPipeline"):
        self.model = model
        # skip-layer guidance of the running denoise: (SkipLayerGuidance, its steps, [pos | neg | pos] conditioning)
        self.slg = None
        # FLUX.1 Kontext reference latent of the running denoise, one row per forward row (None: no reference)
        self.reference = None
        # masked inpainting of the running denoise (inpaint.InpaintBlend; None: no mask)
        self.inpaint = None

    def cache_modulation_params(self, pooled_text_embeddings, sigmas, guidance=None, skip_batch: int = 0):
        """guidance: one FLUX.1-dev guidance value per row of pooled (None without a guidance embedder).
        skip_batch: the trailing rows of pooled that condition skip-layer guidance's skip forwards"""
        self.model.mmdit.cache_modulation_params(pooled_text_embeddings, sigmas, guidance, skip_batch=skip_batch)

    def slg_scale(self, step) -> float:
        """the skip-layer guidance scale of solver step `step` (0: plain CFG)"""
        return self.slg[0].scale if self.slg is not None and step in self.slg[1] else 0.0

    def inpaint_step(self, x, sigma_next: float):
        """after a full solver step to sigma_next: reset the latent positions a mask keeps to the re-noised source
        (DESIGN.md §17); nothing, and no launch, without a mask"""
        if self.inpaint is not None:
            self.inpaint.blend(x, sigma_next)

    def clear_cache(self):
        # the reference re-reads the adaLN weights it dropped (:686-689); nothing was dropped here
        pass

    def __call__(self, x_t, timestep, sigma, conditioning, cfg_weight: float = 7.5, pooled_conditioning=None,
                 step=None):
        """step: the solver step this evaluation belongs to; inside the skip-layer guidance window the forward runs on
        [pos | neg | pos] with the listed joint blocks skipped for the last third"""
        m = self.model
        reps = 1 if cfg_weight <= 0 else 2
        B = x_t.shape[0]
        skip = {}
        if self.slg is not None and step in self.slg[1]:
            reps, conditioning = 3, self.slg[2]
            skip = dict(skip_layers=self.slg[0].layers, skip_batch=B)
        xin = torch.empty((reps * B,) + tuple(x_t.shape[1:]), dtype=m.activation_dtype, device=x_t.device)
        ops.sampler_prepare(x_t, xin, reps)
        out = m.mmdit(latent_image_embeddings=xin, token_level_text_embeddings=conditioning, timestep=timestep,
                      reference=self.reference, **skip)
        return xin, out


def _start_sampling(model: CFGDenoiser, sigmas, extra_args):
    """What every sampler does first: the timesteps of the schedule (and, for FLUX.1-dev, the per-row guidance values
    extra_args["guidance"]) into the modulation cache; a Kontext reference extra_args["reference"] onto the denoiser.
    -> (sigmas fp32, timesteps, conditioning, cfg_weight, events (one per sigma, the first recorded))"""
    extra_args = {} if extra_args is None else dict(extra_args)
    pipe = model.model
    sig = np.asarray(sigmas, dtype=np.float32)
    # timesteps = sampler.timestep(sigmas).astype(activation_dtype)  (:769-771; quirk Q5)
    timesteps = torch.from_numpy(np.asarray(pipe.sampler.timestep(sig), dtype=np.float32)).to(
        pipe.activation_dtype).to(torch.float32).tolist()
    pooled = extra_args.pop("pooled_conditioning")
    cfg_weight = float(extra_args.get("cfg_weight", 0.0))
    conditioning = extra_args["conditioning"]
    slg = extra_args.pop("slg", None)
    model.reference = extra_args.pop("reference", None)
    model.inpaint = extra_args.pop("inpaint", None)
    steps = skip_layer_guidance_steps(slg, len(sig) - 1) if slg is not None else []
    skip_batch = 0
    if steps:
        # rows [pos x B | neg x B | pos x B]: the forwards inside the window skip the listed blocks for the last B
        skip_batch = pooled.shape[0] // 2
        pooled = torch.cat([pooled, pooled[:skip_batch]])
        model.slg = (slg, frozenset(steps), torch.cat([conditioning, conditioning[:skip_batch]]))
    model.cache_modulation_params(pooled, timesteps, extra_args.pop("guidance", None), skip_batch)
    events = [torch.cuda.Event(enable_timing=True) for _ in range(len(sig))]
    events[0].record()
    return sig, timesteps, conditioning, cfg_weight, events


def _finish_sampling(model: CFGDenoiser, events):
    """-> iter_time: seconds per step, from the events recorded after each step"""
    model.clear_cache()
    model.slg = None
    model.reference = None
    model.inpaint = None
    torch.cuda.current_stream().synchronize()  # the reference syncs every step (mx.eval, :782); once is enough here
    return [round(events[i].elapsed_time(events[i + 1]) / 1e3, 3) for i in range(len(events) - 1)]


def sample_euler(model: CFGDenoiser, x, sigmas, extra_args=None):
    """Implements Algorithm 2 (Euler steps) from Karras et al. (2022) — reference mlx/__init__.py:761-788.
    x: (B, H, W, 16) fp32 device tensor (updated in place); sigmas: 1-D float32 numpy/torch array."""
    sig, timesteps, conditioning, cfg_weight, events = _start_sampling(model, sigmas, extra_args)
    for i in range(len(sig) - 1):
        xin, out = model(x, timesteps[i], float(sig[i]), conditioning, cfg_weight, step=i)
        # denoised = xin - out * sigma; CFG mix; d = (x - denoised) / sigma; x += d * (sigma_next - sigma)
        ops.sampler_step(x, xin, out, float(sig[i]), float(sig[i + 1]), cfg_weight, slg=model.slg_scale(i))
        model.inpaint_step(x, float(sig[i + 1]))
        events[i + 1].record()
    return x, _finish_sampling(model, events)


def sample_heun(model: CFGDenoiser, x, sigmas, extra_args=None):
    """Heun's method, Algorithm 2 of Karras et al. (2022) without churn, on the ODE sample_euler integrates: an Euler
    predictor to x2, then a corrector with the slope at (x2, sigma_next) — two forwards per step; a step to sigma = 0
    is the plain Euler step.  Same arguments and return value as sample_euler; iter_time has one entry per step."""
    sig, timesteps, conditioning, cfg_weight, events = _start_sampling(model, sigmas, extra_args)
    d = x2 = None
    for i in range(len(sig) - 1):
        s, s_next = float(sig[i]), float(sig[i + 1])
        slg = model.slg_scale(i)                      # both evaluations of a step take that step's decision
        xin, out = model(x, timesteps[i], s, conditioning, cfg_weight, step=i)
        if s_next == 0.0:
            ops.sampler_step(x, xin, out, s, s_next, cfg_weight, slg=slg)
        else:
            if d is None:
                d, x2 = torch.empty_like(x), torch.empty_like(x)
            ops.sampler_heun_predict(x, xin, out, s, s_next, cfg_weight, d, x2, slg=slg)
            xin, out = model(x2, timesteps[i + 1], s_next, conditioning, cfg_weight, step=i)
            ops.sampler_heun_correct(x, d, x2, xin, out, s, s_next, cfg_weight, slg=slg)
        model.inpaint_step(x, s_next)                 # after the full step: the predictor's x2 is not blended
        events[i + 1].record()
    return x, _finish_sampling(model, events)


def sample_dpmpp_2m(model: CFGDenoiser, x, sigmas, extra_args=None):
    """DPM-Solver++(2M) (Lu et al. 2022) on the same ODE: one forward per step, the previous step's denoised estimate
    kept on the device; coefficients from sampler.dpmpp_2m_coefficients.  Same arguments and return value as
    sample_euler."""
    sig, timesteps, conditioning, cfg_weight, events = _start_sampling(model, sigmas, extra_args)
    coef = dpmpp_2m_coefficients(sig)
    d_prev = torch.empty_like(x)
    for i in range(len(sig) - 1):
        xin, out = model(x, timesteps[i], float(sig[i]), conditioning, cfg_weight, step=i)
        a, b, c = (float(v) for v in coef[i])
        ops.sampler_dpmpp_2m(x, d_prev, xin, out, float(sig[i]), a, b, c, cfg_weight, slg=model.slg_scale(i))
        model.inpaint_step(x, float(sig[i + 1]))      # d_prev stays the unblended history
        events[i + 1].record()
    return x, _finish_sampling(model, events)


def seeds_tensor(seeds, device) -> torch.Tensor:
    """per-image 64-bit noise seeds -> the (B,) uint64 device array dk_sampler_sde_step reads"""
    vals = [int(s) for s in seeds]
    if not all(0 <= s < 2 ** 64 for s in vals):
        raise ValueError(f"noise seeds must be in [0, 2^64), got {vals}")
    return torch.from_numpy(np.asarray(vals, dtype=np.uint64)).to(device)


def sampler_sde_step(x, d_prev, xin, out, sigma: float, a: float, b: float, c: float, noise: float, cfg_weight: float,
                     slg: float, seeds: torch.Tensor, step: int):
    """dk_sampler_sde_step: x = a x + b D + c d_prev + noise z, then d_prev = D (both in place; d_prev None: neither
    read nor written, c must be 0).  x (B, ...) fp32; xin / out hold 1, 2 or 3 replicas of x's rows (no CFG, CFG, CFG +
    skip-layer guidance); z is image b's Philox normal of `step` under seeds[b] (DESIGN.md §16).  Kept beside its
    callers rather than in ops: the launch census of the shipped models requires a reference for every launching op
    there, and this one runs only under a stochastic solver, whose GPU test runs a census of its own that wraps it."""
    assert x.dtype == torch.float32 and x.is_contiguous() and xin.is_contiguous() and out.is_contiguous()
    assert d_prev is None or (d_prev.dtype == torch.float32 and d_prev.is_contiguous() and d_prev.shape == x.shape)
    B = x.shape[0]
    assert seeds.dtype == torch.uint64 and tuple(seeds.shape) == (B,) and seeds.device == x.device
    cx = ops.ctx(x.device.index)
    cx.call("dk_sampler_sde_step", dtype_code(xin.dtype), ptr(x), ptr(d_prev), ptr(xin), ptr(out), x.numel() // B, B,
            xin.numel() // x.numel(), sigma, a, b, c, noise, cfg_weight, slg, ptr(seeds), step)
    return x


def _sample_sde(model: CFGDenoiser, x, sigmas, extra_args, coefficients, keep_d: bool):
    """the loop both stochastic samplers share: one forward and one dk_sampler_sde_step per step.  extra_args["eta"]
    (None: 1.0) scales the noise, extra_args["seeds"] holds one noise seed per image of x."""
    extra_args = dict(extra_args or {})
    if "seeds" not in extra_args:
        raise ValueError("a stochastic sampler needs extra_args['seeds']: one noise seed per image")
    eta = extra_args.pop("eta", None)
    coef = coefficients(np.asarray(sigmas, dtype=np.float32), 1.0 if eta is None else eta)
    seeds = seeds_tensor(extra_args.pop("seeds"), x.device)            # one upload per call
    sig, timesteps, conditioning, cfg_weight, events = _start_sampling(model, sigmas, extra_args)
    d_prev = torch.empty_like(x) if keep_d else None
    for i in range(len(sig) - 1):
        xin, out = model(x, timesteps[i], float(sig[i]), conditioning, cfg_weight, step=i)
        a, b, c, n = (float(v) for v in coef[i])
        sampler_sde_step(x, d_prev, xin, out, float(sig[i]), a, b, c, n, cfg_weight, model.slg_scale(i), seeds, i)
        model.inpaint_step(x, float(sig[i + 1]))
        events[i + 1].record()
    return x, _finish_sampling(model, events)


def sample_euler_ancestral(model: CFGDenoiser, x, sigmas, extra_args=None):
    """Euler ancestral for the rectified-flow ODE sample_euler integrates (sampler.euler_ancestral_coefficients): an
    Euler step to sigma_down, rescaled, plus fresh noise, one forward per step.  extra_args as for sample_euler, plus
    "seeds" (one per image, required) and "eta" (None: 1.0; 0: Euler).  Same return value as sample_euler."""
    return _sample_sde(model, x, sigmas, extra_args, euler_ancestral_coefficients, keep_d=False)


def sample_dpmpp_2m_sde(model: CFGDenoiser, x, sigmas, extra_args=None):
    """DPM-Solver++(2M) SDE (Lu et al. 2022; sampler.dpmpp_2m_sde_coefficients), one forward per step, the previous
    step's denoised estimate kept on the device.  extra_args as for sample_euler_ancestral; eta = 0 is sample_dpmpp_2m
    bit for bit.  Same return value as sample_euler."""
    return _sample_sde(model, x, sigmas, extra_args, dpmpp_2m_sde_coefficients, keep_d=True)


# the deterministic (ODE) solvers, and the stochastic ones, which take `eta` and draw per-image noise every step
SOLVERS = {"euler": sample_euler, "heun": sample_heun, "dpmpp_2m": sample_dpmpp_2m}
SDE_SOLVERS = {"euler_ancestral": sample_euler_ancestral, "dpmpp_2m_sde": sample_dpmpp_2m_sde}


def _check_solver(solver: str, eta=None):
    """the solver name and its eta, refused with ValueError before any GPU work"""
    if solver not in SOLVERS and solver not in SDE_SOLVERS:
        raise ValueError(f"unknown solver {solver!r}: expected one of "
                         f"{', '.join(repr(k) for k in (*SOLVERS, *SDE_SOLVERS))}")
    if eta is not None:
        if solver not in SDE_SOLVERS:
            raise ValueError(f"eta scales the noise of the stochastic solvers ({', '.join(map(repr, SDE_SOLVERS))}); "
                             f"solver {solver!r} is deterministic")
        check_eta(eta)


def _check_slg(slg, cfg_weight: float, config: MMDiTConfig):
    """skip-layer guidance arguments, refused with ValueError before any GPU work"""
    if slg is None:
        return
    if config.depth_unified > 0:
        raise ValueError("skip-layer guidance runs on SD3-family models only, not on a FLUX-shaped config")
    check_skip_layer_guidance(slg, cfg_weight, config.depth_multimodal)


def _load_image_sized(image) -> Tuple[np.ndarray, Tuple[int, int]]:
    """-> (uint8 (H, W, >=3) with H, W multiples of 64 (read_image's resize rule, :540-546), (width, height) of the
    image as given)"""
    from PIL import Image

    if isinstance(image, (str, bytes)) or hasattr(image, "__fspath__"):
        image = Image.open(image)
    if isinstance(image, np.ndarray):
        if image.dtype != np.uint8 or image.ndim != 3 or image.shape[2] < 3:
            raise ValueError("image array must be uint8 (H, W, >=3)")
        image = Image.fromarray(image[:, :, :3])
    size = (image.width, image.height)
    W, H = (dim - dim % 64 for dim in size)
    if W == 0 or H == 0:
        raise ValueError(f"image {image.width}x{image.height} is smaller than 64x64")
    if W != image.width or H != image.height:
        image = image.resize((W, H), Image.LANCZOS)
    arr = np.asarray(image)
    if arr.ndim == 2:
        raise ValueError("greyscale images are not supported (the reference indexes img[:, :, :3])")
    return np.ascontiguousarray(arr), size


class DiffusionPipeline:
    _default_model = "argmaxinc/mlx-stable-diffusion-3-medium"

    def __init__(
        self,
        w16: bool = False,
        shift: float = 1.0,
        use_t5: bool = True,
        model_version: str = "argmaxinc/mlx-stable-diffusion-3-medium",
        low_memory_mode: bool = True,
        a16: bool = False,
        local_ckpt=None,
        *,
        device: Optional[Union[int, str, torch.device]] = None,
        params: Optional[Dict[str, torch.Tensor]] = None,
        vae_params: Optional[Dict[str, torch.Tensor]] = None,
        mmdit_config: Optional[MMDiTConfig] = None,
        weight_seed: int = 0,
        load_decoder: bool = True,
        vae_encoder_params: Optional[Dict[str, torch.Tensor]] = None,
        load_encoder: bool = False,
    ):
        self.float16_dtype = torch.float16                                  # :76 (quirk Q10)
        self._vae_encoder_params, self._load_encoder = vae_encoder_params, load_encoder
        self._setup(w16, a16, shift, model_version, low_memory_mode, local_ckpt, device, params, vae_params,
                    mmdit_config, weight_seed, load_decoder)
        self.use_t5 = use_t5
        self.sampler = ModelSamplingDiscreteFlow(shift=shift)
        self.latent_format = SD3LatentFormat()
        self.use_clip_g = True

    def _setup(self, w16, a16, shift, model_version, low_memory_mode, local_ckpt, device, params, vae_params,
               mmdit_config, weight_seed, load_decoder):
        self.mmdit_ckpt = MMDIT_CKPT[model_version]                          # KeyError on unknown model (:81)
        if not (w16 and a16):
            raise NotImplementedError(
                "the H100 engine computes in 16-bit only: pass w16=True, a16=True (what the reference CLI forces, "
                "scripts/generate_images.py:117-118)")
        self._local_ckpt = local_ckpt
        self.dtype = self.float16_dtype
        self.activation_dtype = self.float16_dtype
        self.low_memory_mode = low_memory_mode
        self.model_version = model_version
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else None
        if device is None:
            raise DkError("no CUDA device: diffusionkit_b200 runs on H100 only; there is no CPU fallback")
        self.device = torch.device(device) if not isinstance(device, int) else torch.device("cuda", device)
        if mmdit_config is not None:
            self.config = mmdit_config
        else:
            self.config = MODEL_CONFIGS.get(model_version) or CONTROL_MODEL_CONFIGS[model_version]
        self._weight_seed = weight_seed
        self._params, self._vae_params = params, vae_params
        self._load_decoder = load_decoder
        self._loras = {}                            # adapter name -> [lora.LoRA, scale], in load order
        self.check_and_load_models()
        self._params = self._vae_params = None      # the models hold packed copies; drop the caller's tensors
        if hasattr(self, "encoder"):
            self._vae_encoder_params = None

    # ------------------------------------------------------------------ model loading (:90-143)
    def _load_local_ckpt(self):
        """`local_ckpt`: path of an upstream .safetensors file (BFL FLUX / Stability SD3 layout), or a dict
        {"mmdit": path, "vae": path}.  Key remapping: model_io.py (reference mlx/model_io.py:130-486)."""
        from . import model_io

        ck = self._local_ckpt
        paths = ck if isinstance(ck, dict) else {"mmdit": ck}
        out = {}
        if paths.get("mmdit"):
            sd = model_io.load_safetensors(paths["mmdit"])
            if self.model_version.endswith("-4bit-quantized"):
                # saved from the reference's own module tree: names already final, Linear weights as MLX 4-bit triples
                # (reference model_io.py:728-734 SD3.5, :772-775 FLUX); expanded to dense 16-bit once, here
                flux = isinstance(self, FluxPipeline)
                tree = model_io.preadjusted_checkpoint_to_params(sd, "" if flux else "model.diffusion_model.")
                if flux:
                    tree = {k: v for k, v in tree.items() if not k.startswith(("decoder.", "encoder."))}
                params = model_io.dequantize_q4_params(tree, self.device, self.dtype)
                if not flux and "vae" not in paths:
                    for part, pref in (("vae", "first_stage_model.decoder."), ("vae_encoder", "first_stage_model.encoder.")):
                        sub = model_io.preadjusted_checkpoint_to_params(sd, pref)
                        if sub:
                            out[part] = sub
            elif isinstance(self, FluxPipeline):
                params = model_io.flux_checkpoint_to_params(sd, self.config.hidden_size, self.config.mlp_ratio,
                                                            guidance_embed=self.config.guidance_embed,
                                                            cond_channels=self.config.x_embedder_cond_channels)
            else:
                params = model_io.sd3_checkpoint_to_params(sd, k_bias=self.config.attn_k_bias)
                if "vae" not in paths and any("decoder." in k for k in sd):
                    out["vae"] = model_io.vae_decoder_checkpoint_to_params(sd)     # single-file SD3 checkpoints
                if "vae" not in paths and any("encoder.down." in k for k in sd):
                    out["vae_encoder"] = model_io.vae_encoder_checkpoint_to_params(sd)
            model_io.check_against_specs(params, mmdit_param_specs(self.config))
            out["mmdit"] = params
        if paths.get("vae"):
            vsd = model_io.load_safetensors(paths["vae"])
            out["vae"] = model_io.vae_decoder_checkpoint_to_params(vsd)
            if any("encoder.down." in k for k in vsd):                             # ae.safetensors holds both halves
                out["vae_encoder"] = model_io.vae_encoder_checkpoint_to_params(vsd)
        if "vae" in out:
            model_io.check_against_specs(out["vae"], vae_decoder_param_specs(VAEDecoderConfig()))
        if "vae_encoder" in out:
            model_io.check_against_specs(out["vae_encoder"], vae_encoder_param_specs(VAEEncoderConfig()))
        return out

    def load_mmdit(self, only_modulation_dict=False):
        params = self._params
        if params is None and self._local_ckpt is not None:
            loaded = self._load_local_ckpt()
            params = loaded.get("mmdit")
            if self._vae_params is None:
                self._vae_params = loaded.get("vae")
            if self._vae_encoder_params is None:
                self._vae_encoder_params = loaded.get("vae_encoder")
            if params is not None:
                params = {k: v.to(device=self.device, dtype=self.dtype) for k, v in params.items()}
        if params is None:
            params = init_params(mmdit_param_specs(self.config), seed=self._weight_seed, dtype=self.dtype,
                                 device=self.device)
        self.mmdit = MMDiT(self.config, params, device=self.device)

    def check_and_load_models(self):
        if not hasattr(self, "mmdit"):
            self.load_mmdit()
        if not hasattr(self, "decoder") and self._load_decoder:
            vp = self._vae_params
            if vp is None:
                vp = init_params(vae_decoder_param_specs(VAEDecoderConfig()), seed=self._weight_seed + 1,
                                 dtype=self.dtype, device=self.device)
            self.decoder = VAEDecoder(vp, VAEDecoderConfig(), device=self.device)
        if not hasattr(self, "encoder") and self._load_encoder:
            self.load_encoder()

    def load_encoder(self):
        """reference check_and_load_models (:115-116) loads the encoder eagerly; here it is built on the first img2img
        call (or at construction with load_encoder=True) so text-to-image runs do not carry its 34 M parameters."""
        ep = self._vae_encoder_params
        if ep is None:
            ep = init_params(vae_encoder_param_specs(VAEEncoderConfig()), seed=self._weight_seed + 2,
                             dtype=self.dtype, device=self.device)
        else:
            ep = {k: v.to(device=self.device, dtype=self.dtype) for k, v in ep.items()}
        self.encoder = VAEEncoder(ep, VAEEncoderConfig(), device=self.device)
        self._vae_encoder_params = None

    # ------------------------------------------------------------------ LoRA adapters (DESIGN.md §8)
    def load_lora_weights(self, path_or_dict, scale: float = 1.0, adapter_name: Optional[str] = None) -> str:
        """Load a kohya or PEFT LoRA (.safetensors path or state dict) for the MMDiT and merge it into the weights
        together with the adapters already loaded.  Returns the adapter's name (default: the file name without its
        extension, or "adapter")."""
        from .lora import load_lora

        lora = load_lora(path_or_dict, self.config, name=adapter_name)
        if lora.name in self._loras:
            raise ValueError(f"a LoRA adapter named {lora.name!r} is already loaded: pass another adapter_name")
        self._loras[lora.name] = [lora, float(scale)]
        try:
            self._apply_loras()
        except Exception:
            del self._loras[lora.name]
            self._apply_loras()
            raise
        return lora.name

    def set_lora_scale(self, adapter_name: str, scale: float):
        """Change one adapter's scale and re-merge the stack (in place: captured CUDA graphs keep replaying)."""
        if adapter_name not in self._loras:
            raise KeyError(f"no LoRA adapter named {adapter_name!r} is loaded")
        old = self._loras[adapter_name][1]
        self._loras[adapter_name][1] = float(scale)
        try:
            self._apply_loras()
        except Exception:
            self._loras[adapter_name][1] = old
            self._apply_loras()
            raise

    def unload_lora_weights(self, adapter_name: Optional[str] = None):
        """Remove one adapter (or all of them with None) and re-merge the rest; with none left the MMDiT runs on its
        original weights again, bit for bit."""
        if adapter_name is None:
            self._loras.clear()
        elif adapter_name not in self._loras:
            raise KeyError(f"no LoRA adapter named {adapter_name!r} is loaded")
        else:
            del self._loras[adapter_name]
        self._apply_loras()

    @property
    def lora_adapters(self) -> Dict[str, float]:
        """{adapter name: scale} of the loaded adapters, in load order"""
        return {n: s for n, (_, s) in self._loras.items()}

    def _apply_loras(self):
        self.mmdit.apply_lora([(lora, s) for lora, s in self._loras.values()])

    # ------------------------------------------------------------------ FP8 linears (DESIGN.md "FP8 linears")
    def set_fp8(self, enabled: bool):
        """Run the MMDiT's block linears in e4m3 (MMDiT.set_fp8): faster, less accurate; off by default."""
        self.mmdit.set_fp8(enabled)

    @property
    def fp8(self) -> bool:
        return self.mmdit.fp8

    # ------------------------------------------------------------------ step cache (DESIGN.md §10)
    def set_step_cache(self, threshold: Optional[float], max_consecutive_skips: Optional[int] = None):
        """Skip the MMDiT blocks after the first on denoise steps whose first-block residual changed by less than
        `threshold` (relative L1) since the last full step (MMDiT.set_step_cache): faster, less accurate; off by
        default, None turns it off.  generate_image then logs each step's change and decision."""
        self.mmdit.set_step_cache(threshold, max_consecutive_skips)

    @property
    def step_cache(self) -> Optional[Tuple[float, Optional[int]]]:
        """(threshold, max_consecutive_skips) while the step cache is on, else None"""
        return self.mmdit.step_cache

    # ------------------------------------------------------------------ text (SURVEY.md §8 row f2)
    def load_text_encoders(self, clip_l=None, clip_g=None, t5=None, *, tokenizer_l=None, tokenizer_g=None,
                           t5_tokenizer=None, clip_l_config=None, clip_g_config=None, t5_config=None):
        """Build CLIP-L (+ CLIP-G for SD3) and the T5 encoder on the device, and attach their tokenizers.
        clip_l / clip_g / t5: parameter dicts with the reference's names (model_io.clip_checkpoint_to_params /
        t5_checkpoint_to_params convert upstream safetensors), or None for the deterministic synthetic initialiser.
        tokenizer_*: tokenizer.Tokenizer / tokenizer.T5Tokenizer objects built from local vocabulary files (the
        reference downloads all of this in check_and_load_models, :118-143; no network here)."""
        from .config import CLIP_G, CLIP_L, T5EncoderConfig
        from .text_encoders import CLIPTextModel, SD3T5Encoder, clip_param_specs, t5_param_specs

        def build(cls, params, cfg, specs, seed, dtype=None):
            dtype = dtype or self.dtype
            if params is None:
                params = init_params(specs(cfg), seed=self._weight_seed + seed, dtype=dtype, device=self.device)
            return cls({k: v.to(device=self.device, dtype=dtype) for k, v in params.items()}, cfg, device=self.device)

        self.clip_l = build(CLIPTextModel, clip_l, clip_l_config or CLIP_L, clip_param_specs, 3)
        if self.use_clip_g:
            self.clip_g = build(CLIPTextModel, clip_g, clip_g_config or CLIP_G, clip_param_specs, 4)
        if self.use_t5:
            # T5-XXL's feed-forward overflows fp16 — the reference runs it in fp32 for that reason (t5.py:214-224).
            # Here its GEMMs take 16-bit inputs, so the T5 stack always computes in bf16 (fp32's range), also
            # inside the fp16 SD3 pipeline; the output is cast to the activation dtype.
            self.t5_encoder = build(SD3T5Encoder, t5, t5_config or T5EncoderConfig(), t5_param_specs, 5,
                                    dtype=torch.bfloat16)
        self.tokenizer_l, self.tokenizer_g, self.t5_tokenizer = tokenizer_l, tokenizer_g, t5_tokenizer

    def _need_text_stack(self, *names):
        missing = [n for n in names if getattr(self, n, None) is None]
        if missing:
            raise DkError(
                f"encode_text needs {', '.join(missing)}: call load_text_encoders(...) with local weights and "
                "tokenizer files first (nothing can be downloaded here), or pass `conditioning` / `pooled_conditioning`")

    def _tokenize(self, tokenizer, text: str, negative_text: Optional[str] = None):
        """reference :174-195 — note that a None negative prompt becomes "" first, so two rows always come back (Q11)"""
        if negative_text is None:
            negative_text = ""
        pad_token = tokenizer.eos_token if tokenizer.pad_with_eos else 0
        tokens = [list(tokenizer.tokenize(text))]
        if tokenizer.pad_to_max_length:
            tokens[0].extend([pad_token] * (tokenizer.max_length - len(tokens[0])))
        tokens += [list(tokenizer.tokenize(negative_text))]
        N = max(len(t) for t in tokens)
        tokens = [t + [pad_token] * (N - len(t)) for t in tokens]
        return torch.tensor(tokens, dtype=torch.int64)

    def encode_text(self, text: str, cfg_weight: float = 7.5, negative_text: str = ""):
        """reference :197-251 -> (conditioning (2, 77 + T5, 4096), pooled (2, 2048)) in the activation dtype"""
        need = ["clip_l", "tokenizer_l", "clip_g", "tokenizer_g"] + (["t5_encoder", "t5_tokenizer"] if self.use_t5 else [])
        self._need_text_stack(*need)
        neg = negative_text if cfg_weight > 1 else None
        cl = self.clip_l(self._tokenize(self.tokenizer_l, text, neg))
        cg = self.clip_g(self._tokenize(self.tokenizer_g, text, neg))
        conditioning = torch.cat([cl.hidden_states[-2], cg.hidden_states[-2]], dim=-1)
        pooled_conditioning = torch.cat([cl.pooled_output, cg.pooled_output], dim=-1)
        pad = torch.zeros((conditioning.shape[0], conditioning.shape[1], 4096 - conditioning.shape[2]),
                          dtype=conditioning.dtype, device=self.device)
        conditioning = torch.cat([conditioning, pad], dim=-1)
        if self.use_t5:
            t5_conditioning = self.t5_encoder(self._tokenize(self.t5_tokenizer, text, neg)).to(conditioning.dtype)
        else:
            t5_conditioning = torch.zeros_like(conditioning)
        conditioning = torch.cat([conditioning, t5_conditioning], dim=1)
        return conditioning, pooled_conditioning

    def text_shapes(self, cfg_weight: float) -> Tuple[Tuple[int, int], Tuple[int, int]]:
        """(conditioning (Bc, T, 4096), pooled (Bc, P)) shapes the reference produces for ONE image."""
        c = self.config
        if isinstance(self, FluxPipeline):
            return (1, T5_MAX_LENGTH.get(self.model_version, 256), c.token_level_text_embed_dim), (
                1, c.pooled_text_embed_dim)
        T = 77 + (T5_MAX_LENGTH.get(self.model_version, 512) if self.use_t5 else 77)    # :186-187, :239-249 (Q2)
        return (2, T, c.token_level_text_embed_dim), (2, c.pooled_text_embed_dim)        # always 2 (Q11)

    def synthetic_text_embeddings(self, n_images: int = 1, seed: int = 1234, text_len: Optional[int] = None):
        """N(0,1) stand-ins for encode_text's outputs (SURVEY.md §8d), laid out [positive(n) | negative(n)] for SD3."""
        (bc, T, E), (_, P) = self.text_shapes(1.0)
        if text_len is not None:
            T = text_len
        g = torch.Generator(device="cpu").manual_seed(seed)
        cond = torch.randn((bc * n_images, T, E), generator=g, dtype=torch.float32)
        pooled = torch.randn((bc * n_images, P), generator=g, dtype=torch.float32)
        return cond.to(self.activation_dtype), pooled.to(self.activation_dtype)

    # ------------------------------------------------------------------ denoise (:253-292)
    def denoise_latents(
        self,
        conditioning,
        pooled_conditioning,
        num_steps: int = 2,
        cfg_weight: float = 0.0,
        latent_size: Tuple[int, int] = (64, 64),
        seed=None,
        image_path: Optional[str] = None,
        denoise: float = 1.0,
        *,
        noise: Optional[torch.Tensor] = None,
        solver: str = "euler",
        slg: Optional[SkipLayerGuidance] = None,
        eta: Optional[float] = None,
        mask_image=None,
    ):
        """-> (latent NHWC (B, H, W, 16) fp32 on the device, iter_time list).  `noise` (optional, device fp32
        (B, H, W, 16)) replaces the host-side numpy draw of get_noise for callers whose inputs already live in HBM.
        `image_path` (img2img): a file path, a PIL image or a uint8 HWC array; the latent size then follows the image
        (the reference ignores latent_size in that case too, :273).  `solver`: "euler" (the reference's sampler),
        "heun" (two model evaluations per step but the last) or "dpmpp_2m" (one per step), DESIGN.md §11; or the
        stochastic "euler_ancestral" and "dpmpp_2m_sde" (one per step, fresh noise drawn on the device every step from
        each image's seed), DESIGN.md §16.  `eta`: the stochastic solvers' noise scale, >= 0 (None: 1.0; 0: the
        deterministic step, for "dpmpp_2m_sde" exactly "dpmpp_2m"); a deterministic solver refuses it.
        `slg`: skip-layer guidance (sampler.SkipLayerGuidance, needs cfg_weight > 0; None: off), DESIGN.md §13.
        `mask_image` (masked inpainting, needs image_path; DESIGN.md §17): a path, a PIL image or a uint8 (H, W) /
        (H, W, 1|3|4) array of the source image's size; white (>= 128 in grayscale) marks what to regenerate.  After
        every solver step the other latent positions are reset to the re-noised source, so the returned latent holds
        the encoded source there exactly; one mask for all seeds."""
        return self._denoise_latents(conditioning, pooled_conditioning, num_steps, cfg_weight, latent_size, seed,
                                     image_path, denoise, noise=noise, solver=solver, guidance=None, slg=slg, eta=eta,
                                     mask_image=mask_image)

    def _guidance_values(self, guidance, n_images: int) -> Optional[List[float]]:
        """FluxPipeline's `guidance` -> one FLUX.1-dev guidance value per image, or None for a model without a
        guidance embedder.  Raises ValueError, before any GPU work, for a value the model cannot take."""
        if not self.config.guidance_embed:
            if guidance is not None:
                raise ValueError("guidance is FLUX.1-dev's distilled guidance, and this model has no guidance embedder:"
                                 " build the pipeline with mmdit_config=FLUX_DEV (or guidance_embed=True)")
            return None
        if guidance is None:
            if self.config.control:
                guidance = control.DEFAULT_GUIDANCE[self.config.control]
            else:
                guidance = fill.DEFAULT_GUIDANCE if self.config.x_embedder_cond_channels else DEFAULT_GUIDANCE
        if np.ndim(guidance) == 0:
            vals = [float(guidance)] * n_images
        else:
            vals = [float(g) for g in guidance]
            if len(vals) != n_images:
                raise ValueError(f"guidance has {len(vals)} values for {n_images} image(s): pass one float, or one "
                                 "per seed")
        if not all(math.isfinite(g) for g in vals):
            raise ValueError(f"guidance must be finite, got {vals}")
        return vals

    def _check_fill(self, image_path, mask_image, reference_image, reference_latents):
        """FLUX.1 Fill's arguments, refused with ValueError before any GPU work (nothing to check on other models)"""
        if not self.config.x_embedder_cond_channels or self.config.control:
            return
        if not isinstance(self, FluxPipeline):
            raise ValueError("a FLUX.1 Fill config (x_embedder_cond_channels) runs in FluxPipeline only")
        if image_path is None or mask_image is None:
            raise ValueError("FLUX.1 Fill needs image_path and mask_image: the model is conditioned on the masked "
                             "source and the mask")
        if reference_image is not None or reference_latents is not None:
            raise ValueError("FLUX.1 Fill takes no Kontext reference")

    def _check_control(self, control_image, canny_thresholds, reference_image, reference_latents,
                       estimate_depth=False):
        """FLUX.1 Canny / Depth's arguments, refused with ValueError (DkError for a missing depth estimator) before
        any GPU work -> canny_thresholds checked ((low, high) or None) on a Canny model, None otherwise"""
        kind = self.config.control
        if estimate_depth:
            if kind != "depth" or not isinstance(self, FluxPipeline):
                raise ValueError("estimate_depth runs on a FLUX.1 Depth model in FluxPipeline only")
            if control_image is None:
                raise ValueError("estimate_depth needs control_image: the photo the depth map is estimated from")
            self._need_depth_estimator()
        if kind != "canny" and canny_thresholds != control.DEFAULT_THRESHOLDS:
            raise ValueError("canny_thresholds applies to a FLUX.1 Canny model only")
        if kind is None:
            if control_image is not None:
                raise ValueError("control_image conditions a FLUX.1 Canny or Depth model (config.control); this model "
                                 "has none")
            return None
        if kind not in control.KINDS:
            raise ValueError(f"config.control must be one of {control.KINDS}, got {kind!r}")
        if self.config.x_embedder_cond_channels != control.LATENT_CHANNELS:
            raise ValueError(f"a {kind} control model takes {control.LATENT_CHANNELS} conditioning channels, the "
                             f"config has x_embedder_cond_channels = {self.config.x_embedder_cond_channels}")
        name = f"FLUX.1 {kind.capitalize()}"
        if not isinstance(self, FluxPipeline):
            raise ValueError(f"a {name} config runs in FluxPipeline only")
        if control_image is None:
            raise ValueError(f"{name} needs control_image: the model is conditioned on it")
        if reference_image is not None or reference_latents is not None:
            raise ValueError(f"{name} takes no Kontext reference")
        return control.check_thresholds(canny_thresholds) if kind == "canny" else None

    def _reference_input(self, reference_image, reference_latents, n_images: int):
        """FluxPipeline's Kontext reference -> None, or (uint8 HWC image or fp32 latents, its (Hr, Wr) latent size).
        Raises ValueError, before any GPU work, for a reference the pipeline cannot take."""
        if reference_image is None and reference_latents is None:
            return None
        if reference_image is not None and reference_latents is not None:
            raise ValueError("pass reference_image or reference_latents, not both")
        if self.config.depth_unified == 0:
            raise ValueError("a Kontext reference runs on FLUX-shaped configs only")
        if reference_image is not None:
            arr = self._load_image_u8(reference_image)
            return arr, (arr.shape[0] // 8, arr.shape[1] // 8)
        r = reference_latents
        if not torch.is_tensor(r) or r.dtype != torch.float32 or r.dim() != 4 or r.shape[3] != 16:
            raise ValueError("reference_latents must be an fp32 (1 or B, Hr, Wr, 16) latent in the process_in space, got "
                             f"{tuple(r.shape) if torch.is_tensor(r) else type(r).__name__}"
                             f"{' ' + str(r.dtype) if torch.is_tensor(r) else ''}")
        Br, Hr, Wr = (int(v) for v in r.shape[:3])
        if Br not in (1, n_images):
            raise ValueError(f"reference_latents has batch {Br}: pass one reference, or one per seed ({n_images})")
        if Hr % 2 or Wr % 2 or Hr == 0 or Wr == 0:
            raise ValueError(f"reference latent height and width must be positive and even, got {Hr}x{Wr}")
        return r, (Hr, Wr)

    def _reference_latent(self, ref, rows: int) -> torch.Tensor:
        """a checked Kontext reference -> the (rows, Hr, Wr, 16) activation-dtype latent every forward row takes.
        An image is encoded once and represented by its posterior mean (zero noise), as diffusers' Kontext pipeline
        does; BFL's reference code samples the posterior instead (DESIGN.md §14)."""
        if isinstance(ref, np.ndarray):
            hidden = self._encode_u8(ref)
            zero = torch.zeros(tuple(hidden.shape[:3]) + (hidden.shape[3] // 2,), dtype=torch.float32,
                               device=self.device)
            lf = self.latent_format
            ref = ops.vae_sample_latent(hidden, zero, lf.shift_factor, lf.scale_factor)
        ref16 = ops.cast_to_16(ref.to(self.device).contiguous(), self.activation_dtype)
        return ref16.repeat(rows // ref16.shape[0], 1, 1, 1)     # rows [positive x B | negative x B]

    def _redux_input(self, redux_image, cfg_weight: float, n_images: int):
        """FluxPipeline's `redux_image` -> None, or the list of 1 or n_images uint8 (S, S, 3) host arrays to encode.
        Raises, before any GPU work, for an image prompt the pipeline cannot take."""
        if redux_image is None:
            return None
        if cfg_weight > 0:
            raise ValueError("redux_image needs cfg_weight == 0: every row of a batch shares one text length and there is "
                             "no attention mask, so a negative row without image tokens cannot run beside it")
        self._need_redux()
        if not isinstance(redux_image, (list, tuple)):
            redux_image = [redux_image]
        elif len(redux_image) != n_images:
            raise ValueError(f"redux_image has {len(redux_image)} images for {n_images} seed(s): pass one image, or a "
                             "list with one per seed")
        return [self._redux_image_u8(im) for im in redux_image]

    def _need_redux(self):
        missing = [n for n in ("siglip", "redux") if getattr(self, n, None) is None]
        if missing:
            raise DkError(
                f"redux_image needs {', '.join(missing)}: call load_redux(...) with local weights first (nothing can be "
                "downloaded here), or pass `conditioning` with the image tokens appended")

    def _redux_image_u8(self, image) -> np.ndarray:
        """a path, PIL image or uint8 (H, W), (H, W, 3) or (H, W, 4) array -> uint8 (S, S, 3), S = the SigLIP image
        size: converted to RGB as BFL does, resized with PIL bicubic to exactly S x S (aspect ratio not kept,
        reducing_gap=None), as the SigLIP image processor BFL calls resizes"""
        from PIL import Image

        if isinstance(image, (str, bytes)) or hasattr(image, "__fspath__"):
            image = Image.open(image)
        if isinstance(image, np.ndarray):
            if image.dtype != np.uint8 or not (image.ndim == 2 or (image.ndim == 3 and image.shape[2] in (3, 4))):
                raise ValueError(f"redux_image array must be uint8 (H, W), (H, W, 3) or (H, W, 4), got {image.dtype} "
                                 f"{image.shape}")
            image = Image.fromarray(image)
        S = self.siglip.config.image_size
        image = image.convert("RGB").resize((S, S), Image.BICUBIC, reducing_gap=None)
        return np.ascontiguousarray(np.asarray(image))

    def _redux_tokens(self, arrs, out: torch.Tensor, T: int):
        """SigLIP + Redux of the n checked host images, one batch: image i's tokens go to rows [T, T + tokens) of
        sequence i of out (>= n, T + tokens, txt_dim)"""
        host = torch.from_numpy(np.stack(arrs)).pin_memory()
        h = self.siglip(host.to(self.device, non_blocking=True))
        P = h.shape[1]
        self.redux(h.reshape(-1, h.shape[2]), P, out=out.view(-1, out.shape[2]), out_seq_rows=T + P, out_row_off=T)

    def _redux_conditioning(self, conditioning: torch.Tensor, arrs) -> torch.Tensor:
        """(B, T, E) conditioning + checked images -> (B, T + tokens, E): each sequence's T5 rows, then its image's
        tokens (BFL's txt = cat(txt, img_cond)); one shared image is encoded once and its tokens copied"""
        B, T, E = conditioning.shape
        P = self.siglip.config.num_patches
        out = torch.empty((B, T + P, E), dtype=self.activation_dtype, device=self.device)
        ops.copy_rows(conditioning.contiguous(), out, B, T, E, T + P, 0, T, 0)
        self._redux_tokens(arrs, out, T)
        if len(arrs) < B:
            ops.copy_rows(out, out, B - 1, P, E, T + P, T + P + T, 0, T)
        return out

    def _denoise_latents(self, conditioning, pooled_conditioning, num_steps, cfg_weight, latent_size, seed, image_path,
                         denoise, *, noise, solver, guidance, slg=None, reference_image=None, reference_latents=None,
                         redux_image=None, redux_log=None, eta=None, sde_log=None, mask_image=None, fill_log=None,
                         control_image=None, canny_thresholds=control.DEFAULT_THRESHOLDS, control_log=None,
                         estimate_depth=False):
        _check_solver(solver, eta)
        _check_slg(slg, cfg_weight, self.config)
        self._check_fill(image_path, mask_image, reference_image, reference_latents)
        thresholds = self._check_control(control_image, canny_thresholds, reference_image, reference_latents,
                                         estimate_depth)
        if image_path is None:
            denoise = 1.0                                                   # :270-271
        elif not (0.0 <= denoise <= 1.0):
            raise ValueError(f"denoise must be in [0, 1], got {denoise}")
        source = None
        if mask_image is not None:
            # generate_image passes the source array and the mask it prepared; the source is read once either way
            source, mask_image = self._inpaint_input(image_path, mask_image)
        if control_image is not None:
            # the control image takes the target's pixel size: the source's when there is one (read once here)
            if image_path is not None and source is None:
                image_path = self._load_image_u8(image_path)
            target = source if source is not None else image_path
            size = ((target.shape[1], target.shape[0]) if target is not None
                    else (8 * latent_size[1], 8 * latent_size[0]))
            control_image = control.load_control_image(control_image, size)
        seeds: List[int]
        if seed is None:
            seeds = [int(time.time())]
        elif isinstance(seed, (list, tuple)):
            seeds = [int(s) for s in seed]
        else:
            seeds = [int(seed)]
        B = len(seeds)
        guidance = self._guidance_values(guidance, B)
        reference = self._reference_input(reference_image, reference_latents, B)
        redux = self._redux_input(redux_image, cfg_weight, B)
        H, W = latent_size
        conditioning = torch.as_tensor(conditioning).to(device=self.device, dtype=self.activation_dtype)
        pooled_conditioning = torch.as_tensor(pooled_conditioning).to(device=self.device, dtype=self.activation_dtype)
        if conditioning.dim() == 4:
            conditioning = conditioning.squeeze(2)
        reps = 2 if cfg_weight > 0 else 1
        if B > 1 and conditioning.shape[0] == reps and pooled_conditioning.shape[0] == reps:
            # one prompt (what encode_text returns: [positive] or [positive | negative]), several seeds: every image of
            # the batch shares it -> [positive x B | negative x B], the layout CFGDenoiser splits (:718)
            conditioning = conditioning.repeat_interleave(B, dim=0)
            pooled_conditioning = pooled_conditioning.repeat_interleave(B, dim=0)
        if conditioning.shape[0] != reps * B:
            raise DkError(
                f"conditioning has batch {conditioning.shape[0]}, expected {reps * B} "
                f"({'[positive | negative] x ' if reps == 2 else ''}{B} image(s)) for cfg_weight={cfg_weight}")
        if redux is not None:
            t0 = time.time()
            conditioning = self._redux_conditioning(conditioning, redux)
            if redux_log is not None:
                torch.cuda.synchronize(self.device)
                redux_log.update(images=len(redux), tokens=self.siglip.config.num_patches,
                                 time=round(time.time() - t0, 3))

        hidden = None
        if source is not None:
            hidden = self._encode_u8(source)
            H, W = hidden.shape[1], hidden.shape[2]
        elif image_path is not None:
            hidden = self._encode_image_hidden(image_path)                  # (1, H, W, 32) = (mean | logvar)
            H, W = hidden.shape[1], hidden.shape[2]
        x_T = self.get_empty_latent(H, W)                                   # (1, H, W, 16) host
        if noise is None:
            noise = self._get_noise_batch(seeds, x_T)                              # (B, H, W, 16) host fp32
        elif tuple(noise.shape) != (B, H, W, 16):
            raise DkError(f"noise has shape {tuple(noise.shape)}, expected {(B, H, W, 16)}")
        sigmas = self.get_sigmas(self.sampler, num_steps)
        sigmas = sigmas[int(num_steps * (1 - denoise)):]
        s0 = float(sigmas[0])
        if hidden is None:
            x = noise.to(self.device, dtype=torch.float32, non_blocking=True).clone()
            # noise_scaling: sigma0 * noise + (1 - sigma0) * x_T (sampler.py:41-42); x_T is the constant 0.0609
            x = ops.axpb(x.contiguous(), s0, (1.0 - s0) * 0.0609)
        else:
            # x_T = process_in(mean + std * noise), with the SAME seeded draw the diffusion noise uses (:273-275,
            # :586-594: both get_noise(seed, .) calls see the same shape); then sigma0 * noise + (1 - sigma0) * x_T
            noise = noise.to(self.device, dtype=torch.float32, non_blocking=True).contiguous()
            lf = self.latent_format
            x_T = torch.empty_like(noise)
            for b in range(B):
                ops.vae_sample_latent(hidden, noise[b:b + 1], lf.shift_factor, lf.scale_factor, out=x_T[b:b + 1])
            x = ops.axpby(noise, x_T, s0, 1.0 - s0)
        extra_args = {"conditioning": conditioning, "cfg_weight": cfg_weight,
                      "pooled_conditioning": pooled_conditioning}
        if guidance is not None:
            # rows [positive x B | negative x B]: both rows of an image get its value
            extra_args["guidance"] = guidance * reps
        if slg is not None:
            extra_args["slg"] = slg
        if reference is not None:
            extra_args["reference"] = self._reference_latent(reference[0], reps * B)
        if control_image is not None:
            # FLUX.1 Canny / Depth: the control image's latent conditions the x-embedder, once per call
            t0 = time.time()
            if not hasattr(self, "encoder"):
                self.load_encoder()
            lf = self.latent_format
            if estimate_depth:
                # FLUX.1 Depth from a photo: BFL's DepthImageEncoder, then the estimated map is the control image
                t1 = time.time()
                image = self._depth_image(control_image, rgb=True)
                if control_log is not None:
                    torch.cuda.synchronize(self.device)
                    depth_log = {"input_size": depth.network_size(*control_image.shape[:2]),
                                 "time": round(time.time() - t1, 3)}
            else:
                image = torch.from_numpy(control_image).to(self.device)
            rows = control.control_rows(self.encoder, image, self.config.control, lf.shift_factor, lf.scale_factor,
                                        self.activation_dtype, thresholds)
            self.mmdit.cache_fill_conditioning(rows)
            if control_log is not None:
                torch.cuda.synchronize(self.device)
                control_log.update(kind=self.config.control, latent_size=(H, W), time=round(time.time() - t0, 3))
                if estimate_depth:
                    control_log["depth"] = depth_log
        if source is not None and self.config.x_embedder_cond_channels and not self.config.control:
            # FLUX.1 Fill: the masked source and the mask condition the x-embedder, once per call; no latent blend
            t0 = time.time()
            lf = self.latent_format
            src = torch.from_numpy(source).unsqueeze(0).to(self.device)
            rows = fill.conditioning_rows(self.encoder, src, torch.from_numpy(mask_image.pixels).to(self.device),
                                          lf.shift_factor, lf.scale_factor, self.activation_dtype)
            self.mmdit.cache_fill_conditioning(rows)
            if fill_log is not None:
                torch.cuda.synchronize(self.device)
                fill_log.update(latent_size=tuple(mask_image.latent.shape), masked_fraction=mask_image.masked_fraction,
                                time=round(time.time() - t0, 3))
        elif source is not None:
            # eps = the seeded noise and x0 = the encoded source of the start above, both (B, H, W, 16) in process_in
            lm = torch.from_numpy(mask_image.latent).to(self.device)
            extra_args["inpaint"] = inpaint.InpaintBlend(noise, x_T, lm)
        if solver in SDE_SOLVERS:
            extra_args.update(eta=eta, seeds=seeds)
            if sde_log is not None:
                sde_log.update(solver=solver, eta=1.0 if eta is None else float(eta), seeds=seeds)
            latent, iter_time = SDE_SOLVERS[solver](CFGDenoiser(self), x, sigmas, extra_args=extra_args)
        else:
            latent, iter_time = SOLVERS[solver](CFGDenoiser(self), x, sigmas, extra_args=extra_args)
        latent = ops.axpb(latent, 1.0 / self.latent_format.scale_factor, self.latent_format.shift_factor)  # process_out
        return latent, iter_time

    # ------------------------------------------------------------------ generate (:294-534)
    def generate_image(
        self,
        text: str,
        num_steps: int = 2,
        cfg_weight: float = 0.0,
        negative_text: str = "",
        latent_size: Tuple[int, int] = (64, 64),
        seed=None,
        verbose: bool = True,
        image_path: Optional[str] = None,
        denoise: float = 1.0,
        *,
        conditioning=None,
        pooled_conditioning=None,
        solver: str = "euler",
        slg: Optional[SkipLayerGuidance] = None,
        eta: Optional[float] = None,
        mask_image=None,
    ):
        """`slg`: skip-layer guidance as in denoise_latents; the log then holds its scale, layers and the steps it
        applied to under log["denoising"]["skip_layer_guidance"].  `solver` and `eta` as in denoise_latents; under a
        stochastic solver the log holds {"solver", "eta", "seeds"} under log["denoising"]["sde"] (the seeds also when
        seed=None picked one from the clock), which reproduces the run.  `mask_image` as in denoise_latents; every
        unmasked pixel of the returned images is then the source pixel (the resized image that was encoded), bit for
        bit, and the log holds {"latent_size", "masked_fraction"} under log["denoising"]["inpaint"]."""
        return self._generate_image(text, num_steps, cfg_weight, negative_text, latent_size, seed, verbose, image_path,
                                    denoise, conditioning=conditioning, pooled_conditioning=pooled_conditioning,
                                    solver=solver, guidance=None, slg=slg, eta=eta, mask_image=mask_image)

    def _generate_image(self, text, num_steps, cfg_weight, negative_text, latent_size, seed, verbose, image_path,
                        denoise, *, conditioning, pooled_conditioning, solver, guidance, slg=None, reference_image=None,
                        reference_latents=None, redux_image=None, eta=None, mask_image=None, control_image=None,
                        canny_thresholds=control.DEFAULT_THRESHOLDS, estimate_depth=False):
        _check_solver(solver, eta)
        _check_slg(slg, cfg_weight, self.config)
        self._check_fill(image_path, mask_image, reference_image, reference_latents)
        self._check_control(control_image, canny_thresholds, reference_image, reference_latents, estimate_depth)
        n_images = len(seed) if isinstance(seed, (list, tuple)) else 1
        guidance = self._guidance_values(guidance, n_images)
        reference = self._reference_input(reference_image, reference_latents, n_images)
        redux = self._redux_input(redux_image, cfg_weight, n_images)   # the checked 384^2 arrays go on: read once
        source = None
        if mask_image is not None:                  # the source array goes on to the encoder and the paste-back
            source, mask_image = self._inpaint_input(image_path, mask_image)
            image_path = source
        if reference is not None:                   # the checked image array goes on, so the file is read once
            ref_kw = {"reference_image" if isinstance(reference[0], np.ndarray) else "reference_latents": reference[0]}
        else:
            ref_kw = {}
        assert latent_size[0] % 2 == 0, f"Height must be divisible by 16 ({latent_size[0]*8}/16={latent_size[0]/2})"
        assert latent_size[1] % 2 == 0, f"Width must be divisible by 16 ({latent_size[1]*8}/16={latent_size[1]/2})"
        self.check_and_load_models()
        start_time = time.time()

        def mem():
            return {"peak_memory": round(_bytes2gigabytes(torch.cuda.max_memory_allocated(self.device)), 3),
                    "active_memory": round(_bytes2gigabytes(torch.cuda.memory_allocated(self.device)), 3)}

        log = {
            "text_encoding": {"pre": mem(), "post": {"peak_memory": None, "active_memory": None}},
            "denoising": {"pre": {"peak_memory": None, "active_memory": None},
                          "post": {"peak_memory": None, "active_memory": None}},
            "decoding": {"pre": {"peak_memory": None, "active_memory": None},
                         "post": {"peak_memory": None, "active_memory": None}},
            "peak_memory": 0.0,
        }
        t0 = time.time()
        if conditioning is None or pooled_conditioning is None:
            conditioning, pooled_conditioning = self.encode_text(text, cfg_weight, negative_text)
        log["text_encoding"]["post"] = mem()
        log["text_encoding"]["time"] = round(time.time() - t0, 3)
        log["peak_memory"] = max(log["peak_memory"], log["text_encoding"]["post"]["peak_memory"])

        torch.cuda.reset_peak_memory_stats(self.device)
        t0 = time.time()
        log["denoising"]["pre"] = mem()
        redux_log, sde_log, fill_log, control_log = {}, {}, {}, {}
        latents, iter_time = self._denoise_latents(conditioning, pooled_conditioning, num_steps, cfg_weight,
                                                   latent_size, seed, image_path, denoise, noise=None, solver=solver,
                                                   guidance=guidance, slg=slg, redux_log=redux_log, eta=eta,
                                                   sde_log=sde_log, mask_image=mask_image, fill_log=fill_log,
                                                   control_image=control_image, canny_thresholds=canny_thresholds,
                                                   control_log=control_log, estimate_depth=estimate_depth,
                                                   redux_image=redux if redux is None or len(redux) == n_images
                                                   else redux[0], **ref_kw)
        torch.cuda.synchronize(self.device)
        log["denoising"]["post"] = mem()
        log["denoising"]["time"] = round(time.time() - t0, 3)
        log["denoising"]["iter_time"] = iter_time
        if solver != "euler":
            # every schedule ends at sigma = 0, and only there: a Heun step costs two forwards except the last
            n = len(iter_time)
            log["denoising"]["solver"] = solver
            log["denoising"]["nfe"] = max(2 * n - 1, 0) if solver == "heun" else n
        if sde_log:
            log["denoising"]["sde"] = sde_log
        if guidance is not None:
            log["denoising"]["guidance"] = guidance
        if reference is not None:
            Hr, Wr = reference[1]
            log["denoising"]["reference"] = {"latent_size": (Hr, Wr), "tokens": (Hr // 2) * (Wr // 2)}
        if redux is not None:
            log["denoising"]["redux"] = redux_log
        if control_log:
            log["denoising"]["control"] = control_log
        if fill_log:
            log["denoising"]["fill"] = fill_log
        elif source is not None:
            log["denoising"]["inpaint"] = {"latent_size": tuple(mask_image.latent.shape),
                                           "masked_fraction": mask_image.masked_fraction}
        if slg is not None:
            log["denoising"]["skip_layer_guidance"] = {
                "scale": slg.scale, "layers": list(slg.layers),
                "steps": skip_layer_guidance_steps(slg, len(iter_time))}
        if self.mmdit.step_cache is not None:
            log["denoising"]["step_cache"] = [{"rel": rel, "skipped": skipped}
                                              for rel, skipped in self.mmdit.step_cache_log]
        log["peak_memory"] = max(log["peak_memory"], log["denoising"]["post"]["peak_memory"])

        torch.cuda.reset_peak_memory_stats(self.device)
        t0 = time.time()
        log["decoding"]["pre"] = mem()
        latents16 = ops.cast_to_16(latents, self.activation_dtype)          # latents.astype(activation_dtype) (:459)
        _, u8 = self._decode(latents16, want_u8=True)
        if source is not None:                      # unmasked pixels: the source, without the VAE round trip
            inpaint.inpaint_paste(u8, torch.from_numpy(np.ascontiguousarray(source[:, :, :3])).to(self.device),
                                  torch.from_numpy(mask_image.pixels).to(self.device))
        host = getattr(self, "_host_u8", None)                              # pinned staging, reused across calls
        if host is None or host.shape != u8.shape:
            host = self._host_u8 = torch.empty(u8.shape, dtype=torch.uint8, pin_memory=True)
        host.copy_(u8, non_blocking=True)                                   # device -> host: the result
        torch.cuda.current_stream().synchronize()
        images_u8 = host.numpy()         # Image.fromarray copies RGB data, so reusing the staging buffer is safe
        log["decoding"]["post"] = mem()
        log["decoding"]["time"] = round(time.time() - t0, 3)
        log["peak_memory"] = max(log["peak_memory"], log["decoding"]["post"]["peak_memory"])
        log["total_time"] = round(time.time() - start_time, 3)

        from PIL import Image

        images = [Image.fromarray(images_u8[i]) for i in range(images_u8.shape[0])]
        # batch 1 returns a single image like the reference; a list of seeds returns a list (quirk Q9)
        return (images[0] if not isinstance(seed, (list, tuple)) else images), log

    # ------------------------------------------------------------------ helpers (:553-584)
    def get_noise(self, seed, x_T):
        # np.random.seed(seed); np.random.randn(...) of the reference (:553-557).  RandomState(seed) is the same
        # MT19937 stream as the seeded global generator, without the global state (thread-safe for batches).
        shape = tuple(x_T.shape)
        noise = np.random.RandomState(seed).randn(shape[0], shape[3], shape[1], shape[2])
        # float64 -> float32 and NCHW -> NHWC in numpy: the same values as mx.array(noise).transpose(0, 2, 3, 1), and
        # ~100x cheaper on a many-core host than a strided multi-threaded torch CPU copy
        return torch.from_numpy(np.ascontiguousarray(noise.astype(np.float32).transpose(0, 2, 3, 1)))

    def _get_noise_batch(self, seeds, x_T):
        if len(seeds) == 1:
            return self.get_noise(seeds[0], x_T)
        from concurrent.futures import ThreadPoolExecutor

        with ThreadPoolExecutor(max_workers=min(len(seeds), 8)) as ex:   # numpy releases the GIL while drawing
            parts = list(ex.map(lambda sd: self.get_noise(sd, x_T), seeds))
        return torch.cat(parts, dim=0)

    def get_sigmas(self, sampler, num_steps: int):
        start = float(sampler.timestep(sampler.sigma_max))
        end = float(sampler.timestep(sampler.sigma_min))
        if isinstance(sampler, FluxSampler):
            num_steps += 1
        timesteps = np.linspace(start, end, num_steps, dtype=np.float32)
        sigs = [float(sampler.sigma(ts)) for ts in timesteps]
        if not isinstance(sampler, FluxSampler):
            sigs += [0.0]
        return np.asarray(sigs, dtype=np.float32)

    def _load_image_u8(self, image) -> np.ndarray:
        """-> uint8 (H, W, >=3) with H, W multiples of 64 (read_image's resize rule, :540-546)"""
        return _load_image_sized(image)[0]

    def _inpaint_input(self, image_path, mask_image):
        """-> (the source as _load_image_u8 returns it, inpaint.InpaintMask); a prepared mask passes through with
        image_path, which is then that source array.  Raises ValueError, before any GPU work, for a mask the pipeline
        cannot take."""
        if image_path is None:
            raise ValueError("mask_image needs image_path: the mask marks what to regenerate in that source image")
        if isinstance(mask_image, inpaint.InpaintMask):
            return image_path, mask_image
        source, size = _load_image_sized(image_path)
        return source, inpaint.prepare_mask(mask_image, size)

    def read_image(self, image_path):
        """-> (1, H, W, 3) float32 in [-1, 1] on the host (reference :536-551)"""
        arr = self._load_image_u8(image_path)
        return (torch.from_numpy(arr[:, :, :3].astype(np.float32)) / 255 * 2 - 1.0).unsqueeze(0)

    def _encode_image_hidden(self, image_path) -> torch.Tensor:
        return self._encode_u8(self._load_image_u8(image_path))

    def _encode_u8(self, arr: np.ndarray) -> torch.Tensor:
        """a _load_image_u8 array -> the VAE encoder's (1, H/8, W/8, 32) (mean | logvar)"""
        if not hasattr(self, "encoder"):
            self.load_encoder()
        host = torch.from_numpy(arr).unsqueeze(0).pin_memory()
        return self.encoder(host.to(self.device, non_blocking=True))       # the /255*2-1 runs in dk_image_pre

    def encode_image_to_latents(self, image_path, seed):
        """mean + exp(0.5 * clip(logvar, -30, 20)) * get_noise(seed)  (reference :586-594) -> (1, H/8, W/8, 16) fp32"""
        hidden = self._encode_image_hidden(image_path)
        mean_like = torch.empty((1, hidden.shape[1], hidden.shape[2], hidden.shape[3] // 2))
        noise = self.get_noise(seed, mean_like).to(self.device)
        return ops.vae_sample_latent(hidden, noise.contiguous(), 0.0, 1.0)

    def get_empty_latent(self, *shape):
        return torch.ones([1, *shape, 16], dtype=torch.float32) * 0.0609

    def max_denoise(self, sigmas):
        max_sigma = float(self.sampler.sigma_max)
        sigma = float(sigmas[0])
        return math.isclose(max_sigma, sigma, rel_tol=1e-05) or sigma > max_sigma

    def _decode(self, x_t, want_u8: bool):
        x = self.decoder(x_t)                                               # (B, 8H, 8W, 3) view of a padded buffer
        B, Ho, Wo, _ = x.shape
        padded = x.as_strided((B, Ho, Wo, x.stride(2)), (x.stride(0), x.stride(1), x.stride(2), 1))
        return ops.image_post(padded, want_u8=want_u8)

    def decode_latents_to_image(self, x_t):
        """x = decoder(x_t); clip(x / 2 + 0.5, 0, 1)  (:581-584) -> (B, 8H, 8W, 3) float in [0, 1]"""
        x_t = torch.as_tensor(x_t).to(device=self.device)
        if x_t.dtype == torch.float32:
            x_t = ops.cast_to_16(x_t.contiguous(), self.activation_dtype)
        f, _ = self._decode(x_t, want_u8=False)
        return f


class FluxPipeline(DiffusionPipeline):
    _default_model = "argmaxinc/mlx-FLUX.1-schnell"

    def __init__(
        self,
        w16: bool = False,
        shift: float = 1.0,
        use_t5: bool = True,
        model_version: str = "argmaxinc/mlx-FLUX.1-schnell",
        low_memory_mode: bool = True,
        a16: bool = False,
        local_ckpt=None,
        quantize_mmdit: bool = False,
        *,
        device=None,
        params=None,
        vae_params=None,
        mmdit_config=None,
        weight_seed: int = 0,
        load_decoder: bool = True,
        vae_encoder_params=None,
        load_encoder: bool = False,
    ):
        self.float16_dtype = torch.bfloat16                                 # :610
        self._vae_encoder_params, self._load_encoder = vae_encoder_params, load_encoder
        self._setup(w16, a16, shift, model_version, low_memory_mode, local_ckpt, device, params, vae_params,
                    mmdit_config, weight_seed, load_decoder)
        self.sampler = FluxSampler(shift=shift)
        self.latent_format = FluxLatentFormat()
        self.use_t5 = True
        self.use_clip_g = False
        self.quantize_mmdit = quantize_mmdit

    def denoise_latents(self, conditioning, pooled_conditioning, num_steps: int = 2, cfg_weight: float = 0.0,
                        latent_size: Tuple[int, int] = (64, 64), seed=None, image_path: Optional[str] = None,
                        denoise: float = 1.0, *, noise: Optional[torch.Tensor] = None, solver: str = "euler",
                        guidance=None, reference_image=None, reference_latents: Optional[torch.Tensor] = None,
                        redux_image=None, eta: Optional[float] = None, mask_image=None, control_image=None,
                        canny_thresholds=control.DEFAULT_THRESHOLDS, estimate_depth: bool = False):
        """DiffusionPipeline.denoise_latents (`solver`, `eta` and `mask_image` included), plus FLUX.1-dev's distilled guidance (DESIGN.md §12): `guidance` is one
        float for every image or one per seed, and None means DEFAULT_GUIDANCE (3.5) when the model has a guidance
        embedder (mmdit_config=FLUX_DEV).  A model without one refuses any value but None.

        FLUX.1 Kontext editing (DESIGN.md §14): `reference_image` (a path, a PIL image or a uint8 HWC RGB array, sides
        cut to multiples of 64 like image_path) is encoded once by the VAE encoder into its posterior mean;
        `reference_latents` is a device fp32 (1 or B, Hr, Wr, 16) latent already in the process_in space (B: one
        reference per seed).  Every forward then sees the reference tokens after the target's; the result covers the
        target alone.  Pass at most one of the two.  `image_path` still sets the target's starting point.

        FLUX.1 Redux image prompt (DESIGN.md §15, after load_redux): `redux_image` is one image for every seed or a list
        with one per seed (each as encode_redux takes it).  It is encoded once per call, and its tokens are appended to
        each image's conditioning rows, which then hold T + tokens rows.  Needs cfg_weight == 0.

        FLUX.1 Fill [dev] (DESIGN.md §18; model_version "black-forest-labs/FLUX.1-Fill-dev" or mmdit_config=
        FLUX_FILL_DEV): `image_path` and `mask_image` are required, `mask_image` as in DiffusionPipeline.  The source with
        its masked pixels zeroed is encoded once into its posterior mean and, with the mask, conditions every forward
        through the x-embedder; there is no latent blend.  `guidance` None means 30.0 on this model.  No Kontext
        reference.

        FLUX.1 Canny / Depth [dev] (DESIGN.md §19; model_version "black-forest-labs/FLUX.1-Canny-dev" / "-Depth-dev",
        or mmdit_config=FLUX_CANNY_DEV / FLUX_DEPTH_DEV): `control_image` is required, a path, a PIL image or a uint8
        (H, W) / (H, W, 1|3|4) array, converted to RGB and resized with PIL LANCZOS to exactly the target's pixel size
        (the source's with image_path, else 8 x latent_size).  On Canny it goes through BFL's round trip and
        cv2.Canny(img, *canny_thresholds) on the GPU first (canny_thresholds None: it is already an edge map); on
        Depth it is the depth map.  It is encoded once into its posterior mean and conditions every forward through
        the x-embedder.  `guidance` None means 30.0 on Canny and 10.0 on Depth.  img2img, mask_image (§17's blend),
        Redux and every solver combine with it; a Kontext reference does not.  Other models refuse control_image.

        `estimate_depth=True` (FLUX.1 Depth only, after load_depth_estimator; DESIGN.md §20): `control_image` is a photo,
        and the depth map is estimated from it once per call as BFL's DepthImageEncoder does (estimate_depth)
        before it is encoded."""
        return self._denoise_latents(conditioning, pooled_conditioning, num_steps, cfg_weight, latent_size, seed,
                                     image_path, denoise, noise=noise, solver=solver, guidance=guidance,
                                     reference_image=reference_image, reference_latents=reference_latents,
                                     redux_image=redux_image, eta=eta, mask_image=mask_image,
                                     control_image=control_image, canny_thresholds=canny_thresholds,
                                     estimate_depth=estimate_depth)

    def generate_image(self, text: str, num_steps: int = 2, cfg_weight: float = 0.0, negative_text: str = "",
                       latent_size: Tuple[int, int] = (64, 64), seed=None, verbose: bool = True,
                       image_path: Optional[str] = None, denoise: float = 1.0, *, conditioning=None,
                       pooled_conditioning=None, solver: str = "euler", guidance=None, reference_image=None,
                       reference_latents: Optional[torch.Tensor] = None, redux_image=None, eta: Optional[float] = None,
                       mask_image=None, control_image=None, canny_thresholds=control.DEFAULT_THRESHOLDS,
                       estimate_depth: bool = False):
        """DiffusionPipeline.generate_image (`solver`, `eta`, `mask_image` and their logs included) with `guidance`, `reference_image`, `reference_latents` and `redux_image`
        as in denoise_latents; with a guidance embedder the log holds the value of each image under
        log["denoising"]["guidance"], with a reference its latent size and token count under
        log["denoising"]["reference"], and with an image prompt {"images", "tokens", "time"} of its encode under
        log["denoising"]["redux"].  On a FLUX.1 Fill model the unmasked source pixels are pasted back as with any mask,
        and the log holds {"latent_size", "masked_fraction", "time"} of the conditioning under log["denoising"]["fill"]
        instead of log["denoising"]["inpaint"].  `control_image` and `canny_thresholds` as in denoise_latents; on a
        Canny or Depth model the log holds {"kind", "latent_size", "time"} of the conditioning under
        log["denoising"]["control"], and with `estimate_depth` also "depth": {"input_size", "time"} of the estimator."""
        return self._generate_image(text, num_steps, cfg_weight, negative_text, latent_size, seed, verbose, image_path,
                                    denoise, conditioning=conditioning, pooled_conditioning=pooled_conditioning,
                                    solver=solver, guidance=guidance, reference_image=reference_image,
                                    reference_latents=reference_latents, redux_image=redux_image, eta=eta,
                                    mask_image=mask_image, control_image=control_image,
                                    canny_thresholds=canny_thresholds, estimate_depth=estimate_depth)

    def load_depth_estimator(self, params=None, *, config=None):
        """Build FLUX.1 Depth's depth estimator on the device: Depth Anything (config, default
        LiheYoung/depth-anything-large-hf).  params: the engine's tree (model_io.depth_anything_checkpoint_to_params
        converts the upstream safetensors), or None for the deterministic synthetic initialiser.  It runs in the
        pipeline's 16-bit dtype; BFL runs it in fp32 (DESIGN.md §20)."""
        from .config import DEPTH_ANYTHING_LARGE

        cfg = config or DEPTH_ANYTHING_LARGE
        if params is None:
            params = depth.init_depth_params(cfg, seed=self._weight_seed + 8)
        self.depth_estimator = depth.DepthAnythingModel(params, cfg, dtype=self.dtype, device=self.device)

    def _need_depth_estimator(self):
        if getattr(self, "depth_estimator", None) is None:
            raise DkError("estimate_depth needs the depth estimator: call load_depth_estimator(...) with local weights "
                          "first (nothing can be downloaded here), or pass the depth map itself as control_image")

    def _depth_image(self, image_u8: np.ndarray, rgb: bool) -> torch.Tensor:
        """BFL's DepthImageEncoder of a uint8 (H, W, 3) host image at the target size: the round trip and the
        processor's resize on the host, the estimator, the antialiased bicubic back to (H, W) -> fp32 depth (H, W), or
        with rgb the VAE's (H, W, 3) input depth / 127.5 - 1 in the pipeline dtype"""
        net = torch.from_numpy(depth.network_input(image_u8)).to(self.device)
        est = self.depth_estimator
        return est.depth(est(net), image_u8.shape[:2], rgb=rgb)

    def estimate_depth(self, image) -> torch.Tensor:
        """BFL's `depth` of one image (a path, a PIL image or a uint8 (H, W) / (H, W, 1|3|4) array, converted to RGB):
        fp32 (H, W) on the device, before depth / 127.5 - 1, at the image's own size (after load_depth_estimator)"""
        self._need_depth_estimator()
        arr = control.load_control_image(image, None)
        return self._depth_image(arr, rgb=False)

    def load_redux(self, siglip=None, redux=None, *, siglip_config=None):
        """Build FLUX.1 Redux's image encoder on the device: SigLIP (siglip_config, default
        google/siglip-so400m-patch14-384) and the Redux projector.  siglip / redux: parameter dicts in the engine's names
        (model_io.siglip_checkpoint_to_params / redux_checkpoint_to_params convert the upstream safetensors), or None for
        the deterministic synthetic initialiser.  Weights are 16-bit in the pipeline's dtype."""
        from .config import SIGLIP_SO400M_PATCH14_384
        from .image_encoders import (ReduxImageEncoder, SiglipVisionModel, init_siglip_params, redux_param_specs)

        cfg = siglip_config or SIGLIP_SO400M_PATCH14_384
        txt_dim = self.config.token_level_text_embed_dim
        if siglip is None:
            siglip = init_siglip_params(cfg, seed=self._weight_seed + 6, dtype=self.dtype, device=self.device)
        if redux is None:
            redux = init_params(redux_param_specs(cfg.hidden_size, txt_dim), seed=self._weight_seed + 7,
                                dtype=self.dtype, device=self.device)
        enc = ReduxImageEncoder({k: v.to(device=self.device, dtype=self.dtype) for k, v in redux.items()},
                                device=self.device)
        if (enc.siglip_hidden, enc.txt_dim) != (cfg.hidden_size, txt_dim):
            raise ValueError(f"Redux projector maps {enc.siglip_hidden} -> {enc.txt_dim}; this pipeline needs "
                             f"{cfg.hidden_size} (SigLIP) -> {txt_dim} (token_level_text_embed_dim)")
        self.siglip = SiglipVisionModel({k: v.to(device=self.device, dtype=self.dtype) for k, v in siglip.items()}, cfg,
                                        device=self.device)
        self.redux = enc

    def encode_redux(self, images) -> torch.Tensor:
        """FLUX.1 Redux tokens of one image or a list (paths, PIL images or uint8 HWC arrays; converted to RGB and
        resized to SigLIP's square size on the host), encoded as one batch -> (n, tokens, token_level_text_embed_dim)
        on the device in the activation dtype.  Appending them to the T5 rows of `conditioning` is what
        `redux_image=` does."""
        self._need_redux()
        arrs = [self._redux_image_u8(im) for im in (images if isinstance(images, (list, tuple)) else [images])]
        out = torch.empty((len(arrs), self.siglip.config.num_patches, self.redux.txt_dim), dtype=self.activation_dtype,
                          device=self.device)
        self._redux_tokens(arrs, out, 0)
        return out

    def encode_text(self, text: str, cfg_weight: float = 7.5, negative_text: str = ""):
        """reference :642-671: CLIP-L pooled output + T5 sequence of the POSITIVE prompt only, T5 padded with zeros to
        T5_MAX_LENGTH -> (conditioning (1, T5, 4096), pooled (1, 768))"""
        self._need_text_stack("clip_l", "tokenizer_l", "t5_encoder", "t5_tokenizer")
        neg = negative_text if cfg_weight > 1 else None
        tokens_l = self._tokenize(self.tokenizer_l, text, neg)
        pooled_conditioning = self.clip_l(tokens_l[[0], :]).pooled_output
        tokens_t5 = self._tokenize(self.t5_tokenizer, text, neg)
        padded = torch.zeros((1, T5_MAX_LENGTH[self.model_version]), dtype=tokens_t5.dtype)
        padded[:, : tokens_t5.shape[1]] = tokens_t5[[0], :]
        conditioning = self.t5_encoder(padded).to(self.activation_dtype)
        return conditioning, pooled_conditioning
