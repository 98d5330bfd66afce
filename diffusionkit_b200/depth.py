"""FLUX.1 Depth [dev]'s depth estimator (DESIGN.md §20): Depth Anything (transformers' DepthAnythingForDepthEstimation,
`predicted_depth`, relative depth) on the engine's kernels, and BFL's DepthImageEncoder around it.

Backbone (DINOv2 ViT-L/14): the stride-14 patch convolution is dk_image_patches + one wgmma GEMM whose rows land at
rows 1.. of the token buffer, the (interpolated) position table added as a residual broadcast over the batch; row 0 is
CLS + pos[0].  Then pre-LN layers of LayerNorm, packed QKV GEMM, dk_attention_fwd at head dim 64, o-proj GEMM with an
in-place residual, LayerNorm, fc1 with erf-GELU, fc2 with residual; the backbone LayerNorm of each stage in out_indices.

DPT neck and head, all NHWC: per stage a 1 x 1 projection GEMM of the patch tokens, then the resize (ConvTranspose
k = s as s GEMMs whose output rows interleave, identity, or dk_conv3x3_s2_p1), a bias-free 3 x 3 convolution to the
fusion width; four fusion layers (coarsest first) of pre-activated residual units (dk_depth_add_relu + dk_conv3x3 with
the residual in the epilogue), a bilinear align_corners=True dk_resample and a 1 x 1 projection GEMM; the head's
3 x 3 convolution, bilinear resample to 14 x the patch grid, 3 x 3 convolution and dk_depth_head (relu, 1 x 1 to one
channel, relu) into fp32 depth.

Parameter trees.  `depth_param_specs` describes transformers' layout (without backbone.embeddings.mask_token and the
unused neck.fusion_stage.layers.0.residual_layer1.*), which the synthetic initialiser and
model_io.depth_anything_checkpoint_to_params start from.  `pack_depth_params` turns it, in fp32, into the engine's
tree: q / k / v packed, the layer scales folded into the o-proj and fc2 rows, ImageNet's normalisation folded into the
patch weight and bias (so dk_image_patches' u8 / 255 * 2 - 1 feeds it), convolution weights (O, kh, kw, I),
ConvTranspose weights as s slabs of (s O, I), CLS + pos[0] precomputed.

The small kernels' wrappers live here rather than in ops: the launch census of the shipped models requires a reference
for every launching op there, and these run only under the estimator, whose GPU test runs a census of its own.
"""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import numpy as np
import torch

from . import ops
from ._lib import ACT_GELU_ERF, DK_F32, dtype_code, ptr
from .config import DepthAnythingConfig
from .image_encoders import _check_shapes, image_patches, patch_weight_kp

Spec = tuple
IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)
# DPTImageProcessor of LiheYoung/depth-anything-large-hf: 518 x 518 target, aspect ratio kept, multiples of 14
NET_SIZE = 518
NET_MULTIPLE = 14
# engine-tree tensors the model keeps in fp32: the position table (interpolated in fp32) and the head tail's 1 x 1
FP32_KEYS = ("pos", "head.conv3.weight", "head.conv3.bias")


def check_config(cfg: DepthAnythingConfig):
    """ValueError for a configuration the kernels cannot run"""
    if cfg.depth_estimation_type != "relative":
        raise ValueError(f"Depth Anything: only the relative-depth head is implemented, got {cfg.depth_estimation_type!r}")
    if cfg.hidden_act != "gelu":
        raise ValueError(f"Depth Anything: only the erf-GELU MLP is implemented, got {cfg.hidden_act!r}")
    if cfg.hidden_size != cfg.num_attention_heads * 64:
        raise ValueError(f"Depth Anything: the head dim must be 64 (hidden {cfg.hidden_size}, "
                         f"{cfg.num_attention_heads} heads)")
    if len(cfg.neck_hidden_sizes) != 4 or len(cfg.reassemble_factors) != 4 or len(cfg.out_indices) != 4:
        raise ValueError("Depth Anything: four stages (out_indices, neck_hidden_sizes, reassemble_factors)")
    if not all(1 <= i <= cfg.num_hidden_layers for i in cfg.out_indices):
        raise ValueError(f"Depth Anything: out_indices {cfg.out_indices} must name layers 1..{cfg.num_hidden_layers}")
    if tuple(cfg.reassemble_factors) != (4, 2, 1, 0.5):
        raise ValueError(f"Depth Anything: reassemble_factors must be (4, 2, 1, 0.5), got {cfg.reassemble_factors}")
    F = cfg.fusion_hidden_size
    for name, c in [("neck_hidden_sizes", c) for c in cfg.neck_hidden_sizes] + [("fusion_hidden_size", F),
                                                                               ("fusion_hidden_size / 2", F // 2)]:
        if c % 64:
            raise ValueError(f"Depth Anything: {name} ({c}) must be a multiple of 64 (the 3 x 3 convolution's Cin)")
    if cfg.head_hidden_size % 8:
        raise ValueError(f"Depth Anything: head_hidden_size ({cfg.head_hidden_size}) must be a multiple of 8")


def depth_param_specs(cfg: DepthAnythingConfig) -> List[Spec]:
    """transformers' DepthAnythingForDepthEstimation tree without backbone.embeddings.mask_token and
    neck.fusion_stage.layers.0.residual_layer1.* (neither is used by predicted_depth)"""
    D, Fm, p, F = cfg.hidden_size, cfg.intermediate_size, cfg.patch_size, cfg.fusion_hidden_size
    specs: List[Spec] = [("backbone.embeddings.cls_token", (1, 1, D), "e"),
                         ("backbone.embeddings.position_embeddings", (1, 1 + cfg.pos_grid ** 2, D), "e"),
                         ("backbone.embeddings.patch_embeddings.projection.weight", (D, 3, p, p), "w"),
                         ("backbone.embeddings.patch_embeddings.projection.bias", (D,), "b")]

    def lin(name, cout, cin, kernel=()):
        specs.append((name + ".weight", (cout, cin, *kernel), "w"))
        specs.append((name + ".bias", (cout,), "b"))

    def ln(name):
        specs.append((name + ".weight", (D,), "g"))
        specs.append((name + ".bias", (D,), "b"))

    for i in range(cfg.num_hidden_layers):
        l = f"backbone.encoder.layer.{i}."
        ln(l + "norm1")
        for n in ("query", "key", "value"):
            lin(l + "attention.attention." + n, D, D)
        lin(l + "attention.output.dense", D, D)
        specs.append((l + "layer_scale1.lambda1", (D,), "g"))
        ln(l + "norm2")
        lin(l + "mlp.fc1", Fm, D)
        lin(l + "mlp.fc2", D, Fm)
        specs.append((l + "layer_scale2.lambda1", (D,), "g"))
    ln("backbone.layernorm")
    for k, (c, f) in enumerate(zip(cfg.neck_hidden_sizes, cfg.reassemble_factors)):
        r = f"neck.reassemble_stage.layers.{k}."
        lin(r + "projection", c, D, (1, 1))
        if f > 1:
            specs.append((r + "resize.weight", (c, c, int(f), int(f)), "w"))
            specs.append((r + "resize.bias", (c,), "b"))
        elif f < 1:
            lin(r + "resize", c, c, (3, 3))
    for k, c in enumerate(cfg.neck_hidden_sizes):
        specs.append((f"neck.convs.{k}.weight", (F, c, 3, 3), "w"))
    for j in range(4):
        fl = f"neck.fusion_stage.layers.{j}."
        lin(fl + "projection", F, F, (1, 1))
        for u in (1, 2) if j else (2,):
            for n in (1, 2):
                lin(f"{fl}residual_layer{u}.convolution{n}", F, F, (3, 3))
    lin("head.conv1", F // 2, F, (3, 3))
    lin("head.conv2", cfg.head_hidden_size, F // 2, (3, 3))
    lin("head.conv3", 1, cfg.head_hidden_size, (1, 1))
    return specs


def fold_layer_scale(w: torch.Tensor, b: torch.Tensor, lam: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """lam * (x W^T + b) = x (lam W)^T + lam b: the layer scale folded into the rows of the linear before it"""
    return w * lam[:, None], b * lam


def fold_imagenet(w: torch.Tensor, b: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """patch convolution (O, 3, p, p) of ImageNet-normalised pixels (x / 255 - mu_c) / sigma_c -> the same convolution
    of u = x / 255 * 2 - 1: W' = W / (2 sigma_c), b' = b + sum W (0.5 - mu_c) / sigma_c"""
    mu = torch.tensor(IMAGENET_MEAN, dtype=w.dtype, device=w.device)
    sd = torch.tensor(IMAGENET_STD, dtype=w.dtype, device=w.device)
    w2 = w / (2 * sd)[None, :, None, None]
    b2 = b + (w * ((0.5 - mu) / sd)[None, :, None, None]).sum(dim=(1, 2, 3))
    return w2, b2


def conv_transpose_slabs(w: torch.Tensor, b: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """ConvTranspose2d(k = s = stride) weight (I, O, s, s), bias (O,) -> slabs (s, s O, I) and the bias repeated s
    times: slab di, row dj O + o, column i is W[i, o, di, dj], so GEMM di of the input rows gives output row s y + di"""
    s = w.shape[2]
    return w.permute(2, 3, 1, 0).reshape(s, s * w.shape[1], w.shape[0]).contiguous(), b.repeat(s)


def conv_weight(w: torch.Tensor) -> torch.Tensor:
    """OIHW -> (O, kh, kw, I)"""
    return w.permute(0, 2, 3, 1).contiguous()


def pack_depth_params(params: Dict[str, torch.Tensor], cfg: DepthAnythingConfig) -> Dict[str, torch.Tensor]:
    """transformers-layout tree (depth_param_specs) -> the engine's, computed in fp32 (module docstring)"""
    P = {k: v.float() for k, v in params.items()}
    D, p, g = cfg.hidden_size, cfg.patch_size, cfg.pos_grid
    out: Dict[str, torch.Tensor] = {}
    e = "backbone.embeddings."
    w, b = fold_imagenet(P[e + "patch_embeddings.projection.weight"], P[e + "patch_embeddings.projection.bias"])
    w = w.permute(0, 2, 3, 1).reshape(D, 3 * p * p)
    out["patch.weight"] = torch.cat([w, w.new_zeros((D, patch_weight_kp(cfg) - 3 * p * p))], 1).contiguous()
    out["patch.bias"] = b
    pos = P[e + "position_embeddings"].reshape(1 + g * g, D)
    out["cls_pos"] = (P[e + "cls_token"].reshape(1, D) + pos[:1]).contiguous()
    out["pos"] = pos[1:].reshape(g, g, D).contiguous()
    for i in range(cfg.num_hidden_layers):
        l, o = f"backbone.encoder.layer.{i}.", f"layers.{i}."
        a = l + "attention.attention."
        for n in ("norm1", "norm2"):
            out[o + n + ".weight"], out[o + n + ".bias"] = P[l + n + ".weight"], P[l + n + ".bias"]
        out[o + "qkv.weight"] = torch.cat([P[a + n + ".weight"] for n in ("query", "key", "value")]).contiguous()
        out[o + "qkv.bias"] = torch.cat([P[a + n + ".bias"] for n in ("query", "key", "value")])
        out[o + "o.weight"], out[o + "o.bias"] = fold_layer_scale(P[l + "attention.output.dense.weight"],
                                                                  P[l + "attention.output.dense.bias"],
                                                                  P[l + "layer_scale1.lambda1"])
        out[o + "fc1.weight"], out[o + "fc1.bias"] = P[l + "mlp.fc1.weight"], P[l + "mlp.fc1.bias"]
        out[o + "fc2.weight"], out[o + "fc2.bias"] = fold_layer_scale(P[l + "mlp.fc2.weight"], P[l + "mlp.fc2.bias"],
                                                                      P[l + "layer_scale2.lambda1"])
    out["norm.weight"], out["norm.bias"] = P["backbone.layernorm.weight"], P["backbone.layernorm.bias"]
    for k, f in enumerate(cfg.reassemble_factors):
        r = f"neck.reassemble_stage.layers.{k}."
        w = P[r + "projection.weight"]
        out[f"reassemble.{k}.proj.weight"] = w.reshape(w.shape[0], w.shape[1]).contiguous()
        out[f"reassemble.{k}.proj.bias"] = P[r + "projection.bias"]
        if f > 1:
            out[f"reassemble.{k}.resize.weight"], out[f"reassemble.{k}.resize.bias"] = conv_transpose_slabs(
                P[r + "resize.weight"], P[r + "resize.bias"])
        elif f < 1:
            out[f"reassemble.{k}.resize.weight"] = conv_weight(P[r + "resize.weight"])
            out[f"reassemble.{k}.resize.bias"] = P[r + "resize.bias"]
        out[f"convs.{k}.weight"] = conv_weight(P[f"neck.convs.{k}.weight"])
    for j in range(4):
        fl = f"neck.fusion_stage.layers.{j}."
        w = P[fl + "projection.weight"]
        out[f"fusion.{j}.proj.weight"] = w.reshape(w.shape[0], w.shape[1]).contiguous()
        out[f"fusion.{j}.proj.bias"] = P[fl + "projection.bias"]
        for u in (1, 2) if j else (2,):
            for n in (1, 2):
                c = f"{fl}residual_layer{u}.convolution{n}."
                out[f"fusion.{j}.rcu{u}.conv{n}.weight"] = conv_weight(P[c + "weight"])
                out[f"fusion.{j}.rcu{u}.conv{n}.bias"] = P[c + "bias"]
    for n in ("conv1", "conv2"):
        out[f"head.{n}.weight"], out[f"head.{n}.bias"] = conv_weight(P[f"head.{n}.weight"]), P[f"head.{n}.bias"]
    out["head.conv3.weight"] = P["head.conv3.weight"].reshape(-1).contiguous()
    out["head.conv3.bias"] = P["head.conv3.bias"].reshape(1)
    return out


def engine_depth_shapes(cfg: DepthAnythingConfig) -> Dict[str, tuple]:
    """names and shapes of the engine's tree (pack_depth_params of depth_param_specs)"""
    params = {n: torch.empty(s, device="meta") for n, s, _ in depth_param_specs(cfg)}
    return {k: tuple(v.shape) for k, v in pack_depth_params(params, cfg).items()}


def init_depth_params(cfg: DepthAnythingConfig, seed: int = 0, device="cpu") -> Dict[str, torch.Tensor]:
    """deterministic synthetic weights (weights.init_params of depth_param_specs, fp32, condition_depth_params) in the
    engine's layout (fp32)"""
    from .weights import init_params

    p = init_params(depth_param_specs(cfg), seed=seed, dtype=torch.float32, device=device)
    condition_depth_params(p, cfg)
    return pack_depth_params(p, cfg)


def condition_depth_params(p: Dict[str, torch.Tensor], cfg: DepthAnythingConfig):
    """in place, on a transformers-layout tree of weights.init_params scale: the head's last 1 x 1 convolution scaled
    by 30 with bias 100, so that predicted depth spreads over about 0 .. 170 (std near 25) like a real relative-depth
    map and BFL's depth / 127.5 - 1 spans a real part of [-1, 1]; unconditioned it stays within a few units of 0"""
    p["head.conv3.weight"] = 30.0 * p["head.conv3.weight"]
    p["head.conv3.bias"] = torch.full_like(p["head.conv3.bias"], 100.0)


# ------------------------------------------------------------------------------------------------ preprocessing
def network_size(height: int, width: int, size: int = NET_SIZE, multiple: int = NET_MULTIPLE) -> Tuple[int, int]:
    """DPTImageProcessor's get_resize_output_image_size(keep_aspect_ratio=True, ensure_multiple_of=14) to a size x size
    target -> (height, width): the scale closer to 1 for both sides, each side rounded to a multiple of 14"""
    sh, sw = size / height, size / width
    if abs(1 - sw) < abs(1 - sh):
        sh = sw
    else:
        sw = sh

    def constrain(v):
        return round(v / multiple) * multiple

    return constrain(sh * height), constrain(sw * width)


def network_input(image_u8: np.ndarray) -> np.ndarray:
    """BFL's DepthImageEncoder before the model: the control image's fp32 round trip ((u8 / 127.5 - 1 + 1) * 127.5,
    truncated), then the processor's PIL BICUBIC resize to network_size -> uint8 (h, w, 3)"""
    from PIL import Image

    from .control import ROUNDTRIP

    h, w = network_size(image_u8.shape[0], image_u8.shape[1])
    img = Image.fromarray(ROUNDTRIP[image_u8[..., :3]])
    return np.ascontiguousarray(np.asarray(img.resize((w, h), Image.BICUBIC)))


# ------------------------------------------------------------------------------------------------ tap tables
def _band(rows: List[Dict[int, float]], n_in: int) -> Tuple[np.ndarray, np.ndarray]:
    """per-output {input index: weight} -> (first index int32 [n_out], weights fp64 [n_out, T]) with every index
    first + t inside [0, n_in)"""
    T = min(max(max(r) - min(r) + 1 for r in rows), n_in)
    first = np.zeros(len(rows), dtype=np.int32)
    wts = np.zeros((len(rows), T), dtype=np.float64)
    for o, r in enumerate(rows):
        i0 = min(min(r), n_in - T)
        first[o] = i0
        for i, v in r.items():
            wts[o, i - i0] += v
    return first, wts


def taps_linear(n_in: int, n_out: int, align_corners: bool) -> Tuple[np.ndarray, np.ndarray]:
    """PyTorch's bilinear (one axis of interpolate(mode="bilinear", size=...))"""
    rows = []
    for o in range(n_out):
        if align_corners:
            src = o * (n_in - 1) / (n_out - 1) if n_out > 1 else 0.0
        else:
            src = max((o + 0.5) * n_in / n_out - 0.5, 0.0)
        i0 = min(int(math.floor(src)), n_in - 1)
        i1 = min(i0 + 1, n_in - 1)
        lam = src - i0
        r: Dict[int, float] = {}
        r[i0] = r.get(i0, 0.0) + 1.0 - lam
        r[i1] = r.get(i1, 0.0) + lam
        rows.append(r)
    return _band(rows, n_in)


def taps_cubic(n_in: int, n_out: int, a: float = -0.75) -> Tuple[np.ndarray, np.ndarray]:
    """PyTorch's bicubic without antialiasing, align_corners=False: Keys' kernel (a = -0.75) at the four neighbours of
    (o + 0.5) n_in / n_out - 0.5, indices clamped to the border"""
    def c1(x):
        return ((a + 2) * x - (a + 3)) * x * x + 1

    def c2(x):
        return ((a * x - 5 * a) * x + 8 * a) * x - 4 * a

    rows = []
    for o in range(n_out):
        src = (o + 0.5) * n_in / n_out - 0.5
        i = int(math.floor(src))
        t = src - i
        r: Dict[int, float] = {}
        for d, w in zip((-1, 0, 1, 2), (c2(t + 1), c1(t), c1(1 - t), c2(2 - t))):
            j = min(max(i + d, 0), n_in - 1)
            r[j] = r.get(j, 0.0) + w
        rows.append(r)
    return _band(rows, n_in)


def taps_cubic_aa(n_in: int, n_out: int, a: float = -0.5) -> Tuple[np.ndarray, np.ndarray]:
    """PyTorch's antialiased bicubic (interpolate(mode="bicubic", antialias=True)): the kernel (a = -0.5) stretched by
    the scale when downsampling, over the taps inside the input, normalised to sum 1"""
    def f(x):
        x = abs(x)
        if x < 1:
            return ((a + 2) * x - (a + 3)) * x * x + 1
        if x < 2:
            return (((x - 5) * x + 8) * x - 4) * a
        return 0.0

    scale = n_in / n_out
    support = 2.0 * scale if scale >= 1.0 else 2.0
    inv = 1.0 / scale if scale >= 1.0 else 1.0
    rows = []
    for o in range(n_out):
        center = scale * (o + 0.5)
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), n_in)
        ws = [f((j + xmin - center + 0.5) * inv) for j in range(xmax - xmin)]
        total = sum(ws)
        rows.append({xmin + j: (w / total if total != 0 else w) for j, w in enumerate(ws)})
    return _band(rows, n_in)


TAPS = {"bilinear": lambda i, o: taps_linear(i, o, False), "bilinear_ac": lambda i, o: taps_linear(i, o, True),
        "bicubic": taps_cubic, "bicubic_aa": taps_cubic_aa}


class Taps:
    """device tap tables of one axis resampling, made once per (kind, n_in, n_out) and device"""

    _cache: Dict[tuple, "Taps"] = {}

    def __init__(self, first: np.ndarray, weights: np.ndarray, device):
        self.first = torch.from_numpy(first).to(device)
        self.weights = torch.from_numpy(weights.astype(np.float32)).to(device)
        self.taps = weights.shape[1]
        self.n_out = weights.shape[0]

    @classmethod
    def get(cls, kind: str, n_in: int, n_out: int, device) -> "Taps":
        key = (kind, n_in, n_out, torch.device(device))
        t = cls._cache.get(key)
        if t is None:
            t = cls._cache[key] = Taps(*TAPS[kind](n_in, n_out), device)
        return t


_DT = {torch.bfloat16: 0, torch.float16: 1, torch.float32: DK_F32}


def resample(x: torch.Tensor, ty: Taps, tx: Taps, out_dtype=None, depth_rgb: bool = False, out=None) -> torch.Tensor:
    """dk_resample: NHWC x (Hi, Wi, C) -> (ty.n_out, tx.n_out, C) (16-bit or fp32 both ways); depth_rgb: C == 1 and
    the output is BFL's v / 127.5 - 1 in 3 channels"""
    assert x.dim() == 3 and x.is_contiguous() and x.is_cuda and x.dtype in _DT
    Hi, Wi, C = x.shape
    out_dtype = out_dtype or x.dtype
    shape = (ty.n_out, tx.n_out, 3 if depth_rgb else C)
    if out is None:
        out = torch.empty(shape, dtype=out_dtype, device=x.device)
    assert out.dtype in _DT and out.is_contiguous() and tuple(out.shape[-3:]) == shape
    c = ops.ctx(x.device.index)
    c.call("dk_resample", _DT[x.dtype], _DT[out.dtype], ptr(x), ptr(out), Hi, Wi, C, ty.n_out, tx.n_out, ptr(ty.first),
           ptr(ty.weights), ty.taps, ptr(tx.first), ptr(tx.weights), tx.taps, 1 if depth_rgb else 0)
    return out


def add_relu(a: torch.Tensor, b=None, sum_out=None, relu_out=None):
    """dk_depth_add_relu: sum_out = a (+ b), relu_out = max(a (+ b), 0); either output may be a (in place)"""
    assert a.is_contiguous() and a.is_cuda and (sum_out is not None or relu_out is not None)
    for t in (b, sum_out, relu_out):
        assert t is None or (t.dtype == a.dtype and t.is_contiguous() and t.numel() == a.numel())
    c = ops.ctx(a.device.index)
    c.call("dk_depth_add_relu", dtype_code(a.dtype), ptr(a), ptr(b), ptr(sum_out), ptr(relu_out), a.numel())
    return sum_out if relu_out is None else relu_out


def head_tail(x: torch.Tensor, w: torch.Tensor, b: float, out=None) -> torch.Tensor:
    """dk_depth_head: x (..., C) 16-bit, w fp32 (C,) -> fp32 (...) = relu(w . relu(x) + b)"""
    assert x.is_contiguous() and x.is_cuda and w.dtype == torch.float32 and w.is_contiguous()
    C = x.shape[-1]
    assert w.numel() == C
    if out is None:
        out = torch.empty(x.shape[:-1], dtype=torch.float32, device=x.device)
    assert out.dtype == torch.float32 and out.is_contiguous() and out.numel() * C == x.numel()
    c = ops.ctx(x.device.index)
    c.call("dk_depth_head", dtype_code(x.dtype), ptr(x), ptr(w), float(b), ptr(out), out.numel(), C)
    return out


def conv3x3_s2_p1(x: torch.Tensor, w: torch.Tensor, bias=None, out=None) -> torch.Tensor:
    """dk_conv3x3_s2_p1: x NHWC [B, H, W, Cin], w [Cout, 3, 3, Cin] -> [B, ceil(H/2), ceil(W/2), Cout]"""
    ops._chk16(x, "conv3x3_s2_p1.x")
    B, H, W, Cin = x.shape
    Cout = w.shape[0]
    assert tuple(w.shape) == (Cout, 3, 3, Cin) and x.is_contiguous() and w.is_contiguous()
    if out is None:
        out = torch.empty((B, (H + 1) // 2, (W + 1) // 2, Cout), dtype=x.dtype, device=x.device)
    c = ops.ctx(x.device.index)
    c.call("dk_conv3x3_s2_p1", dtype_code(x.dtype), ptr(x), ptr(w), ptr(bias), ptr(out), B, H, W, Cin, Cout)
    return out


# ------------------------------------------------------------------------------------------------ model
class DepthAnythingModel:
    """Depth Anything's predicted_depth (transformers DepthAnythingForDepthEstimation) on the device.
    params: the engine's tree (pack_depth_params), any float dtype; it runs in `dtype` (16-bit), with the position
    table and the head's last 1 x 1 convolution kept in fp32."""

    def __init__(self, params: Dict[str, torch.Tensor], config: DepthAnythingConfig, dtype=torch.bfloat16,
                 device=None):
        check_config(config)
        _check_shapes(params, engine_depth_shapes(config), "DepthAnythingModel")
        if dtype not in (torch.bfloat16, torch.float16):
            raise ValueError(f"DepthAnythingModel runs in bf16 or fp16, got {dtype}")
        dev = torch.device(device) if device is not None else next(iter(params.values())).device
        if dev.type != "cuda":
            raise ValueError("DepthAnythingModel: parameters must live on a CUDA device (no CPU fallback)")
        self.device, self.dtype, self.config = dev, dtype, config
        self.p = {k: v.to(device=dev, dtype=torch.float32 if k in FP32_KEYS else dtype).contiguous()
                  for k, v in params.items()}
        self.conv3_bias = float(self.p["head.conv3.bias"].item())
        self.kp = patch_weight_kp(config)
        self._pos: Dict[tuple, torch.Tensor] = {}

    def _taps(self, kind, n_in, n_out):
        return Taps.get(kind, n_in, n_out, self.device)

    def position_table(self, gh: int, gw: int) -> torch.Tensor:
        """(gh gw, D) 16-bit patch position rows: the table itself on a 37 x 37 grid, else its bicubic interpolation
        (a = -0.75, align_corners=False, fp32), made once per grid"""
        t = self._pos.get((gh, gw))
        if t is None:
            g, D = self.config.pos_grid, self.config.hidden_size
            if (gh, gw) == (g, g):
                t = self.p["pos"].to(self.dtype).reshape(g * g, D)
            else:
                t = resample(self.p["pos"], self._taps("bicubic", g, gh), self._taps("bicubic", g, gw),
                             self.dtype).reshape(gh * gw, D)
            self._pos[(gh, gw)] = t
        return t

    def _rcu(self, h, t, pre: str):
        """pre-activated residual unit: conv2(relu(conv1(t))) + h, t = relu(h) already computed"""
        p = self.p
        u = ops.conv3x3(t, p[pre + ".conv1.weight"], p[pre + ".conv1.bias"])
        add_relu(u, relu_out=u)
        return ops.conv3x3(u, p[pre + ".conv2.weight"], p[pre + ".conv2.bias"], res=h)

    def __call__(self, image: torch.Tensor) -> torch.Tensor:
        """image: uint8 (h, w, 3) on the device, h and w multiples of 14 -> predicted_depth fp32 (h, w)"""
        c, p = self.config, self.p
        if image.dim() != 3 or image.dtype != torch.uint8 or image.shape[0] % 14 or image.shape[1] % 14:
            raise ValueError(f"DepthAnythingModel takes a uint8 (h, w, 3) image with h, w multiples of 14, got "
                             f"{image.dtype} {tuple(image.shape)}")
        gh, gw = image.shape[0] // c.patch_size, image.shape[1] // c.patch_size
        P, D, H, F = gh * gw, c.hidden_size, c.num_attention_heads, c.fusion_hidden_size
        S = 1 + P
        x = image_patches(image.contiguous().unsqueeze(0), self.dtype, c.patch_size, self.kp)
        h = torch.empty((S, D), dtype=self.dtype, device=self.device)
        ops.copy_rows(p["cls_pos"], h, 1, 1, D, S, 0, 1, 0)
        ops.gemm(x, p["patch.weight"], bias=p["patch.bias"], res=self.position_table(gh, gw), out=h,
                 rows_per_batch=P, out_batch_rows=S, out_row_off=1, res_batch_rows=0)
        att = torch.empty((S, D), dtype=self.dtype, device=self.device)
        eps = c.layer_norm_eps
        stages = {}
        for i in range(max(c.out_indices)):
            l = f"layers.{i}."
            y = ops.layernorm(h, p[l + "norm1.weight"], p[l + "norm1.bias"], eps)
            qkv = ops.gemm(y, p[l + "qkv.weight"], bias=p[l + "qkv.bias"])
            ops.attention(qkv, 1, S, H, 64, att)
            ops.gemm(att, p[l + "o.weight"], bias=p[l + "o.bias"], res=h, out=h)
            y = ops.layernorm(h, p[l + "norm2.weight"], p[l + "norm2.bias"], eps)
            y = ops.gemm(y, p[l + "fc1.weight"], bias=p[l + "fc1.bias"], act=ACT_GELU_ERF)
            ops.gemm(y, p[l + "fc2.weight"], bias=p[l + "fc2.bias"], res=h, out=h)
            if i + 1 in c.out_indices:
                stages[i + 1] = ops.layernorm(h, p["norm.weight"], p["norm.bias"], eps)

        feats = []
        for k, (ch, f) in enumerate(zip(c.neck_hidden_sizes, c.reassemble_factors)):
            r = ops.gemm(stages[c.out_indices[k]][1:], p[f"reassemble.{k}.proj.weight"],
                         bias=p[f"reassemble.{k}.proj.bias"])
            if f > 1:
                s = int(f)
                m = torch.empty((1, s * gh, s * gw, ch), dtype=self.dtype, device=self.device)
                for di in range(s):
                    ops.gemm(r, p[f"reassemble.{k}.resize.weight"][di], bias=p[f"reassemble.{k}.resize.bias"],
                             out=m.view(s * gh * gw, s * ch), rows_per_batch=gw, out_batch_rows=s * gw,
                             out_row_off=di * gw)
            elif f < 1:
                m = conv3x3_s2_p1(r.view(1, gh, gw, ch), p[f"reassemble.{k}.resize.weight"],
                                  p[f"reassemble.{k}.resize.bias"])
            else:
                m = r.view(1, gh, gw, ch)
            feats.append(ops.conv3x3(m, p[f"convs.{k}.weight"]))

        h = t = None
        for j in range(4):
            f = feats[3 - j]
            if h is None:
                h = f
                t = add_relu(h, relu_out=torch.empty_like(h))
            else:
                r = self._rcu(f, add_relu(f, relu_out=torch.empty_like(f)), f"fusion.{j}.rcu1")
                t = torch.empty_like(h)
                add_relu(h, r, sum_out=h, relu_out=t)
            h = self._rcu(h, t, f"fusion.{j}.rcu2")
            _, hh, hw, _ = h.shape
            th, tw = feats[2 - j].shape[1:3] if j < 3 else (2 * hh, 2 * hw)
            h = resample(h[0], self._taps("bilinear_ac", hh, th), self._taps("bilinear_ac", hw, tw))
            h = ops.gemm(h.view(th * tw, F), p[f"fusion.{j}.proj.weight"], bias=p[f"fusion.{j}.proj.bias"])
            h = h.view(1, th, tw, F)

        y = ops.conv3x3(h, p["head.conv1.weight"], p["head.conv1.bias"])
        oh, ow = c.patch_size * gh, c.patch_size * gw
        y = resample(y[0], self._taps("bilinear_ac", y.shape[1], oh), self._taps("bilinear_ac", y.shape[2], ow))
        y = ops.conv3x3(y.unsqueeze(0), p["head.conv2.weight"], p["head.conv2.bias"])
        return head_tail(y[0], p["head.conv3.weight"], self.conv3_bias)

    def depth(self, predicted: torch.Tensor, size: Tuple[int, int], rgb: bool = False) -> torch.Tensor:
        """BFL's interpolate(depth, (H, W), mode="bicubic", antialias=True) of predicted_depth (h, w) fp32 -> (H, W)
        fp32; rgb: instead (H, W, 3) in the model dtype holding depth / 127.5 - 1 in every channel (the VAE's input)"""
        H, W = size
        ph, pw = predicted.shape
        ty, tx = self._taps("bicubic_aa", ph, H), self._taps("bicubic_aa", pw, W)
        if rgb:
            return resample(predicted.view(ph, pw, 1), ty, tx, self.dtype, depth_rgb=True)
        return resample(predicted.view(ph, pw, 1), ty, tx, torch.float32).view(H, W)
