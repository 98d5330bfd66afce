"""fp32 oracle of FLUX.1 Depth's depth estimator (DESIGN.md §20) on the engine's packed tree, and the references the
GPU test's launch census needs for the estimator's own kernels.

DepthAnythingRef is transformers' DepthAnythingForDepthEstimation restated with torch.nn.functional on the packed
tree: the folds are undone only where a standard operator needs the upstream layout (the ConvTranspose slabs go back
to (I, O, s, s)), so the row-map of the engine's ConvTranspose GEMMs is not part of the oracle.  It takes the uint8
network input, as the engine does; the ImageNet normalisation is inside the folded patch weight."""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from diffusionkit_b200.config import DepthAnythingConfig


def unfold_slabs(slabs: torch.Tensor) -> torch.Tensor:
    """(s, s O, I) -> ConvTranspose2d weight (I, O, s, s)"""
    s, sO, I = slabs.shape
    return slabs.reshape(s, s, sO // s, I).permute(3, 2, 0, 1)


def oihw(w: torch.Tensor) -> torch.Tensor:
    """(O, kh, kw, I) -> OIHW"""
    return w.permute(0, 3, 1, 2)


def rcu(x, p, pre):
    y = F.conv2d(F.relu(x), oihw(p[pre + ".conv1.weight"]), p[pre + ".conv1.bias"], padding=1)
    return F.conv2d(F.relu(y), oihw(p[pre + ".conv2.weight"]), p[pre + ".conv2.bias"], padding=1) + x


class DepthAnythingRef:
    def __init__(self, params: Dict[str, torch.Tensor], cfg: DepthAnythingConfig, dtype=torch.float32):
        self.p = {k: v.detach().to("cpu", dtype) for k, v in params.items()}
        self.cfg = cfg
        self.dtype = dtype

    def __call__(self, img_u8: torch.Tensor) -> torch.Tensor:
        """uint8 (h, w, 3) -> predicted_depth (h, w)"""
        c, p = self.cfg, self.p
        D, pz, g = c.hidden_size, c.patch_size, c.pos_grid
        h_, w_ = img_u8.shape[:2]
        gh, gw = h_ // pz, w_ // pz
        u = img_u8.to("cpu", self.dtype) / 255 * 2 - 1
        x = u[:gh * pz, :gw * pz, :3].reshape(gh, pz, gw, pz, 3).permute(0, 2, 1, 3, 4).reshape(gh * gw, 3 * pz * pz)
        tok = x @ p["patch.weight"][:, :3 * pz * pz].T + p["patch.bias"]
        pos = p["pos"]
        if (gh, gw) != (g, g):
            pos = F.interpolate(pos.permute(2, 0, 1)[None].float(), size=(gh, gw), mode="bicubic",
                                align_corners=False)[0].permute(1, 2, 0).to(self.dtype)
        h = torch.cat([p["cls_pos"], tok + pos.reshape(gh * gw, D)])
        H = c.num_attention_heads
        S = h.shape[0]
        stages = {}
        for i in range(max(c.out_indices)):
            l = f"layers.{i}."
            y = F.layer_norm(h, (D,), p[l + "norm1.weight"], p[l + "norm1.bias"], c.layer_norm_eps)
            q, k, v = (y @ p[l + "qkv.weight"].T + p[l + "qkv.bias"]).reshape(S, 3, H, D // H).permute(1, 2, 0, 3)
            a = F.scaled_dot_product_attention(q, k, v).permute(1, 0, 2).reshape(S, D)
            h = h + a @ p[l + "o.weight"].T + p[l + "o.bias"]
            y = F.layer_norm(h, (D,), p[l + "norm2.weight"], p[l + "norm2.bias"], c.layer_norm_eps)
            y = F.gelu(y @ p[l + "fc1.weight"].T + p[l + "fc1.bias"])
            h = h + y @ p[l + "fc2.weight"].T + p[l + "fc2.bias"]
            if i + 1 in c.out_indices:
                stages[i + 1] = F.layer_norm(h, (D,), p["norm.weight"], p["norm.bias"], c.layer_norm_eps)
        feats = []
        for k, f in enumerate(c.reassemble_factors):
            t = stages[c.out_indices[k]][1:].T.reshape(1, D, gh, gw)
            w = p[f"reassemble.{k}.proj.weight"]
            t = F.conv2d(t, w[:, :, None, None], p[f"reassemble.{k}.proj.bias"])
            if f > 1:
                t = F.conv_transpose2d(t, unfold_slabs(p[f"reassemble.{k}.resize.weight"]),
                                       p[f"reassemble.{k}.resize.bias"][:w.shape[0]], stride=int(f))
            elif f < 1:
                t = F.conv2d(t, oihw(p[f"reassemble.{k}.resize.weight"]), p[f"reassemble.{k}.resize.bias"], stride=2,
                             padding=1)
            feats.append(F.conv2d(t, oihw(p[f"convs.{k}.weight"]), padding=1))
        h = None
        for j in range(4):
            f = feats[3 - j]
            h = f if h is None else h + rcu(f, p, f"fusion.{j}.rcu1")
            h = rcu(h, p, f"fusion.{j}.rcu2")
            size = tuple(feats[2 - j].shape[2:]) if j < 3 else (2 * h.shape[2], 2 * h.shape[3])
            h = F.interpolate(h, size=size, mode="bilinear", align_corners=True)
            h = F.conv2d(h, p[f"fusion.{j}.proj.weight"][:, :, None, None], p[f"fusion.{j}.proj.bias"])
        y = F.conv2d(h, oihw(p["head.conv1.weight"]), p["head.conv1.bias"], padding=1)
        y = F.interpolate(y, size=(pz * gh, pz * gw), mode="bilinear", align_corners=True)
        y = F.relu(F.conv2d(y, oihw(p["head.conv2.weight"]), p["head.conv2.bias"], padding=1))
        y = F.conv2d(y, p["head.conv3.weight"][None, :, None, None], p["head.conv3.bias"])
        return F.relu(y)[0, 0]


def bfl_depth(predicted: torch.Tensor, size) -> torch.Tensor:
    """BFL's interpolate(depth, (H, W), mode="bicubic", antialias=True) of one (h, w) map"""
    return F.interpolate(predicted[None, None].float(), size=tuple(size), mode="bicubic", antialias=True)[0, 0]


# ------------------------------------------------------------------------------------------------ kernel references
def ref_resample(x: torch.Tensor, ty, tx, out_dtype, depth_rgb=False) -> torch.Tensor:
    """dk_resample's statement in fp64 from the tap tables (first, weights) of each axis; x (Hi, Wi, C)"""
    (fy, wy), (fx, wx) = ty, tx
    Hi, Wi, C = x.shape
    My = torch.zeros((len(fy), Hi), dtype=torch.float64)
    for o, (i0, ws) in enumerate(zip(fy, wy)):
        for t, w in enumerate(ws):
            My[o, min(max(int(i0) + t, 0), Hi - 1)] += float(w)
    Mx = torch.zeros((len(fx), Wi), dtype=torch.float64)
    for o, (i0, ws) in enumerate(zip(fx, wx)):
        for t, w in enumerate(ws):
            Mx[o, min(max(int(i0) + t, 0), Wi - 1)] += float(w)
    v = torch.einsum("yh,hwc,xw->yxc", My, x.double().cpu(), Mx)
    if depth_rgb:
        v = (v / 127.5 - 1).expand(-1, -1, 3)
    return v.to(out_dtype)


def ref_add_relu(a, b=None):
    s = a if b is None else (a.float() + b.float()).to(a.dtype)
    return s, torch.clamp_min(s, 0)


def ref_head_tail(x: torch.Tensor, w: torch.Tensor, b: float) -> torch.Tensor:
    """dk_depth_head's statement with the kernel's rounding: fp32 products and sums in channel order, no fma"""
    r = torch.clamp_min(x.float(), 0)
    acc = torch.zeros(x.shape[:-1], dtype=torch.float32, device=x.device)
    for k in range(x.shape[-1]):
        acc = acc + w[k].float() * r[..., k]
    return torch.clamp_min(acc + torch.tensor(b, dtype=torch.float32), 0)
