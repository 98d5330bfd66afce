"""Synthetic LoRA adapters for the tests, and the fp32 reference merge the GPU results are compared with.

The upstream module list comes from the upstream checkpoint layouts the checkpoint-loader tests build
(test_model_io_cpu.py), not from diffusionkit_b200.lora, so the adapter parser is checked against an independent list.
"""
from typing import Dict, List, Tuple

import torch

from tests.test_model_io_cpu import _flux_upstream, _sd3_upstream
from diffusionkit_b200.weights import init_params, mmdit_param_specs


def upstream_modules(cfg) -> Dict[str, Tuple[int, ...]]:
    """upstream module name -> weight shape, for every Linear / conv of the upstream FLUX or SD3 checkpoint layout"""
    params = init_params(mmdit_param_specs(cfg), seed=0, dtype=torch.float32)
    sd = _flux_upstream(params, cfg) if cfg.depth_unified > 0 else _sd3_upstream(params, cfg, prefix="")
    return {k[:-len(".weight")]: tuple(v.shape) for k, v in sd.items()
            if k.endswith(".weight") and v.dim() >= 2 and not k.startswith("guidance_in.")}


def make_factors(modules: Dict[str, Tuple[int, ...]], rank: int, seed: int, gain: float = 0.15,
                 alphas: bool = True) -> Dict[str, Tuple[torch.Tensor, torch.Tensor, float]]:
    """module -> (up, down, alpha) in the upstream layout (conv modules get OIHW factors), ΔW ~ gain / sqrt(fan_in)"""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for i, (m, shape) in enumerate(sorted(modules.items())):
        fan_in = 1
        for s in shape[1:]:
            fan_in *= s
        down = torch.randn((rank,) + shape[1:], generator=g) / fan_in ** 0.5
        up = torch.randn((shape[0], rank) + (1, 1) * (len(shape) == 4), generator=g) * gain / rank ** 0.5
        alpha = float(rank) * (0.5 + 0.5 * (i % 3)) if alphas else None
        if alpha is not None:
            up = up * (rank / alpha)                      # the same ΔW for every alpha
        out[m] = (up, down, alpha)
    return out


def kohya_dict(factors) -> Dict[str, torch.Tensor]:
    sd = {}
    for m, (up, down, alpha) in factors.items():
        k = "lora_unet_" + m.replace(".", "_")
        sd[k + ".lora_down.weight"], sd[k + ".lora_up.weight"] = down, up
        sd[k + ".alpha"] = torch.tensor(alpha if alpha is not None else float(down.shape[0]))
    return sd


def peft_dict(factors, prefix: str = "") -> Dict[str, torch.Tensor]:
    sd = {}
    for m, (up, down, alpha) in factors.items():
        sd[f"{prefix}{m}.lora_A.weight"], sd[f"{prefix}{m}.lora_B.weight"] = down, up
        if alpha is not None:
            sd[f"{prefix}{m}.alpha"] = torch.tensor(alpha)
    return sd


def upstream_delta(factors) -> Dict[str, torch.Tensor]:
    """module.weight -> ΔW = alpha / rank · up @ down in the upstream weight's own shape"""
    out = {}
    for m, (up, down, alpha) in factors.items():
        r = down.shape[0]
        a = alpha if alpha is not None else float(r)
        out[m + ".weight"] = ((a / r) * up.reshape(up.shape[0], r) @ down.reshape(r, -1)).reshape(
            (up.shape[0],) + tuple(down.shape[1:]))
    return out


def merge_lora(params: Dict[str, torch.Tensor], targets_with_scales: List[tuple]) -> Dict[str, torch.Tensor]:
    """fp32 reference merge on reference-named params: W + Σ scale · up @ down for every target of every adapter"""
    out = {k: v.detach().to("cpu", torch.float32).clone() for k, v in params.items()}
    for targets, scale in targets_with_scales:
        for name, (up, down) in targets.items():
            out[name] += (scale * (up.float() @ down.float())).reshape(out[name].shape)
    return out
