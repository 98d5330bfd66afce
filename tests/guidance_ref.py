"""CPU fp32 restatement of FLUX.1-dev's guidance embedder (DESIGN.md §12) on top of oracle.mmdit_ref.MMDiTRef.  Kept
beside the tests, like tests/solver_ref.py, so no file under oracle/ changes.

The reference cannot pin it: its own guidance_embed branch feeds the timestep embedding through guidance_in (quirk Q1).
It states BFL's formula instead, and tests/test_guidance_cpu.py pins it by properties (a zero embedder is the plain
oracle, the vector equals a numpy evaluation, g = 3.5 enters as 3504):

    vec = t_embedder(sinusoid_Q5(t)) + y_embedder(pooled) + guidance_in(sinusoid_g(v))
    v   = round_act(1000 · round_act(g))
    sinusoid_g(v) = round_act(cat[cos(v·f), sin(v·f)]),  f_k = exp(-ln(max_period)·k/half), fp32 angles
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle.mmdit_ref import MMDiTRef, _r, timestep_embedding


def guidance_input(guidance, act_dtype: torch.dtype) -> torch.Tensor:
    """v = round_act(1000 · round_act(g)): BFL's guidance tensor in the model dtype times time_factor 1000 -> (B,) fp32"""
    g = torch.as_tensor(guidance, dtype=torch.float32).reshape(-1)
    return (g.to(act_dtype).float() * 1000.0).to(act_dtype).float()


def guidance_sinusoid(v: torch.Tensor, frequency_embed_dim: int, max_period: float,
                      act_dtype: torch.dtype) -> torch.Tensor:
    """BFL timestep_embedding of v: fp32 angles, cos first, rounded to the activation dtype -> (B, dim) fp32"""
    half = frequency_embed_dim // 2
    f = torch.exp(-math.log(max_period) * torch.arange(0, half, dtype=torch.float32) / half)
    ang = v.float()[:, None] * f[None, :]
    return torch.cat([torch.cos(ang), torch.sin(ang)], dim=-1).to(act_dtype).float()


class GuidanceMMDiTRef(MMDiTRef):
    """MMDiTRef whose modulation cache adds guidance_in(sinusoid_g(v)) to the conditioning vector.  act_dtype of the
    rounding rule is the config dtype (bf16 for FLUX); the embedder output is rounded like the other embedders'."""

    def guidance_vector(self, guidance) -> torch.Tensor:
        c = self.cfg
        v = guidance_input(guidance, c.dtype)
        return self._mlp_embedder(guidance_sinusoid(v, c.frequency_embed_dim, c.max_period, c.dtype), "guidance_in")

    def cache_modulation_params(self, pooled: torch.Tensor, timesteps: torch.Tensor, guidance=None):
        """guidance: one value per row of pooled"""
        B = pooled.shape[0]
        gvec = self.guidance_vector(guidance)
        assert gvec.shape[0] == B, "one guidance value per conditioning row"
        y = _r(self._mlp_embedder(pooled.float(), "y_embedder") + gvec, self.dt)
        for t in timesteps.reshape(-1):
            temb = timestep_embedding(t.reshape(1).repeat(B), self.cfg)
            tvec = self._mlp_embedder(temb, "t_embedder")
            sc = _r(F.silu(_r(y + tvec, self.dt)), self.dt)
            self._mod[float(t)] = {bn: self._lin(sc, bn + ".adaLN_modulation.layers.1") for bn in self.block_names()}
