"""CPU fp32 restatement of SD3.5 Medium's MMDiT-X forward and of skip-layer guidance (DESIGN.md §13), on top of
oracle.mmdit_ref.MMDiTRef and the solver loops of oracle.sampler_ref / tests/solver_ref.py.  Kept beside the tests,
like tests/guidance_ref.py, so no file under oracle/ changes.

No runnable reference exists for MMDiT-X, so tests/test_sd35_medium_cpu.py pins this restatement by properties (a zero
attn2 output is MMDiTRef, one x-block equals an fp64 transcription of Stability's pre_attention_x / post_attention_x,
block 0's attn2 ignores the text, the k bias matters).  An x-block, modulation chunks in Stability's order
(shift, scale, gate)_msa, (shift, scale, gate)_mlp, (shift, scale, gate)_msa2:

    n  = LN(x)
    o  = joint attention of attn.qkv(n (1 + scale_msa) + shift_msa) with the text stream
    o2 = attention over the image tokens of RMSNorm'd attn2.qkv(n (1 + scale_msa2) + shift_msa2)
    x += gate_msa · attn.proj(o);  x += gate_msa2 · attn2.proj(o2)
    x += gate_mlp · MLP(LN(x) (1 + scale_mlp) + shift_mlp)

Skip-layer guidance, Stability's SkipLayerCFGDenoiser: on the steps i of n with start·n < i < end·n,
D = D_neg + w (D_pos - D_neg) + s (D_pos - D_skip), D_skip the positive prompt's estimate from a forward that skips the
listed joint blocks entirely.
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import torch

from oracle.mmdit_ref import MMDiTRef, _r, affine_transform, linear, rms_norm, sdpa


class MMDiTXRef(MMDiTRef):
    """MMDiTRef's SD3 branch with MMDiT-X blocks (`x_layers`), the q/k/v k bias kept (`k_bias`) and joint blocks
    skipped (`skip_layers` of __call__).  Rounds at the same 16-bit points as MMDiTRef.  A forward of B rows takes the
    leading B rows of the modulation cache: under CFG ([pos | neg]) a forward of the positive rows alone is the skip
    forward of skip-layer guidance."""

    def __init__(self, cfg, params, act_dtype: Optional[torch.dtype] = None, x_layers: Sequence[int] = (),
                 k_bias: bool = False):
        super().__init__(cfg, params, act_dtype)
        assert cfg.depth_unified == 0, "MMDiT-X is an SD3-family block"
        self.x_layers, self.k_bias = set(x_layers), k_bias

    def _qkv(self, m, attn, norm):
        """q, k, v (B, heads, S, d) of the modulated input m through `attn` ({q,k,v}_proj), per-head RMSNorm `norm`"""
        c = self.cfg
        B, S, _ = m.shape
        d = c.hidden_size // c.num_heads

        def heads(t):
            return t.reshape(B, S, c.num_heads, d).permute(0, 2, 1, 3)

        q = heads(self._lin(m, attn + ".q_proj"))
        k = heads(self._lin(m, attn + ".k_proj", bias=self.k_bias))
        v = heads(self._lin(m, attn + ".v_proj"))
        if c.use_qk_norm:
            q = rms_norm(q, self.p[norm + ".q_norm.weight"], 1e-6, self.dt)
            k = rms_norm(k, self.p[norm + ".k_norm.weight"], 1e-6, self.dt)
        return q, k, v

    def _mlp_post(self, x, mods, bn):
        c = self.cfg
        m2 = affine_transform(x, mods[3][:, None, :], mods[4][:, None, :], c.layer_norm_eps, self.dt)
        h1 = _r(self._gelu(self._lin(m2, bn + ".mlp.fc1")), self.dt)
        return _r(x + mods[5][:, None, :] * self._lin(h1, bn + ".mlp.fc2"), self.dt)

    def __call__(self, latent, text, timestep, skip_layers: Sequence[int] = ()):
        c, dt = self.cfg, self.dt
        B, H, Wd, Cl = latent.shape
        key = float(timestep.reshape(-1)[0])
        hp, wp, p = H // c.patch_size, Wd // c.patch_size, c.patch_size
        d = c.hidden_size // c.num_heads
        scale = 1.0 / math.sqrt(d)
        eps = c.layer_norm_eps

        txt = self._lin(_r(text.float(), dt), "context_embedder")
        rows = _r(latent.float(), dt).reshape(B, hp, p, wp, p, Cl).permute(0, 1, 3, 2, 4, 5).reshape(B, hp * wp, -1)
        wconv = self.p["x_embedder.proj.weight"].float().reshape(c.hidden_size, -1)   # (O, kh, kw, I) flattened
        img = linear(rows, wconv, self.p["x_embedder.proj.bias"], dt)
        mh = c.max_latent_resolution
        y0, x0 = (mh - hp) // 2, (mh - wp) // 2
        pos = self.p["x_pos_embedder.pos_embed.weight"].float().reshape(mh, mh, c.hidden_size)
        img = _r(img + pos[y0:y0 + hp, x0:x0 + wp].reshape(1, hp * wp, c.hidden_size), dt)
        N = img.shape[1]

        for i in range(c.depth_multimodal):
            if i in skip_layers:
                continue
            ibn = f"multimodal_transformer_blocks.{i}.image_transformer_block"
            tbn = f"multimodal_transformer_blocks.{i}.text_transformer_block"
            skip_text = i == c.depth_multimodal - 1
            x_block = i in self.x_layers
            modi = self._mod[key][ibn][:B].chunk(9 if x_block else 6, dim=-1)
            modt = self._mod[key][tbn][:B].chunk(2 if skip_text else 6, dim=-1)
            mi = affine_transform(img, modi[0][:, None, :], modi[1][:, None, :], eps, dt)
            mt = affine_transform(txt, modt[0][:, None, :], modt[1][:, None, :], eps, dt)
            qi, ki, vi = self._qkv(mi, ibn + ".attn", ibn + ".qk_norm")
            qt, kt, vt = self._qkv(mt, tbn + ".attn", tbn + ".qk_norm")
            q, k, v = torch.cat([qi, qt], 2), torch.cat([ki, kt], 2), torch.cat([vi, vt], 2)
            o = _r(sdpa(q, k, v, scale), dt).permute(0, 2, 1, 3).reshape(B, -1, c.hidden_size)
            oi, ot = o[:, :N], o[:, N:]
            x = _r(img + self._lin(oi, ibn + ".attn.o_proj") * modi[2][:, None, :], dt)
            if x_block:
                m2 = affine_transform(img, modi[6][:, None, :], modi[7][:, None, :], eps, dt)
                q2, k2, v2 = self._qkv(m2, ibn + ".attn2", ibn + ".qk_norm2")
                o2 = _r(sdpa(q2, k2, v2, scale), dt).permute(0, 2, 1, 3).reshape(B, -1, c.hidden_size)
                x = _r(x + self._lin(o2, ibn + ".attn2.o_proj") * modi[8][:, None, :], dt)
            img = self._mlp_post(x, modi, ibn)
            if not skip_text:
                xt = _r(txt + self._lin(ot, tbn + ".attn.o_proj") * modt[2][:, None, :], dt)
                txt = self._mlp_post(xt, modt, tbn)

        shift, sc = self._mod[key]["final_layer"][:B].chunk(2, dim=-1)
        y = self._lin(affine_transform(img, shift[:, None, :], sc[:, None, :], eps, dt), "final_layer.linear")
        out = y.reshape(B, hp, wp, p, p, Cl).permute(0, 5, 1, 3, 2, 4).reshape(B, Cl, H, Wd).permute(0, 2, 3, 1)
        return out.contiguous()


# ------------------------------------------------------------------------------------------------ skip-layer guidance
def slg_window(n: int, start: float, end: float):
    """Stability's window: the steps i of the n run with start·n < i < end·n"""
    return [i for i in range(n) if start * n < i < end * n]


def slg_denoiser(model: MMDiTXRef, x, conditioning, timestep, sigma, cfg_weight, cast, scale=0.0, layers=(),
                 active=False):
    """CFG-mixed calculate_denoised (as oracle.sampler_ref.sample_euler inlines it) plus, when `active`,
    scale · (D_pos - D_skip) with D_skip from a forward of the positive rows that skips `layers`"""
    xin = cast(torch.cat([x, x], dim=0))
    out = model(xin, conditioning, timestep.reshape(1).repeat(xin.shape[0]))
    den = xin - out * sigma
    den_text, den_neg = den.chunk(2, dim=0)
    den = den_neg + cfg_weight * (den_text - den_neg)
    if active:
        B = x.shape[0]
        den_skip = den_text      # skipping no block is the positive forward (a batch of B may round differently)
        if layers:
            xs = cast(x)
            out_s = model(xs, conditioning[:B], timestep.reshape(1).repeat(B), skip_layers=tuple(layers))
            den_skip = xs - out_s * sigma
        den = den + scale * (den_text - den_skip)
    return den


def sample(solver: str, model: MMDiTXRef, x, sigmas, conditioning, pooled, cfg_weight: float,
           act_dtype: Optional[torch.dtype], scale: float = 0.0, layers=(), start: float = 0.0, end: float = 0.0):
    """Euler / Heun / DPM-Solver++(2M) under CFG with skip-layer guidance, the update arithmetic of
    oracle.sampler_ref.sample_euler and tests/solver_ref.py; both Heun evaluations of a step take its decision."""
    from tests.solver_ref import _lambda

    def cast(t):
        return t if act_dtype is None else t.to(act_dtype).to(torch.float32)

    timesteps = cast(sigmas * 1000.0)
    model.cache_modulation_params(pooled, timesteps)
    n = len(sigmas) - 1
    window = set(slg_window(n, start, end))
    den_prev, h_prev = None, None
    for i in range(n):
        sigma, sigma_next = float(sigmas[i]), float(sigmas[i + 1])

        def D(xx, t, s):
            return slg_denoiser(model, xx, conditioning, t, s, cfg_weight, cast, scale, layers, i in window)

        den = D(x, timesteps[i], sigma)
        if solver == "euler" or (solver == "heun" and sigma_next == 0):
            d = (x - den) / sigma
            x = x + d * (sigma_next - sigma)
        elif solver == "heun":
            d = (x - den) / sigma
            x2 = x + d * (sigma_next - sigma)
            d2 = (x2 - D(x2, timesteps[i + 1], sigma_next)) / sigma_next
            x = x + (d + d2) / 2 * (sigma_next - sigma)
        else:
            if sigma_next == 0:
                x = den
                continue
            h = _lambda(sigma_next) - _lambda(sigma)
            if i >= 1 and math.isfinite(h_prev) and i < n - 2:
                r = h_prev / h
                den_d = (1 + 1 / (2 * r)) * den - (1 / (2 * r)) * den_prev
            else:
                den_d = den
            x = (sigma_next / sigma) * x - (1.0 - sigma_next) * math.expm1(-h) * den_d
            den_prev, h_prev = den, h
    return x
