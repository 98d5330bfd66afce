"""CPU fp32 restatement of FLUX.1 Kontext's input convention (DESIGN.md §14) on top of tests/guidance_ref.py's
GuidanceMMDiTRef.  Kept beside the tests, like tests/guidance_ref.py, so no file under oracle/ changes.

No runnable Kontext reference exists here, so the forward is written ids-driven, as BFL's and diffusers' FLUX
transformers are: the image-stream tokens come in any order together with their (axis0, r, c) ids, the RoPE angles are
computed from those ids at the rounding points of oracle.mmdit_ref.rope_table, and the output rows are picked by index.
tests/test_kontext_cpu.py pins it by properties (no reference tokens give the parent oracle exactly, a permuted
sequence only reassociates, the ids equal a transcription of BFL's prepare_kontext).

    ids(text)      = (0, 0, 0)
    ids(target)    = (0, r, c),  r < H/2, c < W/2
    ids(reference) = (1, r, c),  r < Hr/2, c < Wr/2
    output         = final_layer(image stream)[target rows]
"""
from __future__ import annotations

import math
from typing import Callable, Optional, Sequence

import torch

from oracle.mmdit_ref import MMDiTRef, _r, affine_transform, linear, rope_apply, sdpa
from tests.guidance_ref import GuidanceMMDiTRef
from tests.step_cache_ref import SplitMMDiTRef


def sharpen(params: dict, gain: float = 2.0) -> dict:
    """params with every QK-RMSNorm weight times `gain`: sharper attention, as in a trained model.  With the synthetic
    initialiser's flat attention a reference's axis-0 id moves the tiny model's output by about 1 % only, which the
    2e-2 forward bound could not tell apart; at gain 2 it moves it by about 10 % (tests/test_kontext_cpu.py), while the
    16-bit rounding error grows from about 0.7 % to 1.1 % (an oracle rounding at bf16 against the fp32 one).  At gain 3
    that error reaches the bound."""
    return {k: (v * gain if ".qk_norm." in k else v) for k, v in params.items()}


def grid_ids(hp: int, wp: int, axis0: float = 0.0) -> torch.Tensor:
    """(hp * wp, 3) fp32 ids of a packed latent grid, row-major: (axis0, r, c)"""
    ids = torch.zeros((hp * wp, 3), dtype=torch.float32)
    ids[:, 0] = axis0
    ids[:, 1] = torch.arange(hp, dtype=torch.float32)[:, None].expand(hp, wp).reshape(-1)
    ids[:, 2] = torch.arange(wp, dtype=torch.float32)[None, :].expand(hp, wp).reshape(-1)
    return ids


def kontext_ids(T: int, hp: int, wp: int, ref_grid=None, ref_axis0: float = 1.0) -> torch.Tensor:
    """ids of the joint sequence [text | target | reference] -> (T + hp·wp (+ hpr·wpr), 3)"""
    parts = [torch.zeros((T, 3), dtype=torch.float32), grid_ids(hp, wp)]
    if ref_grid is not None:
        parts.append(grid_ids(*ref_grid, axis0=ref_axis0))
    return torch.cat(parts)


def rope_from_ids(ids: torch.Tensor, axes_dim, theta: float = 10000.0) -> torch.Tensor:
    """oracle.mmdit_ref.rope_table with the positions given: (S, 3) ids -> (S, D/2, 2) (cos, sin)"""
    outs = []
    for a, dim in enumerate(axes_dim):
        scale = torch.arange(0, dim, 2, dtype=torch.float32) / dim
        omega = 1.0 / (theta ** scale)
        outs.append(ids[:, a:a + 1] * omega[None, :])
    ang = torch.cat(outs, dim=-1)
    return torch.stack([torch.cos(ang), torch.sin(ang)], dim=-1)


def patch_rows(latent: torch.Tensor, p: int = 2) -> torch.Tensor:
    """FLUX packing (mmdit.py:292-302): (B, H, W, C) -> (B, H/p · W/p, C·p·p)"""
    B, H, W, C = latent.shape
    return latent.reshape(B, H // p, p, W // p, p, C).permute(0, 1, 3, 5, 2, 4).reshape(B, (H // p) * (W // p),
                                                                                       C * p * p)


def unpack_rows(y: torch.Tensor, H: int, W: int, C: int, p: int = 2) -> torch.Tensor:
    """the inverse of patch_rows (mmdit.py:304-321): (B, H/p · W/p, C·p·p) -> (B, H, W, C)"""
    B = y.shape[0]
    return y.reshape(B, H // p, W // p, C, p, p).permute(0, 1, 4, 2, 5, 3).reshape(B, H, W, C).contiguous()


class KontextMMDiTRef(GuidanceMMDiTRef):
    """FLUX forward over an explicit token list.  Without a guidance embedder (schnell-shaped weights) pass guidance
    None to cache_modulation_params: the modulation cache is then MMDiTRef's."""

    def cache_modulation_params(self, pooled: torch.Tensor, timesteps: torch.Tensor, guidance=None):
        if guidance is None:
            MMDiTRef.cache_modulation_params(self, pooled, timesteps)
        else:
            super().cache_modulation_params(pooled, timesteps, guidance)

    def forward_tokens(self, text: torch.Tensor, rows: torch.Tensor, ids: torch.Tensor, timestep: torch.Tensor,
                       out_rows) -> torch.Tensor:
        """text (B, T, E); rows (B, N, C·p·p): the packed image-stream tokens in any order; ids (T + N, 3): the id of
        every token of [text | image stream]; out_rows: indices into the image stream -> final layer rows
        (B, len(out_rows), C·p·p)"""
        c, dt = self.cfg, self.dt
        assert c.depth_unified > 0 and c.use_rope, "Kontext is a FLUX forward"
        key = float(timestep.reshape(-1)[0])
        B = rows.shape[0]
        d = c.hidden_size // c.num_heads
        txt = self._lin(_r(text.float(), dt), "context_embedder")
        wconv = self.p["x_embedder.proj.weight"].float().reshape(c.hidden_size, -1)
        img = linear(_r(rows.float(), dt), wconv, self.p["x_embedder.proj.bias"], dt)
        T = txt.shape[1]
        assert ids.shape == (T + img.shape[1], 3)
        rope = rope_from_ids(ids, c.rope_axes_dim)
        scale = 1.0 / math.sqrt(d)
        for i in range(c.depth_multimodal):
            ibn = f"multimodal_transformer_blocks.{i}.image_transformer_block"
            tbn = f"multimodal_transformer_blocks.{i}.text_transformer_block"
            qi, ki, vi, mi, modi = self._pre_sdpa(img, ibn, key, 6)
            qt, kt, vt, mt, modt = self._pre_sdpa(txt, tbn, key, 6)
            q, k, v = torch.cat([qt, qi], 2), torch.cat([kt, ki], 2), torch.cat([vt, vi], 2)
            q, k = rope_apply(q, rope, dt), rope_apply(k, rope, dt)
            o = _r(sdpa(q, k, v, scale), dt).permute(0, 2, 1, 3).reshape(B, -1, c.hidden_size)
            img = self._post_sdpa(img, o[:, T:], mi, modi, ibn, False)
            txt = self._post_sdpa(txt, o[:, :T], mt, modt, tbn, False)
        u = torch.cat([txt, img], dim=1)
        for i in range(c.depth_unified):
            bn = f"unified_transformer_blocks.{i}.transformer_block"
            q, k, v, m, mods = self._pre_sdpa(u, bn, key, 3)
            q, k = rope_apply(q, rope, dt), rope_apply(k, rope, dt)
            o = _r(sdpa(q, k, v, scale), dt).permute(0, 2, 1, 3).reshape(B, -1, c.hidden_size)
            u = self._post_sdpa(u, o, m, mods, bn, True)
        img = u[:, T:][:, torch.as_tensor(out_rows, dtype=torch.long)]
        shift, sc = self._mod[key]["final_layer"].chunk(2, dim=-1)
        y = affine_transform(img, shift[:, None, :], sc[:, None, :], c.layer_norm_eps, dt)
        return self._lin(y, "final_layer.linear")

    def __call__(self, latent: torch.Tensor, text: torch.Tensor, timestep: torch.Tensor,
                 reference: Optional[torch.Tensor] = None, ref_axis0: float = 1.0) -> torch.Tensor:
        """latent (B, H, W, 16), text (B, T, E), timestep (B,), reference (B, Hr, Wr, 16) or None -> (B, H, W, 16).
        ref_axis0: the reference tokens' axis-0 id (1 in Kontext; tests set 0 to show that it matters)"""
        c, dt = self.cfg, self.dt
        p = c.patch_size
        B, H, W, Cl = latent.shape
        rows = patch_rows(_r(latent.float(), dt), p)
        ref_grid = None
        if reference is not None:
            rows = torch.cat([rows, patch_rows(_r(reference.float(), dt), p)], dim=1)
            ref_grid = (reference.shape[1] // p, reference.shape[2] // p)
        ids = kontext_ids(text.shape[1], H // p, W // p, ref_grid, ref_axis0)
        y = self.forward_tokens(text, rows, ids, timestep, torch.arange((H // p) * (W // p)))
        return unpack_rows(y, H, W, Cl, p)


def kontext_pipeline_latents(ref_model: Callable[[], KontextMMDiTRef], sample, sigmas, x0s, cond, pooled,
                             references: Sequence[Optional[torch.Tensor]], guidance: Sequence[Optional[float]],
                             cfg_weight: float, act_dtype, model_hook=None) -> torch.Tensor:
    """The oracle pipeline one image at a time: image i starts from x0s[i], takes rows [i, i + n] (CFG) of cond and
    pooled, guidance[i] (None: no embedder) and the (1, Hr, Wr, 16) reference latent references[i]; `sample` is
    oracle.sampler_ref.sample_euler or a tests/solver_ref sampler, whose model closes over the reference.
    model_hook(ref, i) may wrap each image's model call (e.g. to replay step-cache decisions).
    -> process_out latents (n, H, W, 16)."""
    from oracle import sampler_ref as sr

    n = len(x0s)
    reps = 2 if cfg_weight > 0 else 1
    outs = []
    for i in range(n):
        ref = ref_model()
        idx = [i + k * n for k in range(reps)]
        r = references[i]

        def call(xin, c, t, ref=ref, r=r):
            rr = None if r is None else r.float().expand(xin.shape[0], -1, -1, -1)
            return ref(xin, c, t, reference=rr)

        if model_hook is not None:
            call = model_hook(call, i)
        g = guidance[i]
        x = sample(call, lambda pp, ts, ref=ref, g=g: ref.cache_modulation_params(pp, ts, None if g is None
                                                                                    else [g] * reps),
                   x0s[i], sigmas, cond[idx].float(), pooled[idx].float(), cfg_weight, act_dtype)
        outs.append(sr.process_out(x, "flux"))
    return torch.cat(outs)


class KontextSplitRef(SplitMMDiTRef):
    """tests/step_cache_ref.SplitMMDiTRef with the Kontext reference tokens: `reference` ((1, Hr, Wr, 16) or None) is
    appended to the image stream of every forward, the RoPE table follows kontext_ids, and the final layer reads the
    target rows.  The step-cache rule of tests/step_cache_ref.StepCacheRef then runs on the whole stream."""

    reference: Optional[torch.Tensor] = None

    def embed(self, latent, text, timestep) -> dict:
        s = super().embed(latent, text, timestep)
        r = self.reference
        if r is None:
            return s
        c, dt, p = self.cfg, self.dt, self.cfg.patch_size
        rows = patch_rows(_r(r.float().expand(s["B"], -1, -1, -1), dt), p)
        wconv = self.p["x_embedder.proj.weight"].float().reshape(c.hidden_size, -1)
        s["Nx"] = s["img"].shape[1]
        s["img"] = torch.cat([s["img"], linear(rows, wconv, self.p["x_embedder.proj.bias"], dt)], dim=1)
        s["rope"] = rope_from_ids(kontext_ids(s["T"], s["hp"], s["wp"], (r.shape[1] // p, r.shape[2] // p)),
                                  c.rope_axes_dim)
        return s

    def final(self, s: dict, f: torch.Tensor) -> torch.Tensor:
        return super().final(s, f[:, :s["Nx"]] if "Nx" in s else f)
