"""fp32 restatement of the first-block step cache (DESIGN.md §10) on top of the oracle MMDiT: the forward split after
block 0, and a forward that applies the rule, either deciding for itself or replaying a given decision list.  Kept
beside the tests, like tests/fp8_ref.py, so no file under oracle/ changes; MMDiTRef.__call__ is untouched.

Used with oracle.sampler_ref.sample_euler as the model: it resets its cache in cache_modulation_params, as the
engine does."""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple

import torch

from oracle.mmdit_ref import MMDiTRef, _r, affine_transform, linear, rope_apply, rope_table, sdpa


class SplitMMDiTRef(MMDiTRef):
    """MMDiTRef.__call__ in three pieces: embed (-> e), block 0 (-> a), the remaining blocks (-> f), final layer."""

    def embed(self, latent, text, timestep) -> dict:
        c, dt = self.cfg, self.dt
        B, H, Wd, Cl = latent.shape
        key = float(timestep.reshape(-1)[0])
        hp, wp = H // c.patch_size, Wd // c.patch_size
        txt = self._lin(_r(text.float(), dt), "context_embedder")
        x = _r(latent.float(), dt)
        p = c.patch_size
        wconv = self.p["x_embedder.proj.weight"].float().reshape(c.hidden_size, -1)
        if c.patchify_via_reshape:
            rows = x.reshape(B, hp, p, wp, p, Cl).permute(0, 1, 3, 5, 2, 4).reshape(B, hp * wp, Cl * p * p)
            img = linear(rows, wconv, self.p["x_embedder.proj.bias"], dt)
        else:
            rows = x.reshape(B, hp, p, wp, p, Cl).permute(0, 1, 3, 2, 4, 5).reshape(B, hp * wp, p * p * Cl)
            img = linear(rows, wconv, self.p["x_embedder.proj.bias"], dt)
            mh = c.max_latent_resolution
            y0, x0 = (mh - hp) // 2, (mh - wp) // 2
            pos = self.p["x_pos_embedder.pos_embed.weight"].float().reshape(mh, mh, c.hidden_size)
            img = _r(img + pos[y0:y0 + hp, x0:x0 + wp].reshape(1, hp * wp, c.hidden_size), dt)
        T = txt.shape[1]
        return {"B": B, "H": H, "W": Wd, "Cl": Cl, "hp": hp, "wp": wp, "key": key, "T": T, "img": img, "txt": txt,
                "rope": rope_table(T, hp, wp, c.rope_axes_dim) if c.use_rope else None}

    def double_block(self, s: dict, i: int):
        c, dt, B, T, rope = self.cfg, self.dt, s["B"], s["T"], s["rope"]
        img, txt = s["img"], s["txt"]
        ibn = f"multimodal_transformer_blocks.{i}.image_transformer_block"
        tbn = f"multimodal_transformer_blocks.{i}.text_transformer_block"
        skip_text = (i == c.depth_multimodal - 1) and (c.depth_unified < 1)
        qi, ki, vi, mi, modi = self._pre_sdpa(img, ibn, s["key"], 6)
        qt, kt, vt, mt, modt = self._pre_sdpa(txt, tbn, s["key"], 2 if skip_text else 6)
        if c.depth_unified > 0:
            q, k, v = torch.cat([qt, qi], 2), torch.cat([kt, ki], 2), torch.cat([vt, vi], 2)
        else:
            q, k, v = torch.cat([qi, qt], 2), torch.cat([ki, kt], 2), torch.cat([vi, vt], 2)
        if rope is not None:
            q, k = rope_apply(q, rope, dt), rope_apply(k, rope, dt)
        d = c.hidden_size // c.num_heads
        o = _r(sdpa(q, k, v, 1.0 / math.sqrt(d)), dt).permute(0, 2, 1, 3).reshape(B, -1, c.hidden_size)
        n_img = img.shape[1]
        oi, ot = (o[:, T:], o[:, :T]) if c.depth_unified > 0 else (o[:, :n_img], o[:, n_img:])
        s["img"] = self._post_sdpa(img, oi, mi, modi, ibn, False)
        if not skip_text:
            s["txt"] = self._post_sdpa(txt, ot, mt, modt, tbn, False)

    def remaining_blocks(self, s: dict) -> torch.Tensor:
        """blocks 1.. of the double stream, then FLUX's single blocks -> f, the image stream entering the final layer"""
        c, dt, B, T, rope = self.cfg, self.dt, s["B"], s["T"], s["rope"]
        for i in range(1, c.depth_multimodal):
            self.double_block(s, i)
        if c.depth_unified > 0:
            d = c.hidden_size // c.num_heads
            u = torch.cat([s["txt"], s["img"]], dim=1)
            for i in range(c.depth_unified):
                bn = f"unified_transformer_blocks.{i}.transformer_block"
                par = c.parallel_mlp_for_unified_blocks
                q, k, v, m, mods = self._pre_sdpa(u, bn, s["key"], 3 if par else 6)
                if rope is not None:
                    q, k = rope_apply(q, rope, dt), rope_apply(k, rope, dt)
                o = _r(sdpa(q, k, v, 1.0 / math.sqrt(d)), dt).permute(0, 2, 1, 3).reshape(B, -1, c.hidden_size)
                u = self._post_sdpa(u, o, m, mods, bn, par)
            s["img"] = u[:, T:]
        return s["img"]

    def final(self, s: dict, f: torch.Tensor) -> torch.Tensor:
        c, dt, B, H, Wd, Cl, hp, wp = self.cfg, self.dt, s["B"], s["H"], s["W"], s["Cl"], s["hp"], s["wp"]
        shift, sc = self._mod[s["key"]]["final_layer"].chunk(2, dim=-1)
        y = self._lin(affine_transform(f, shift[:, None, :], sc[:, None, :], c.layer_norm_eps, dt), "final_layer.linear")
        p = c.patch_size
        if c.patchify_via_reshape:
            out = y.reshape(B, hp, wp, Cl, p, p).permute(0, 1, 4, 2, 5, 3).reshape(B, hp * p, wp * p, Cl)
        else:
            out = y.reshape(B, hp, wp, p, p, Cl).permute(0, 5, 1, 3, 2, 4).reshape(B, Cl, H, Wd).permute(0, 2, 3, 1)
        return out.contiguous()

    def __call__(self, latent, text, timestep):
        s = self.embed(latent, text, timestep)
        self.double_block(s, 0)
        return self.final(s, self.remaining_blocks(s))


class StepCacheRef:
    """The step-cache rule around a SplitMMDiTRef.  decisions: replay this list of skip flags (one per forward since the
    last reset) instead of deciding; the rel of every forward is computed and logged either way."""

    def __init__(self, ref: SplitMMDiTRef, threshold: float = 0.0, max_consecutive_skips: Optional[int] = None,
                 decisions: Optional[Sequence[bool]] = None):
        self.ref, self.threshold, self.cap = ref, float(threshold), max_consecutive_skips
        self.decisions = None if decisions is None else list(decisions)
        self.reset()

    def reset(self):
        self.r0prev, self.R, self.run = None, None, 0
        self.log: List[Tuple[Optional[float], bool]] = []

    def cache_modulation_params(self, pooled, timesteps):
        self.ref.cache_modulation_params(pooled, timesteps)
        self.reset()

    def __call__(self, latent, text, timestep):
        s = self.ref.embed(latent, text, timestep)
        e = s["img"]
        self.ref.double_block(s, 0)
        a = s["img"]
        r0 = a.float() - e.float()
        rel = None
        if self.r0prev is not None:
            num = (r0 - self.r0prev).abs().double().sum(dim=(1, 2))
            den = self.r0prev.abs().double().sum(dim=(1, 2))
            rel = max(float(n / d) if d != 0 else math.inf for n, d in zip(num, den))
        if self.decisions is not None:
            skip = bool(self.decisions[len(self.log)])
            assert not (skip and self.r0prev is None), "a replayed decision skips a forward with nothing cached"
        else:
            skip = (rel is not None and rel < self.threshold and (self.cap is None or self.run < self.cap))
        if skip:
            f = _r(a + self.R, self.ref.dt)
            self.run += 1
        else:
            f = self.ref.remaining_blocks(s)
            self.R, self.r0prev, self.run = f.float() - a.float(), r0, 0
        self.log.append((rel, skip))
        return self.ref.final(s, f)
