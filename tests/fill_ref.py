"""CPU fp32 restatement of FLUX.1 Fill [dev]'s input convention (DESIGN.md §18) on top of tests/kontext_ref.py's
KontextMMDiTRef (itself tests/guidance_ref.py's GuidanceMMDiTRef), so no file under oracle/ changes.

BFL's prepare_fill is transcribed with einops and its literal rearrange strings; the forward runs the CONCATENATED
(h, 64 + 320) x-embedder on [x | img_cond | mask] in fp32, where the engine splits it into a per-call conditioning term
and a per-step latent term.  Also here: a plain-loop statement of the mask-channel index formula, pipeline drivers over
the existing oracle samplers, and the launch-census references of fill.image_pre_masked and fill.fill_cond_rows."""
from __future__ import annotations

import numpy as np
import torch
from einops import rearrange

from oracle.mmdit_ref import _r
from tests.kontext_ref import KontextMMDiTRef, kontext_ids, patch_rows, unpack_rows


# ------------------------------------------------------------------------------------------------ prepare_fill
def bfl_img_cond(src_u8, mask) -> torch.Tensor:
    """BFL: img / 127.5 - 1 as the reference normalises it, (x / 255) * 2 - 1, times (1 - mask); (H, W, >=3) uint8 and
    (H, W) 0/1 -> (1, H, W, 3) fp32 (NHWC; masked pixels may be -0.0)"""
    x = torch.as_tensor(np.asarray(src_u8))[..., :3].float() / 255 * 2 - 1.0
    m = torch.as_tensor(np.asarray(mask)).float()
    return (x * (1.0 - m[..., None]))[None]


def bfl_pack_latent(lat_nhwc: torch.Tensor) -> torch.Tensor:
    """(B, H, W, 16) -> (B, (H/2)(W/2), 64): BFL's "b c (h ph) (w pw) -> b (h w) (c ph pw)" on the NCHW latent"""
    return rearrange(lat_nhwc.permute(0, 3, 1, 2), "b c (h ph) (w pw) -> b (h w) (c ph pw)", ph=2, pw=2)


def bfl_pack_mask(mask) -> torch.Tensor:
    """(H, W) 0/1 pixel mask -> (1, (H/16)(W/16), 256) fp32, BFL's two rearranges"""
    m = torch.as_tensor(np.asarray(mask)).float()[None]
    m = rearrange(m, "b (h ph1) (w pw1) -> b (ph1 pw1) h w", ph1=8, pw1=8)
    return rearrange(m, "b c (h ph) (w pw) -> b (h w) (c ph pw)", ph=2, pw=2)


def loop_mask_channels(mask) -> np.ndarray:
    """the index formula, one element at a time: token (h, w), channel c * 4 + ph * 2 + pw with c = ph1 * 8 + pw1 holds
    mask[(2h + ph) * 8 + ph1, (2w + pw) * 8 + pw1]"""
    m = np.asarray(mask)
    Ht, Wt = m.shape[0] // 16, m.shape[1] // 16
    out = np.zeros((Ht * Wt, 256), dtype=np.float32)
    for h in range(Ht):
        for w in range(Wt):
            for ph1 in range(8):
                for pw1 in range(8):
                    for ph in range(2):
                        for pw in range(2):
                            c = ph1 * 8 + pw1
                            out[h * Wt + w, c * 4 + ph * 2 + pw] = m[(2 * h + ph) * 8 + ph1, (2 * w + pw) * 8 + pw1]
    return out


def ref_image_pre_masked(img_u8, mask, dtype, cpad: int = 64) -> torch.Tensor:
    """dk_image_pre_masked's reference: tests/kernel_checks.ref_image_pre with every masked pixel +0.  (1, H, W, >=3)
    uint8 and (H, W) -> (1, H, W, cpad) dtype on img_u8's device"""
    from tests.kernel_checks import ref_image_pre

    ref = ref_image_pre(img_u8.cpu(), dtype, cpad)
    ref[0][mask.cpu() != 0] = 0
    return ref.to(img_u8.device)


def ref_cond_rows(lat_rows, mask) -> torch.Tensor:
    """dk_fill_cond_rows' reference: [lat_rows | bfl_pack_mask(mask != 0)] in lat_rows' dtype"""
    m = bfl_pack_mask((mask.cpu() != 0).to(torch.uint8).numpy())[0]
    return torch.cat([lat_rows.cpu(), m.to(lat_rows.dtype)], dim=1).to(lat_rows.device)


def oracle_cond_rows(enc, src_u8, mask, shift: float, scale: float, dtype) -> torch.Tensor:
    """the whole conditioning in the oracle: BFL's img_cond through an oracle.vae_ref.VAEEncoderRef, its posterior mean,
    (mean - shift) * scale rounded to dtype, packed, then the packed mask -> (N, 320) fp32 holding dtype values"""
    hidden = enc(bfl_img_cond(src_u8, mask))
    mean = hidden[..., :hidden.shape[-1] // 2]
    lat = _r((mean - shift) * scale, dtype)
    return torch.cat([bfl_pack_latent(lat)[0], bfl_pack_mask(mask)[0]], dim=1)


# ------------------------------------------------------------------------------------------------ forward
class FillMMDiTRef(KontextMMDiTRef):
    """FLUX forward with the concatenated x-embedder: every token is [x | cond], cond the (N, 320) rows of
    oracle_cond_rows, shared by every sequence"""

    cond: torch.Tensor = None

    def __call__(self, latent, text, timestep, reference=None):
        assert reference is None, "FLUX.1 Fill takes no Kontext reference"
        c, dt = self.cfg, self.dt
        p = c.patch_size
        B, H, W, Cl = latent.shape
        rows = patch_rows(_r(latent.float(), dt), p)
        rows = torch.cat([rows, self.cond.float()[None].expand(B, -1, -1)], dim=-1)
        ids = kontext_ids(text.shape[1], H // p, W // p)
        y = self.forward_tokens(text, rows, ids, timestep, torch.arange((H // p) * (W // p)))
        return unpack_rows(y, H, W, Cl, p)


def fill_pipeline_latents(make_ref, solver: str, sigmas, x0s, cond_rows, cond, pooled, guidance, cfg_weight: float,
                          act_dtype, seeds) -> torch.Tensor:
    """The oracle pipeline one image at a time: image i starts from x0s[i] (img2img's start), takes rows [i, i + n] of
    cond and pooled (CFG) and guidance[i]; solver "euler", "dpmpp_2m" or "dpmpp_2m_sde" (tests/inpaint_ref.sample with
    a mask that keeps nothing, so no blend) -> process_out latents (n, H, W, 16)"""
    from oracle import sampler_ref as sr
    from tests import inpaint_ref

    n = len(x0s)
    reps = 2 if cfg_weight > 0 else 1
    outs = []
    for i in range(n):
        ref = make_ref()
        ref.cond = cond_rows
        idx = [i + k * n for k in range(reps)]
        x0 = x0s[i]
        nothing_kept = torch.ones(x0.shape[1:3], dtype=torch.uint8)
        x = inpaint_ref.sample_model(
            solver, lambda xin, cc, t, ref=ref: ref(xin, cc, t),
            lambda pp, ts, ref=ref, g=guidance[i]: ref.cache_modulation_params(pp, ts, [g] * reps),
            x0, sigmas, cond[idx].float(), pooled[idx].float(), cfg_weight, act_dtype, eps=x0, x0=x0,
            mask=nothing_kept, seed=seeds[i])
        outs.append(sr.process_out(x, "flux"))
    return torch.cat(outs)


# ------------------------------------------------------------------------------------------------ census checks
def census_check_image_pre_masked(L, a, s, r, census):
    """tests/launch_parity check of one fill.image_pre_masked launch, bit for bit"""
    L.exact("x16", r, ref_image_pre_masked(s["img_u8"], s["mask"], a["dtype"], a["cpad"]))
    L.own(r)
    L.sig.update(H=r.shape[1], W=r.shape[2], cpad=r.shape[3], masked=round(float((s["mask"] != 0).float().mean()), 3),
                 dtype=str(r.dtype)[6:])


def census_check_cond_rows(L, a, s, r, census):
    """tests/launch_parity check of one fill.fill_cond_rows launch, bit for bit"""
    L.exact("rows", r, ref_cond_rows(s["lat_rows"], s["mask"]))
    L.own(r)
    L.sig.update(N=r.shape[0], H=s["mask"].shape[0], W=s["mask"].shape[1], dtype=str(r.dtype)[6:])
