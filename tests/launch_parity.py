"""Launch census: every kernel launch of a model run, checked against the fp32 reference of that one launch.

Inside `census()` every public function of diffusionkit_b200.ops that launches a kernel is replaced by a wrapper
(the library modules call `ops.X(...)` by attribute lookup, so a model run goes through it).  For each launch the
wrapper snapshots the inputs (clones, so in-place outputs cannot change them) and the whole underlying buffer of every
tensor the launch may write, runs the real op, synchronises, and then

  * compares the output with that op's one reference in tests/kernel_checks.py (ref_*), by global rel-L2 with the op's
    table-check tolerance and by the 128 x 128 block map with the full-size block bounds (a block of near-zero
    reference values is judged by its absolute error at the tensor's scale), or bit for bit where the op is exact;
  * checks that every element of those buffers outside what the launch owns is bit-identical to its snapshot (the
    joint-sequence scatter, the `cat` column windows, the o_txt / o_img splits, the skip-layer cuts);
  * records one row per launch: op, shape / layout signature, rel-L2, worst block.

A failing launch raises with its call index, op, signature and run name, and its inputs go to $DK_DUMP_DIR.  FP8 GEMMs
are checked once, in the `gemm` wrapper (ops.gemm_fp8 calls the module-global gemm, which the census rebinds).  Only
eager runs can be checked: the wrapper refuses to run while the stream is capturing a CUDA graph.
"""
from __future__ import annotations

import contextlib
import inspect
import math
import re
from collections import defaultdict
from typing import Callable, Dict, List

import torch

from diffusionkit_b200 import ops

_LAUNCH_SRC = re.compile(r"\.call\(|\.lib\.dk_")


def launching_ops() -> List[str]:
    """names of the ops functions that reach a dk_* entry point themselves (c.call(...) / c.lib.dk_*(...))"""
    out = []
    for name, fn in vars(ops).items():
        if inspect.isfunction(fn) and fn.__module__ == ops.__name__ and not name.startswith("_"):
            if _LAUNCH_SRC.search(inspect.getsource(fn)):
                out.append(name)
    return sorted(out)


# Ops no census run reaches, with the reason; every other launching op must be checked at least once.
NOT_REACHED = {
    "dequant_q4": "only loading a 4-bit checkpoint dequantises; the census runs on synthetic 16-bit weights",
    "vae_sample_latent": "only img2img samples the posterior; no census run encodes an image into a latent",
    "axpby": "only img2img mixes the noise with the encoded latent; no census run starts from an image",
    "qk_norm_rope": "the models fuse QK-norm and RoPE into the QKV GEMM epilogue; the unfused kernel has no caller",
    "act": "no model path applies a standalone activation; the GEMM epilogues fuse them",
}

# per-op bounds: global rel-L2 of 16-bit outputs (kernel_checks), attention, the fused QK path, and the block maps of
# the full-size checks
TOL16, TOL_ATT, TOL_ATT_SMALL, TOL_QK, TOL_F32 = 4e-3, 1e-2, 6e-3, 6e-3, 1e-5
BLK16, BLK_ATT, BLK_QK = 1.2e-2, 3e-2, 1.5e-2
BLOCK_FLOOR = 0.05

_INT = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def _kc():
    from tests import kernel_checks

    return kernel_checks


def _storage_words(t: torch.Tensor) -> torch.Tensor:
    """t's whole underlying buffer as a flat integer tensor of t's element size (for bit comparisons)"""
    st = t.untyped_storage()
    isz = t.element_size()
    w = torch.empty(0, dtype=_INT[isz], device=t.device)
    return w.set_(st, 0, (st.nbytes() // isz,), (1,))


def _clone(v):
    if torch.is_tensor(v):
        return v.clone()
    if isinstance(v, tuple):
        return tuple(_clone(x) for x in v)
    return v


class _Launch:
    """what the check of one launch collects: comparisons, owned output elements, signature"""

    def __init__(self):
        self.sig: Dict[str, object] = {}
        self.owned: List[tuple] = []
        self.err = 0.0
        self.worst = 0.0

    def own(self, view: torch.Tensor, idx=None):
        self.owned.append((view, idx))

    def close(self, what, got, ref, tol, block_tol=None, bc=128):
        kc = _kc()
        got2 = got.reshape(-1, got.shape[-1]) if got.dim() > 1 else got.reshape(1, -1)
        ref2 = ref.reshape(-1, ref.shape[-1]) if ref.dim() > 1 else ref.reshape(1, -1)
        if block_tol is None:
            err, worst = kc._assert_close(what, got2, ref2, tol), 0.0
        else:
            r = kc._assert_close_blocks(what, got2, ref2, tol, block_tol, bc=min(bc, got2.shape[-1]),
                                        floor=BLOCK_FLOOR)
            err, worst = r["rel_l2"], r["worst_block"]
        self.err, self.worst = max(self.err, err), max(self.worst, worst)

    def exact(self, what, got, ref):
        """bit for bit, except that a NaN matches a NaN (a bit copy of fp32 rows viewed as 16-bit words holds NaN
        patterns)"""
        same = got.shape == ref.shape and got.dtype == ref.dtype
        if same and not torch.equal(got, ref):
            diff = got != ref
            if got.is_floating_point():
                diff &= ~(torch.isnan(got) & torch.isnan(ref))
            same = not bool(diff.any())
        if not same:
            n = int(diff.sum()) if got.shape == ref.shape and got.dtype == ref.dtype else -1
            raise AssertionError(f"{what}: not bit-identical to the reference ({n} elements differ, "
                                 f"{tuple(got.shape)} {got.dtype} vs {tuple(ref.shape)} {ref.dtype})")


# ------------------------------------------------------------------------------------------------ per-op checks
# Each check gets the launch record L, the bound arguments `a` (the caller's tensors), their snapshots `s` (clones taken
# before the launch) and the op's return value.  WRITES lists the arguments the op may write in place.
WRITES = {
    "gemm": ["out"], "quantize_rows_e4m3": ["out", "scale"], "ln_modulate_fp8": ["out", "out_scale"],
    "ln_modulate": ["out"], "qk_norm_rope": ["qkv"], "attention": ["out0", "out1"], "silu_add": ["out"],
    "act": ["out"], "patchify": ["out"], "unpatchify": ["out"], "copy_rows": ["dst"], "sampler_prepare": ["xin"],
    "sampler_step": ["x"], "sampler_heun_predict": ["x", "d", "x2"], "sampler_heun_correct": ["x", "d", "x2"],
    "sampler_dpmpp_2m": ["x", "d_prev"], "axpb": ["out"], "embedding": ["out"], "layernorm": ["out"],
    "rmsnorm_f32": ["out"], "add_f32_16": ["x"], "glu_gelu": ["out"], "attention_small": ["out"],
    "dequant_q4": ["out"], "axpby": ["out"], "vae_sample_latent": ["out"], "cast_to_16": ["out"],
    "cast_to_f32": ["out"], "residual_delta": ["r_out", "sums", "ws"], "residual_apply": ["out"],
    "groupnorm_stats": ["ws"], "groupnorm_apply": ["out"], "conv3x3": ["out"], "conv3x3_s2": ["out"],
    "conv3x3_fused": ["out", "out_partial"], "groupnorm_finalize": ["stats"], "upsample_nearest2x": ["out"],
    "softmax_rows": ["x"],
}


def _c_gemm(L, a, s, r, census):
    kc = _kc()
    A, W = s["A"], s["W"]
    M, K = A.shape
    fp8 = a["fp8_scales"] is not None
    n = a["N"] if a["N"] is not None else (W.shape[1] if a["w_n_major"] else W.shape[0])
    rpb = a["rows_per_batch"]
    if fp8:
        a_s, w_s = s["fp8_scales"]
        A, W = A.float() * a_s[:, None], W.float() * w_s[:W.shape[0], None]
    gate = s["gate"]
    if gate is not None and not rpb:
        gate = gate[:1]                                  # one batch of all M rows: gate row 0
    y = kc.ref_gemm(A, W, s["bias"], a["act"], gate, s["res"], rows_per_batch=rpb, res_batch_rows=a["res_batch_rows"],
                    res_row_off=a["res_row_off"], N=n, w_n_major=a["w_n_major"])
    qk = a["qk"]
    if qk is not None:
        heads, hd, qw, kw, rope, eps = s["qk"]
        pos = a["out_row_off"] + torch.arange(M, device=y.device) % (rpb or M)
        y = kc.ref_qk_norm_rope(y, pos, heads, hd, qw, kw, rope, eps=eps)
    rows = kc.gemm_out_rows(M, rpb, a["out_batch_rows"], a["out_row_off"], device=r.device)
    L.close("out", r[rows, :n], y, TOL_QK if qk is not None else TOL16, BLK_QK if qk is not None else BLK16)
    L.own(r, (rows, slice(0, n)))
    terms = [t for t, on in (("fp8", fp8), ("bias", a["bias"] is not None), (f"act{a['act']}", a["act"]),
                             ("gate", a["gate"] is not None), ("res", a["res"] is not None),
                             ("inplace", a["res"] is not None and a["out"] is not None
                              and a["res"].data_ptr() == a["out"].data_ptr()),
                             ("remap", rpb and (a["out_batch_rows"] != rpb or a["out_row_off"])),
                             ("n_major", a["w_n_major"]), ("qk", qk is not None)) if on]
    L.sig.update(M=M, N=n, K=K, n256=n % 256, epi="+".join(terms) or "plain", ldc=r.stride(0),
                 gate_ld=a["gate"].stride(0) if a["gate"] is not None else None,
                 res_batch_rows=(a["res_batch_rows"] if a["res_batch_rows"] is not None else rpb)
                 if a["res"] is not None and rpb else None, dtype=str(r.dtype)[6:])
    if qk is not None:
        L.sig["qk_heads"], L.sig["qk_hd"] = qk[0], qk[1]


def _c_quantize_rows_e4m3(L, a, s, r, census):
    from tests.fp8_ref import quantize_rows_e4m3

    q, sc = r
    want_q, want_s = quantize_rows_e4m3(s["x"].cpu())
    L.exact("scale", sc.cpu(), want_s)
    L.exact("q", q.float().cpu(), want_q)
    L.own(q)
    L.own(sc)


def _c_ln_modulate_fp8(L, a, s, r, census):
    ref = _kc().ref_ln_modulate(s["x"], s["shift"], s["scale"], a["rows_per_batch"], a["eps"])
    q, sc = r
    want_s = ref.abs().amax(dim=1) / 448.0
    e = float(((sc - want_s).abs() / want_s).max())
    if not e <= 1e-5:
        raise AssertionError(f"row scales: max relative error {e:.3e} (tol 1e-5)")
    # half an e4m3 ulp of each element times the row's scale, plus the slack of another fp32 LayerNorm order
    y = ref / sc[:, None]
    ulp = torch.floor(torch.log2(y.abs().clamp(2.0 ** -6, 448.0))).exp2() * 2.0 ** -3
    over = ((q.float() * sc[:, None] - ref).abs() / ((0.5 * ulp + 1e-4 * y.abs() + 1e-4) * sc[:, None])).max()
    if not float(over) <= 1.0:
        raise AssertionError(f"e4m3 values: error {float(over):.3f} x the half-ulp bound")
    L.err = e
    L.own(q)
    L.own(sc)


def _c_ln_modulate(L, a, s, r, census):
    ref = _kc().ref_ln_modulate(s["x"], s["shift"], s["scale"], a["rows_per_batch"], a["eps"])
    L.close("out", r, ref, TOL16, BLK16)
    L.own(r)
    L.sig.update(h=r.shape[1], mod_ld=a["shift"].stride(0))


def _c_qk_norm_rope(L, a, s, r, census):
    kc = _kc()
    qkv, S, split, hd = s["qkv"], a["S"], a["split"], a["d"]
    pos = torch.arange(qkv.shape[0], device=qkv.device) % S
    first = (pos < split)[:, None, None]

    def pick(w1, w2):
        return None if w1 is None else torch.where(first, w1.float(), w2.float())

    ref = kc.ref_qk_norm_rope(qkv, pos, a["heads"], hd, pick(s["q_w"], s["q_w2"]), pick(s["k_w"], s["k_w2"]),
                              s["rope"], round_to=qkv.dtype, eps=a["eps"])
    h2 = 2 * a["heads"] * hd
    L.close("qk", r[:, :h2], ref[:, :h2], TOL16, BLK16)
    L.own(r, (slice(None), slice(0, h2)))


def _c_attention(L, a, s, r, census):
    B, S, heads, hd = a["B"], a["S"], a["heads"], a["d"]
    split = S if a["split"] is None else a["split"]
    h = heads * hd
    scale = a["scale"] if a["scale"] is not None else 1.0 / math.sqrt(hd)
    if abs(scale - 1.0 / math.sqrt(hd)) > 1e-7:
        raise AssertionError("attention: ref_attention covers the 1/sqrt(d) scale only")
    ref = _kc().ref_attention(s["qkv"], B, S, heads, hd).reshape(B, S, h)
    o0, o1 = a["out0"], a["out1"]
    L.close("out0", o0[:B * split, :h], ref[:, :split].reshape(-1, h), TOL_ATT, BLK_ATT, bc=hd)
    L.own(o0, (slice(0, B * split), slice(0, h)))
    if split < S:
        L.close("out1", o1[:B * (S - split), :h], ref[:, split:].reshape(-1, h), TOL_ATT, BLK_ATT, bc=hd)
        L.own(o1, (slice(0, B * (S - split)), slice(0, h)))
    L.sig.update(B=B, S=S, heads=heads, d=hd, split=split, ld0=o0.stride(0),
                 ld1=o1.stride(0) if o1 is not None else None, dtype=str(o0.dtype)[6:])


def _c_silu_add(L, a, s, r, census):
    L.close("out", r, _kc().ref_silu_add(s["y"], s["temb"]), TOL16)
    L.own(r)


def _c_act(L, a, s, r, census):
    L.close("out", r, _kc().ref_act(s["x"], a["kind"]), TOL16)
    L.own(r)


def _c_patchify(L, a, s, r, census):
    L.exact("rows", r, _kc().ref_patchify(s["latent"], a["order"]))
    L.own(r)


def _c_unpatchify(L, a, s, r, census):
    L.exact("latent", r, _kc().ref_unpatchify(s["rows"], a["B"], a["H"], a["W"], a["Cc"], a["order"]))
    L.own(r)


def _c_pos_embed_crop(L, a, s, r, census):
    L.exact("pos", r, _kc().ref_pos_embed_crop(s["table"], a["max_hw"], a["hp"], a["wp"]))


def _c_copy_rows(L, a, s, r, census):
    B, rows, h = a["B"], a["rows"], a["h"]
    src, dst = s["src"].reshape(-1, h), r.view(-1).view(-1, h)
    i = torch.arange(B * rows, device=r.device)
    di = (i // rows) * a["dst_rows"] + a["dst_off"] + i % rows
    si = (i // rows) * a["src_rows"] + a["src_off"] + i % rows
    L.exact("rows", dst[di], src[si])
    L.own(dst, (di, slice(None)))
    L.sig.update(B=B, rows=rows, h=h, dst=(a["dst_rows"], a["dst_off"]), src=(a["src_rows"], a["src_off"]))


def _c_sampler_prepare(L, a, s, r, census):
    x, n = s["x"], s["x"].numel()
    want = x.reshape(-1).to(r.dtype).repeat(a["reps"])
    L.exact("xin", r.reshape(-1)[:a["reps"] * n], want)
    L.own(r.view(-1), slice(0, a["reps"] * n))


def _c_sampler_step(L, a, s, r, census):
    ref = _kc().ref_sampler_step(s["x"], s["xin"], s["out"], a["sigma"], a["sigma_next"], a["cfg_weight"], a["slg"])
    L.close("x", r, ref, TOL_F32)
    L.own(r)
    L.sig.update(cfg=a["cfg_weight"] > 0, slg=a["slg"] != 0.0)


def _c_sampler_heun_predict(L, a, s, r, census):
    d_ref, x2_ref = _kc().ref_heun_predict(s["x"], s["xin"], s["out"], a["sigma"], a["sigma_next"], a["cfg_weight"],
                                           a["slg"])
    d, x2 = r
    L.close("d", d, d_ref, TOL_F32)
    L.close("x2", x2, x2_ref, TOL_F32)
    L.own(d)
    L.own(x2)
    L.sig.update(cfg=a["cfg_weight"] > 0, slg=a["slg"] != 0.0)


def _c_sampler_heun_correct(L, a, s, r, census):
    ref = _kc().ref_heun_correct(s["x"], s["d"], s["x2"], s["xin"], s["out"], a["sigma"], a["sigma_next"],
                                 a["cfg_weight"], a["slg"])
    L.close("x", r, ref, TOL_F32)
    L.own(r)
    L.sig.update(cfg=a["cfg_weight"] > 0, slg=a["slg"] != 0.0)


def _c_sampler_dpmpp_2m(L, a, s, r, census):
    x_ref, d_ref = _kc().ref_dpmpp_2m(s["x"], s["d_prev"], s["xin"], s["out"], a["sigma"], a["a"], a["b"], a["c"],
                                      a["cfg_weight"], a["slg"])
    L.close("x", r, x_ref, TOL_F32)
    L.close("d_prev", a["d_prev"], d_ref, TOL_F32)
    L.own(r)
    L.own(a["d_prev"])
    L.sig.update(cfg=a["cfg_weight"] > 0, slg=a["slg"] != 0.0, second_order=a["c"] != 0.0)


def _c_axpb(L, a, s, r, census):
    L.close("out", r, s["x"] * a["a"] + a["b"], TOL_F32)
    L.own(r)


def _c_axpby(L, a, s, r, census):
    L.close("out", r, a["a"] * s["x"] + a["b"] * s["y"], TOL_F32)
    L.own(r)


def _c_embedding(L, a, s, r, census):
    L.exact("rows", r, _kc().ref_embedding(s["table"], s["ids"], s["pos"]))
    L.own(r)


def _c_layernorm(L, a, s, r, census):
    L.close("out", r, _kc().ref_layernorm(s["x"], s["weight"], s["bias"], a["eps"]), TOL16, BLK16)
    L.own(r)


def _c_rmsnorm_f32(L, a, s, r, census):
    L.close("out", r, _kc().ref_rmsnorm_f32(s["x"], s["weight"], a["eps"]), TOL16, BLK16)
    L.own(r)


def _c_add_f32_16(L, a, s, r, census):
    L.exact("x", r, s["x"] + s["y"].reshape(s["x"].shape).float())
    L.own(r)


def _c_glu_gelu(L, a, s, r, census):
    L.close("out", r, _kc().ref_glu_gelu(s["h"]), TOL16, BLK16)
    L.own(r)


def _c_attention_small(L, a, s, r, census):
    ref = _kc().ref_attention_small(s["qkv"], a["B"], a["S"], a["heads"], a["scale"], s["rel_bias"], a["causal"])
    L.close("out", r, ref, TOL_ATT_SMALL, BLK_ATT, bc=64)
    L.own(r)
    L.sig.update(B=a["B"], S=a["S"], heads=a["heads"], rel_bias=a["rel_bias"] is not None, causal=a["causal"])


def _c_dequant_q4(L, a, s, r, census):
    import numpy as np

    from oracle import quant_ref as qr

    wq = s["wq"].cpu().numpy().view(np.uint32)
    want = qr.dequantize_q4(wq, s["scales"].float().cpu().numpy(), s["biases"].float().cpu().numpy(), a["group_size"])
    L.exact("w", r.cpu(), torch.from_numpy(want).to(r.dtype))
    L.own(r)


def _c_image_pre(L, a, s, r, census):
    L.exact("x16", r, _kc().ref_image_pre(s["img_u8"], a["dtype"], a["cpad"]))


def _c_vae_sample_latent(L, a, s, r, census):
    L.close("z", r, _kc().ref_vae_sample_latent(s["hidden"], s["noise"], a["shift"], a["scale"]), TOL_F32)
    L.own(r)


def _c_cast_to_16(L, a, s, r, census):
    L.exact("out", r, s["x"].to(a["dtype"]))
    L.own(r)


def _c_cast_to_f32(L, a, s, r, census):
    L.exact("out", r, s["x"].float())
    L.own(r)


def _c_residual_delta(L, a, s, r, census):
    kc = _kc()
    nseq, rows, x = a["nseq"], a["rows"], s["x"]
    x_seq = rows if a["x_seq_rows"] is None else a["x_seq_rows"]
    b_seq = rows if a["b_seq_rows"] is None else a["b_seq_rows"]
    want_r, want = kc.ref_residual_delta(x, s["base"], nseq, rows, x_seq, b_seq, s["prev"])
    if a["r_out"] is not None:
        L.exact("r", a["r_out"].reshape(want_r.shape), want_r)
        L.own(a["r_out"])
    if want is not None:
        e = float(((r.reshape(-1)[:2 * nseq].reshape(nseq, 2).double() - want) / want.clamp(min=1e-30)).abs().max())
        if not e <= 1e-5:
            raise AssertionError(f"sums: max relative error {e:.3e} vs float64 (tol 1e-5)")
        L.err = e
        L.own(r.view(-1), slice(0, 2 * nseq))
        if a["ws"] is not None:
            L.own(a["ws"])
    L.sig.update(nseq=nseq, rows=rows, h=x.shape[1], x_seq=x_seq, ldx=a["x"].stride(0), prev=want is not None)


def _c_residual_apply(L, a, s, r, census):
    L.exact("out", r, (s["x"].float() + s["r"].reshape(s["x"].shape)).to(s["x"].dtype))
    L.own(r)


def _c_groupnorm_stats(L, a, s, r, census):
    mean, rstd = _kc().ref_groupnorm_stats(s["x"], a["G"], a["eps"])
    L.close("mean", r[..., 0], mean, 1e-4)
    L.close("rstd", r[..., 1], rstd, 1e-4)
    if a["ws"] is not None:
        L.own(a["ws"])


def _c_groupnorm_apply(L, a, s, r, census):
    ref = _kc().ref_groupnorm_apply(s["x"], s["stats"], s["gamma"], s["beta"], a["G"], a["silu"])
    L.close("out", r, ref, TOL16, BLK16)
    L.own(r)


def _c_conv3x3(L, a, s, r, census):
    ref = _kc().ref_conv3x3(s["x"], s["w"], s["bias"], s["res"])
    L.close("out", r, ref, TOL16, BLK16)
    L.own(r)


def _c_conv3x3_s2(L, a, s, r, census):
    L.close("out", r, _kc().ref_conv3x3_s2(s["x"], s["w"], s["bias"]), TOL16, BLK16)
    L.own(r)


def _c_conv_up_weights(L, a, s, r, census):
    L.exact("wp", r, _kc().ref_conv_up_weights(s["w"]))
    census.up_source[r.data_ptr()] = s["w"]


def _c_conv3x3_fused(L, a, s, r, census):
    kc = _kc()
    x, up, gn = s["x"], a["up"], s["gn"]
    w = s["w"]
    if up:
        w = census.up_source.get(a["w"].data_ptr())
        if w is None:
            raise AssertionError("phase weights that no checked conv_up_weights launch produced")
    xin = x
    if gn is not None:
        stats, gamma, beta, G = gn
        xin = kc.ref_groupnorm_apply(x, stats, gamma, beta, G, a["silu"]).to(x.dtype)
    if up:
        xin = xin.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    ref = kc.ref_conv3x3(xin, w, s["bias"], s["res"])
    tol = 6e-3 if (gn is not None or up) else TOL16
    L.close("out", r, ref, tol, BLK16)
    L.own(r)
    part = a["out_partial"]
    if part is not None:
        B, Ho, Wo, _ = r.shape
        slots = Ho * Wo // 128
        got = part.reshape(-1)[:B * slots * a["out_G"] * 2].reshape(B, slots, a["out_G"], 2)
        L.close("partial", got, kc.ref_conv_partial_stats(r, a["out_G"], up), 1e-5)
        L.own(part.view(-1), slice(0, got.numel()))
    L.sig.update(shape=tuple(x.shape), Cout=r.shape[-1], norm=gn is not None, up=up, res=a["res"] is not None,
                 stats=part is not None)


def _c_groupnorm_finalize(L, a, s, r, census):
    ref = _kc().ref_groupnorm_finalize(s["partial"].reshape(a["B"], a["slots"], a["G"], 2), a["count"], a["eps"])
    L.close("stats", r, ref, 1e-4)
    L.own(r)


def _c_upsample_nearest2x(L, a, s, r, census):
    L.exact("out", r, s["x"].repeat_interleave(2, dim=1).repeat_interleave(2, dim=2))
    L.own(r)


def _c_softmax_rows(L, a, s, r, census):
    L.close("p", r, _kc().ref_softmax_rows(s["x"], a["scale"]), TOL16, BLK16)
    L.own(r)
    L.sig.update(rows=r.shape[0], cols=r.shape[1], ld=r.stride(0))


def _c_image_post(L, a, s, r, census):
    v, v8 = _kc().ref_image_post(s["x"])
    L.exact("float", r[0], v)
    if r[1] is not None:
        L.exact("uint8", r[1], v8)


CHECKS: Dict[str, Callable] = {name[3:]: fn for name, fn in list(globals().items()) if name.startswith("_c_")}


# ------------------------------------------------------------------------------------------------ the census
class Census:
    def __init__(self):
        self.run = ""
        self.index = 0
        self.records: List[dict] = []
        self.up_source: Dict[int, torch.Tensor] = {}

    def rows(self):
        """one row per (op, signature): count, worst rel-L2, worst block, runs"""
        agg = defaultdict(lambda: {"count": 0, "rel_l2": 0.0, "worst_block": 0.0, "runs": set()})
        for rec in self.records:
            a = agg[(rec["op"], rec["sig"])]
            a["count"] += 1
            a["rel_l2"] = max(a["rel_l2"], rec["rel_l2"])
            a["worst_block"] = max(a["worst_block"], rec["worst_block"])
            a["runs"].add(rec["run"])
        return [dict(op=op, sig=sig, **v) for (op, sig), v in sorted(agg.items())]

    def table(self) -> str:
        lines = [f"{'op':<22} {'n':>4} {'rel_l2':>9} {'block':>9}  signature  [runs]"]
        for r in self.rows():
            lines.append(f"{r['op']:<22} {r['count']:>4} {r['rel_l2']:>9.2e} {r['worst_block']:>9.2e}  {r['sig']}  "
                         f"[{','.join(sorted(r['runs']))}]")
        return "\n".join(lines)

    def _wrap(self, name: str, fn: Callable) -> Callable:
        sig = inspect.signature(fn)
        check = CHECKS[name]

        def wrapper(*args, **kwargs):
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError(f"launch census: ops.{name} reached while a CUDA graph is being captured; captured "
                                   "kernels do not run at capture time (set use_cuda_graphs = False)")
            bound = sig.bind(*args, **kwargs)
            bound.apply_defaults()
            a = dict(bound.arguments)
            torch.cuda.synchronize()
            s = {k: _clone(v) for k, v in a.items()}
            bufs = {}
            for k in WRITES.get(name, []):
                t = a.get(k)
                if torch.is_tensor(t) and t.untyped_storage().data_ptr() not in bufs:
                    w = _storage_words(t)
                    bufs[t.untyped_storage().data_ptr()] = (t, w, w.clone())
            result = fn(*args, **kwargs)
            torch.cuda.synchronize()
            self.index += 1
            L = _Launch()
            try:
                check(L, a, s, result, self)
                self._untouched(L, bufs)
            except AssertionError as e:
                label = f"launch #{self.index} ops.{name} [{self._sig(L, a)}] in run '{self.run}'"
                _kc()._dump(f"launch{self.index}_{name}",
                            **{k: v for k, v in s.items() if torch.is_tensor(v) and v.dtype != torch.bool})
                raise AssertionError(f"{label}: {e}") from None
            self.records.append({"op": name, "sig": self._sig(L, a), "info": dict(L.sig), "run": self.run,
                                 "rel_l2": L.err, "worst_block": L.worst, "index": self.index})
            return result

        wrapper.__wrapped__ = fn
        return wrapper

    @staticmethod
    def _sig(L, a) -> str:
        if not L.sig or "dtype" not in L.sig:
            shapes = [f"{k}={tuple(v.shape)}" for k, v in a.items() if torch.is_tensor(v)]
            dt = next((str(v.dtype)[6:] for v in a.values() if torch.is_tensor(v)), "")
            extra = [f"{k}={v}" for k, v in L.sig.items()]
            return " ".join(shapes + extra + [dt])
        return " ".join(f"{k}={v}" for k, v in L.sig.items() if v is not None)

    @staticmethod
    def _untouched(L, bufs):
        """every element of a written buffer that the launch does not own is bit-identical to its snapshot"""
        for t, words, before in bufs.values():
            mask = torch.zeros(words.shape, dtype=torch.bool, device=words.device)
            sp = t.untyped_storage().data_ptr()
            for view, idx in L.owned:
                if view.untyped_storage().data_ptr() != sp or view.element_size() != t.element_size():
                    continue
                mv = mask.as_strided(view.shape, view.stride(), view.storage_offset())
                if idx is None:
                    mv.fill_(True)
                else:
                    mv[idx] = True
            changed = (words != before) & ~mask
            if bool(changed.any()):
                first = int(changed.nonzero()[0, 0])
                raise AssertionError(f"{int(changed.sum())} elements outside the launch's output changed (first at "
                                     f"element {first} of a buffer of {words.numel()})")


@contextlib.contextmanager
def census(c: Census = None):
    """patch every launching op of diffusionkit_b200.ops with the checking wrapper for the duration"""
    c = c if c is not None else Census()
    names = launching_ops()
    missing = [n for n in names if n not in CHECKS]
    if missing:
        raise RuntimeError(f"launch census: no reference check for {missing}")
    saved = {n: getattr(ops, n) for n in names}
    try:
        for n in names:
            setattr(ops, n, c._wrap(n, saved[n]))
        yield c
    finally:
        for n, fn in saved.items():
            setattr(ops, n, fn)
