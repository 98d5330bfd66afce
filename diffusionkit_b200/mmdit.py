"""MMDiT (SD3 dual-stream / FLUX dual + single-stream) forward on H100.

Host-side mirror of the reference module (python/src/diffusionkit/mlx/mmdit.py:22-266): same public methods
(`cache_modulation_params`, `__call__(latent_image_embeddings, token_level_text_embeddings, timestep)`,
`clear_modulation_params_cache`), same parameter names.  Every FLOP runs in hand-written sm_90a kernels reached
through the C ABI (ops.py -> libdkb200.so); torch tensors are only the HBM containers.

H100 layout decisions (vs. the reference's per-module MLX graph):
  * q/k/v projections of a stream are ONE GEMM (packed [3h, h] weight; k has no bias — quirk Q3) whose epilogue applies
    the per-head QK-RMSNorm and RoPE (FLUX) and scatters rows straight into the joint [text|image] (FLUX) /
    [image|text] (SD3) sequence buffer — no norm / rope / concat kernels.
  * adaLN gate * (.) + residual is fused into the o_proj / fc2 GEMM epilogues (in place on the residual stream);
    bias + exact-erf GELU into fc1's.
  * FLUX single-stream blocks: attention output and GELU(fc1) land in one [B*S, 5h] buffer and
    o_proj + fc2 run as ONE K=5h GEMM with the packed [Wo | W2] weight (upstream `linear2`, mlx/model_io.py:253-259).
  * all adaLN modulations for all timesteps and all blocks are ONE batched GEMM (replaces the reference's
    per-timestep, per-block loop, mmdit.py:91-175); a step selects its rows with one small D2D copy, which keeps the
    forward's launch sequence timestep-invariant (CUDA-graph capturable).
  * opt-in FP8 (`set_fp8`, DESIGN.md "FP8 linears"): the block linears run on row-scaled e4m3 copies of their weights;
    their inputs are quantised per token by the LayerNorm-modulate kernel or by a row quantiser.
  * opt-in first-block step cache (`set_step_cache`, DESIGN.md §10): a forward whose first-block residual
    barely changed since the last full one skips the other blocks and reuses their residual.
  * FLUX.1-dev's guidance embedder (`config.guidance_embed`, DESIGN.md §12) joins the conditioning vector inside
    cache_modulation_params; the per-step forward does not change.
  * SD3.5 Medium's MMDiT-X blocks (`config.x_block_self_attn_layers`, DESIGN.md §13): the image stream's second
    self-attention is one more packed stream (attn2) run by the same kernels, and a forward can skip listed blocks
    for its trailing sequences (skip-layer guidance).
  * FLUX.1 Kontext editing (`reference=` of __call__, DESIGN.md §14): a reference latent's tokens follow the target's
    in the image stream at RoPE positions (1, r, c); every block runs unchanged on the longer stream and the final
    layer reads the target rows.
  * FLUX.1 Fill (`config.x_embedder_cond_channels`, DESIGN.md §18): the x-embedder's conditioning columns run once per
    call (cache_fill_conditioning); every forward adds their product to the latent columns' through the x-embedder
    GEMM's broadcast residual, so the per-step launches are FLUX.1-dev's.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch

from . import ops
from ._lib import ACT_GELU_ERF, ACT_NONE, ACT_SILU, DkError
from .config import MMDiTConfig, PositionalEncoding
from .graphs import ShapeCache, default_settings
from .step_cache import StepCachePolicy


def fp8_covered_linears(config: MMDiTConfig) -> List[str]:
    """Reference names of the linears `MMDiT.set_fp8` moves to e4m3: q/k/v, o, fc1 and fc2 of every transformer block
    stream that has them.  Embedders, adaLN modulation and the final layer stay 16-bit."""
    c = config
    names = []

    def block(prefix, skip_post=False):
        names.extend(f"{prefix}.attn.{n}_proj" for n in "qkv")
        if not skip_post:
            names.extend(f"{prefix}.{n}" for n in ("attn.o_proj", "mlp.fc1", "mlp.fc2"))

    for i in range(c.depth_multimodal):
        block(f"multimodal_transformer_blocks.{i}.image_transformer_block")
        block(f"multimodal_transformer_blocks.{i}.text_transformer_block",
              skip_post=(i == c.depth_multimodal - 1) and (c.depth_unified < 1))
    for i in sorted(c.x_block_self_attn_layers):
        names.extend(f"multimodal_transformer_blocks.{i}.image_transformer_block.attn2.{n}_proj" for n in "qkvo")
    for i in range(c.depth_unified):
        block(f"unified_transformer_blocks.{i}.transformer_block")
    return names


def check_x_layers(config: MMDiTConfig):
    """Raise ValueError for MMDiT-X layers (x_block_self_attn_layers) the engine does not run: on a FLUX-shaped config,
    out of range or listed twice, or without QK-RMSNorm (no published model has that form)."""
    c, xl = config, tuple(config.x_block_self_attn_layers)
    if not xl:
        return
    if c.depth_unified > 0:
        raise ValueError("MMDiT: x_block_self_attn_layers (MMDiT-X) needs an SD3-shaped config (depth_unified == 0)")
    if len(set(xl)) != len(xl) or not all(isinstance(i, int) and 0 <= i < c.depth_multimodal for i in xl):
        raise ValueError(f"MMDiT: x_block_self_attn_layers {xl} must be distinct block indices in "
                         f"[0, {c.depth_multimodal})")
    if not c.use_qk_norm:
        raise ValueError("MMDiT: x_block_self_attn_layers (MMDiT-X) needs use_qk_norm=True")


class _Stream:
    """Packed weights of one TransformerBlock (reference mmdit.py:395-548)."""

    __slots__ = ("name", "n_mod", "mod_off", "w_qkv", "b_qkv", "w_o", "b_o", "w_fc1", "b_fc1", "w_fc2", "b_fc2",
                 "w_out", "q_norm", "k_norm", "skip_post")


class MMDiT:
    def __init__(self, config: MMDiTConfig, params: Dict[str, torch.Tensor], device=None):
        self.config = config
        c = config
        if c.guidance_embed and c.depth_unified == 0:
            raise ValueError("MMDiT: guidance_embed (FLUX.1-dev's guidance embedder) needs a FLUX-shaped config "
                             "(depth_unified > 0)")
        check_x_layers(c)
        any_p = next(iter(params.values()))
        self.device = torch.device(device) if device is not None else any_p.device
        if self.device.type != "cuda":
            raise DkError("MMDiT: parameters must live on a CUDA device (no CPU fallback)")
        self.dtype = any_p.dtype
        if self.dtype not in (torch.bfloat16, torch.float16):
            raise DkError(f"MMDiT: weights must be bf16 or fp16 (w16), got {self.dtype}")
        if c.pos_embed_type not in (PositionalEncoding.LearnedInputEmbedding, PositionalEncoding.PreSDPARope):
            raise ValueError(f"Unsupported positional encoding type: {c.pos_embed_type}")  # mmdit.py:50-52
        self.h = c.hidden_size
        self.heads = c.num_heads
        self.d = c.head_dim
        if self.d not in (64, 128):
            raise DkError(f"MMDiT: head dim {self.d} unsupported by the attention kernel (64 or 128)")
        self.is_flux = c.depth_unified > 0
        self.cond_channels = int(c.x_embedder_cond_channels)
        if self.cond_channels and not (self.is_flux and c.patchify_via_reshape):
            raise ValueError("MMDiT: x_embedder_cond_channels (FLUX.1 Fill) needs a FLUX-shaped config")
        if self.cond_channels % 8:
            raise ValueError(f"MMDiT: x_embedder_cond_channels must be a multiple of 8, got {self.cond_channels}")
        self._pack(params)
        self._mod_index: Dict[float, int] = {}
        self._mod_all: Optional[torch.Tensor] = None
        self._mod_cur: Optional[torch.Tensor] = None
        self._mod_batch = 0
        self._mod_skip_batch = 0
        # workspace, RoPE table and cropped positional embedding live per input shape, next to the CUDA graph of the
        # (timestep-invariant) forward that bakes in their pointers
        self._shapes = ShapeCache()
        self.use_cuda_graphs, self.max_cached_shapes = default_settings()
        # packed tensors a LoRA merge has touched: (id(owner), attribute, tuple index) -> (owner, base, live)
        self._lora_live: Dict[Tuple[int, str, Optional[int]], Tuple[object, torch.Tensor, torch.Tensor]] = {}
        # set_fp8: (id(stream), packed weight attribute) -> (e4m3 copy [N, K], fp32 row scales [N])
        self._fp8_w: Dict[Tuple[int, str], Tuple[torch.Tensor, torch.Tensor]] = {}
        self._fp8 = False
        # set_step_cache: the skip policy (None: off) and the input shape its residuals belong to
        self._step_cache: Optional[StepCachePolicy] = None
        self._step_cache_key = None
        # FLUX.1 Fill: (rows, h) conditioning term of the x-embedder, written once per call by cache_fill_conditioning
        # at a fixed address (captured graphs read it); _fill_rows = its valid rows, 0 until computed or after a LoRA
        # merge changed the x-embedder
        self._fill_cond: Optional[torch.Tensor] = None
        self._fill_rows = 0

    # ------------------------------------------------------------------------------------------ weight packing
    def _pack(self, P: Dict[str, torch.Tensor]):
        c, h = self.config, self.h
        dev, dt = self.device, self.dtype

        def get(name):
            t = P[name]
            if t.device != dev or t.dtype != dt:
                t = t.to(device=dev, dtype=dt)
            return t.contiguous()

        # (h, 64 + cond_channels): the latent columns, then FLUX.1 Fill's conditioning columns
        self.w_x = get("x_embedder.proj.weight").reshape(h, -1).contiguous()
        self.x_in = self.w_x.shape[1] - self.cond_channels
        self.b_x = get("x_embedder.proj.bias")
        self.pos_table = get("x_pos_embedder.pos_embed.weight") if "x_pos_embedder.pos_embed.weight" in P else None
        self.y0 = (get("y_embedder.mlp.layers.0.weight"), get("y_embedder.mlp.layers.0.bias"))
        self.y2 = (get("y_embedder.mlp.layers.2.weight"), get("y_embedder.mlp.layers.2.bias"))
        self.t0 = (get("t_embedder.mlp.layers.0.weight"), get("t_embedder.mlp.layers.0.bias"))
        self.t2 = (get("t_embedder.mlp.layers.2.weight"), get("t_embedder.mlp.layers.2.bias"))
        self.g0 = self.g2 = None
        if c.guidance_embed:
            self.g0 = (get("guidance_in.mlp.layers.0.weight"), get("guidance_in.mlp.layers.0.bias"))
            self.g2 = (get("guidance_in.mlp.layers.2.weight"), get("guidance_in.mlp.layers.2.bias"))
        self.w_ctx, self.b_ctx = get("context_embedder.weight"), get("context_embedder.bias")
        self.w_final, self.b_final = get("final_layer.linear.weight"), get("final_layer.linear.bias")

        mod_w, mod_b = [], []
        self.mod_total = 0

        def add_mod(prefix) -> int:
            off = self.mod_total
            w = get(prefix + ".adaLN_modulation.layers.1.weight")
            mod_w.append(w)
            mod_b.append(get(prefix + ".adaLN_modulation.layers.1.bias"))
            self.mod_total += w.shape[0]
            return off

        def qkv_bias(attn):
            bq, bv = get(attn + ".q_proj.bias"), get(attn + ".v_proj.bias")
            bk = get(attn + ".k_proj.bias") if c.attn_k_bias else torch.zeros_like(bq)  # no k bias: quirk Q3
            return torch.cat([bq, bk, bv]).contiguous()

        def stream(prefix, n_mod, skip_post=False, parallel=False) -> _Stream:
            s = _Stream()
            s.name, s.n_mod, s.skip_post = prefix, n_mod, skip_post
            s.mod_off = add_mod(prefix)
            wq, wk, wv = get(prefix + ".attn.q_proj.weight"), get(prefix + ".attn.k_proj.weight"), get(
                prefix + ".attn.v_proj.weight")
            s.w_qkv = torch.cat([wq, wk, wv], dim=0).contiguous()
            s.b_qkv = qkv_bias(prefix + ".attn")
            s.w_o = s.b_o = s.w_fc1 = s.b_fc1 = s.w_fc2 = s.b_fc2 = s.w_out = None
            if not skip_post:
                s.b_o = get(prefix + ".attn.o_proj.bias")
                s.w_fc1, s.b_fc1 = get(prefix + ".mlp.fc1.weight"), get(prefix + ".mlp.fc1.bias")
                if parallel:
                    # u += gate * ([attn | gelu(fc1)] @ [Wo | W2]^T + bo); fc2.bias is zeroed (mmdit.py:742)
                    s.w_out = torch.cat([get(prefix + ".attn.o_proj.weight"), get(prefix + ".mlp.fc2.weight")],
                                        dim=1).contiguous()
                else:
                    s.w_o = get(prefix + ".attn.o_proj.weight")
                    s.w_fc2, s.b_fc2 = get(prefix + ".mlp.fc2.weight"), get(prefix + ".mlp.fc2.bias")
            s.q_norm = s.k_norm = None
            if c.use_qk_norm:
                s.q_norm = get(prefix + ".qk_norm.q_norm.weight")
                s.k_norm = get(prefix + ".qk_norm.k_norm.weight")
            return s

        def attn2(img: _Stream) -> _Stream:
            """MMDiT-X: the image stream's second self-attention; its shift, scale and gate are modulation chunks 6-8
            of the image stream"""
            p, s = img.name + ".attn2", _Stream()
            s.name, s.n_mod, s.skip_post, s.mod_off = p, 3, False, img.mod_off + 6 * h
            s.w_qkv = torch.cat([get(f"{p}.{n}_proj.weight") for n in "qkv"], dim=0).contiguous()
            s.b_qkv = qkv_bias(p)
            s.w_o, s.b_o = get(p + ".o_proj.weight"), get(p + ".o_proj.bias")
            s.w_fc1 = s.b_fc1 = s.w_fc2 = s.b_fc2 = s.w_out = None
            s.q_norm = get(img.name + ".qk_norm2.q_norm.weight")
            s.k_norm = get(img.name + ".qk_norm2.k_norm.weight")
            return s

        self.double: List[Tuple[_Stream, _Stream]] = []
        self.attn2: Dict[int, _Stream] = {}                                           # block index -> attn2
        for i in range(c.depth_multimodal):
            skip_text = (i == c.depth_multimodal - 1) and (c.depth_unified < 1)       # mmdit.py:62-66
            x_block = i in c.x_block_self_attn_layers
            img = stream(f"multimodal_transformer_blocks.{i}.image_transformer_block", 9 if x_block else 6)
            txt = stream(f"multimodal_transformer_blocks.{i}.text_transformer_block", 2 if skip_text else 6,
                         skip_post=skip_text)
            self.double.append((img, txt))
            if x_block:
                self.attn2[i] = attn2(img)
        self.single: List[_Stream] = []
        par = c.parallel_mlp_for_unified_blocks
        if c.depth_unified > 0 and not par:
            raise DkError("MMDiT: unified blocks without parallel MLP are not used by any reference preset")
        for i in range(c.depth_unified):
            self.single.append(stream(f"unified_transformer_blocks.{i}.transformer_block", 3, parallel=True))
        self.final_mod_off = add_mod("final_layer")
        self.w_mod = torch.cat(mod_w, dim=0).contiguous()                             # (mod_total, h)
        self.b_mod = torch.cat(mod_b, dim=0).contiguous()

    # ------------------------------------------------------------------------------------------ modulation cache
    def timestep_embedding(self, t: torch.Tensor) -> torch.Tensor:
        """Sinusoid in config.dtype arithmetic, cos first (reference mmdit.py:379-389, quirk Q5).  Tiny host math."""
        c = self.config
        half = c.frequency_embed_dim // 2
        cd = c.dtype
        ar = torch.arange(0, half, dtype=torch.float32).to(cd)
        freqs = torch.exp(-math.log(c.max_period) * ar.float() / half).to(cd)
        args = (t.reshape(-1, 1).float().to(cd).float() * freqs.float()[None]).to(cd)
        return torch.cat([torch.cos(args.float()).to(cd), torch.sin(args.float()).to(cd)], dim=-1)

    def guidance_embedding(self, guidance) -> torch.Tensor:
        """FLUX.1-dev's guidance sinusoid, as BFL's timestep_embedding computes it for the checkpoint: v = round(1000 ·
        round(g)) in the activation dtype, fp32 angles v · f_k with f_k = exp(-ln(max_period) · k / half), cos first,
        the result rounded to the activation dtype.  Unlike the timestep's (quirk Q5), the angles are not rounded:
        the reference has no working guidance path to follow.  (B,) floats -> (B, frequency_embed_dim).  Tiny host
        math."""
        c, ad = self.config, self.dtype
        half = c.frequency_embed_dim // 2
        v = (torch.tensor(guidance, dtype=torch.float32).reshape(-1).to(ad).float() * 1000.0).to(ad).float()
        freqs = torch.exp(-math.log(c.max_period) * torch.arange(0, half, dtype=torch.float32) / half)
        args = v[:, None] * freqs[None]
        return torch.cat([torch.cos(args), torch.sin(args)], dim=-1).to(ad)

    def _check_guidance(self, guidance, B: int) -> Optional[List[float]]:
        """guidance as cache_modulation_params takes it -> one float per conditioning row (None without the embedder)"""
        if not self.config.guidance_embed:
            if guidance is not None:
                raise ValueError("guidance is FLUX.1-dev's distilled guidance: this model has no guidance embedder "
                                 "(MMDiTConfig.guidance_embed is False)")
            return None
        if guidance is None:
            raise ValueError("this model has a guidance embedder (FLUX.1-dev): pass one guidance value per "
                             "conditioning row")
        vals = [float(g) for g in (guidance.tolist() if hasattr(guidance, "tolist") else guidance)]
        if len(vals) != B:
            raise ValueError(f"guidance has {len(vals)} values for {B} conditioning rows")
        if not all(math.isfinite(g) for g in vals):
            raise ValueError(f"guidance must be finite, got {vals}")
        return vals

    def cache_modulation_params(self, pooled_text_embeddings: torch.Tensor, timesteps, guidance=None, *,
                                skip_batch: int = 0):
        """All adaLN modulation vectors for every timestep and every block in one batched GEMM
        (reference mmdit.py:77-180).  pooled: (B, P); timesteps: iterable of floats already rounded to the activation
        dtype by the caller (mlx/__init__.py:769-771).  guidance: one float per row of pooled, required with a guidance
        embedder (FLUX.1-dev) and refused without one; its embedding joins the pooled-text one, once per row, ahead of
        the SiLU that feeds the modulation GEMM.  skip_batch: the last skip_batch rows condition only the skip-layer
        forwards of skip-layer guidance; a forward of the leading B - skip_batch rows alone is accepted too."""
        B = pooled_text_embeddings.shape[0]
        if not 0 <= int(skip_batch) < B:
            raise ValueError(f"skip_batch must be in [0, {B}), got {skip_batch}")
        gvals = self._check_guidance(guidance, B)
        pooled = pooled_text_embeddings.reshape(B, -1)
        pooled = pooled.to(device=self.device, dtype=self.dtype).contiguous()
        ts = [float(t) for t in (timesteps.tolist() if hasattr(timesteps, "tolist") else timesteps)]
        n_t = len(ts)
        gvec = None
        if gvals is not None:
            gemb = self.guidance_embedding(gvals).to(device=self.device)
            gvec = ops.gemm(ops.gemm(gemb, self.g0[0], bias=self.g0[1], act=ACT_SILU), self.g2[0], bias=self.g2[1])
        # y = y_embedder(pooled) (+ guidance_in(g) through the epilogue's residual: one rounding of the sum)
        y = ops.gemm(ops.gemm(pooled, self.y0[0], bias=self.y0[1], act=ACT_SILU), self.y2[0], bias=self.y2[1],
                     res=gvec)
        temb = self.timestep_embedding(torch.tensor(ts, dtype=torch.float32)).to(device=self.device, dtype=self.dtype)
        tvec = ops.gemm(ops.gemm(temb.contiguous(), self.t0[0], bias=self.t0[1], act=ACT_SILU), self.t2[0],
                        bias=self.t2[1])
        cin = ops.silu_add(y, tvec)                                                    # (n_t * B, h)
        self._mod_all = ops.gemm(cin, self.w_mod, bias=self.b_mod)                    # (n_t * B, mod_total)
        if self._mod_cur is None or self._mod_batch != B:
            # persistent buffer: captured graphs read the current step's modulation rows from this address
            self._mod_cur = torch.empty((B, self.mod_total), dtype=self.dtype, device=self.device)
            self._shapes.drop_graphs()
        self._mod_batch = B
        self._mod_skip_batch = int(skip_batch)
        self._mod_index = {}
        self._reset_step_cache()
        for i, t in enumerate(ts):
            self._mod_index.setdefault(t, i)
        self._cur_t = None

    def cache_fill_conditioning(self, rows: torch.Tensor):
        """FLUX.1 Fill (DESIGN.md §18): rows (N, cond_channels) 16-bit, the [masked-image latent | mask] columns of the
        N target tokens of one sequence, shared by every forward row -> the conditioning term
        round16(rows @ W_c^T + b_x) of the x-embedder, W_c its conditioning columns, in a buffer every later forward
        adds through the x-embedder GEMM's residual (one rounding of the sum).  Call once per denoise, after any LoRA
        change; the buffer keeps its address while N does."""
        if not self.cond_channels:
            raise ValueError("cache_fill_conditioning: this model has no conditioning channels (not FLUX.1 Fill)")
        if rows.dim() != 2 or rows.shape[1] != self.cond_channels or rows.dtype != self.dtype:
            raise ValueError(f"cache_fill_conditioning: rows must be (N, {self.cond_channels}) {self.dtype}, got "
                             f"{tuple(rows.shape)} {rows.dtype}")
        N = rows.shape[0]
        if self._fill_cond is None or self._fill_cond.shape[0] != N:
            self._fill_cond = torch.empty((N, self.h), dtype=self.dtype, device=self.device)
            self._shapes.drop_graphs()
        ops.gemm(rows.contiguous(), self.w_x[:, self.x_in:], out=self._fill_cond, bias=self.b_x)
        self._fill_rows = N
        self._reset_step_cache()

    def clear_modulation_params_cache(self):
        self._mod_index, self._mod_all = {}, None

    def select_timestep(self, timestep: float):
        """Make `timestep`'s modulation rows current (one D2D copy; keeps the forward timestep-invariant)."""
        key = float(timestep)
        if key not in self._mod_index:
            raise KeyError(f"timestep {key} not in the modulation cache (call cache_modulation_params first)")
        i = self._mod_index[key]
        B = self._mod_batch
        self._mod_cur.copy_(self._mod_all[i * B:(i + 1) * B])
        self._cur_t = key

    def _mod(self, s_off: int, k: int) -> torch.Tensor:
        """k-th h-wide modulation vector of a block: view (B, h) with row stride mod_total."""
        return self._mod_cur[:, s_off + k * self.h: s_off + (k + 1) * self.h]

    # ------------------------------------------------------------------------------------------ FP8 linears
    @property
    def fp8(self) -> bool:
        return self._fp8

    def _fp8_packed(self) -> Dict[Tuple[int, str], _Stream]:
        """(id(stream), attribute) -> stream of every packed weight that holds a covered linear"""
        slots = self.lora_weight_slots()
        out = {}
        for name in fp8_covered_linears(self.config):
            owner, attr = slots[name + ".weight"][:2]
            out[(id(owner), attr)] = owner
        return out

    def set_fp8(self, enabled: bool):
        """Run the covered block linears (fp8_covered_linears) on e4m3 tensor cores: an accuracy-for-speed trade the
        caller makes.  Enabling quantises each covered packed weight once, per output feature, into an e4m3 copy and a
        scale vector kept beside the 16-bit weight (which LoRA merges still need); disabling frees them and the e4m3
        activation buffers.  Either way the captured graphs are dropped: the launch sequence changes."""
        enabled = bool(enabled)
        self._reset_step_cache()
        if enabled == self._fp8:
            return
        self._fp8_w = {}
        if enabled:
            for key, s in self._fp8_packed().items():
                self._fp8_w[key] = ops.quantize_rows_e4m3(getattr(s, key[1]))
        self._fp8 = enabled
        self._shapes.drop("graph")
        self._shapes.drop("ws8")

    # ------------------------------------------------------------------------------------------ step cache
    def set_step_cache(self, threshold: Optional[float], max_consecutive_skips: Optional[int] = None):
        """First-block step cache (DESIGN.md §10), an accuracy-for-speed trade the caller makes; off by default.
        Each forward runs the input adapters and the first block, compares that block's residual with the one of the
        last fully computed forward (step_cache.StepCachePolicy) and, when the relative change of every sequence is
        below `threshold` and fewer than `max_consecutive_skips` forwards in a row were skipped (None: no cap), skips
        the other blocks and reuses their residual from that forward.  threshold None turns the cache off and frees its
        buffers; 0 never skips.  The cache restarts (the next forward runs in full) on every call of this method,
        cache_modulation_params, apply_lora, set_fp8 and a change of input shape or batch."""
        if threshold is not None and not self.double:
            raise DkError("MMDiT: the step cache needs at least one double-stream block")
        self._step_cache = None if threshold is None else StepCachePolicy(threshold, max_consecutive_skips)
        self._step_cache_key = None
        self._shapes.drop("graph")
        self._shapes.drop("sc")

    @property
    def step_cache(self) -> Optional[Tuple[float, Optional[int]]]:
        """(threshold, max_consecutive_skips) while the step cache is on, else None"""
        p = self._step_cache
        return None if p is None else (p.threshold, p.max_consecutive_skips)

    @property
    def step_cache_log(self) -> List[Tuple[Optional[float], bool]]:
        """(max rel, skipped) of every forward since the last reset (rel is None on the first, which never skips);
        empty while the cache is off"""
        return [] if self._step_cache is None else list(self._step_cache.log)

    def _reset_step_cache(self):
        if self._step_cache is not None:
            self._step_cache.reset()

    # ------------------------------------------------------------------------------------------ LoRA merge
    def lora_weight_slots(self) -> Dict[str, Tuple[object, str, Optional[int], slice, slice]]:
        """reference weight name -> (owner, attribute, tuple index or None, rows, columns): where each weight a LoRA
        adapter can change lives inside the packed tensors."""
        h, everything = self.h, slice(None)
        slots = {}

        def put(name, owner, attr, idx=None, rows=everything, cols=everything):
            slots[name + ".weight"] = (owner, attr, idx, rows, cols)

        put("x_embedder.proj", self, "w_x")
        put("context_embedder", self, "w_ctx")
        for emb in ("y", "t"):
            put(f"{emb}_embedder.mlp.layers.0", self, emb + "0", 0)
            put(f"{emb}_embedder.mlp.layers.2", self, emb + "2", 0)
        if self.g0 is not None:
            put("guidance_in.mlp.layers.0", self, "g0", 0)
            put("guidance_in.mlp.layers.2", self, "g2", 0)
        put("final_layer.linear", self, "w_final")
        put("final_layer.adaLN_modulation.layers.1", self, "w_mod",
            rows=slice(self.final_mod_off, self.final_mod_off + 2 * h))
        for s in self.attn2.values():
            for j, n in enumerate("qkv"):
                put(f"{s.name}.{n}_proj", s, "w_qkv", rows=slice(j * h, (j + 1) * h))
            put(f"{s.name}.o_proj", s, "w_o")
        for s in [s for pair in self.double for s in pair] + self.single:
            p = s.name
            for j, n in enumerate("qkv"):
                put(f"{p}.attn.{n}_proj", s, "w_qkv", rows=slice(j * h, (j + 1) * h))
            put(f"{p}.adaLN_modulation.layers.1", self, "w_mod", rows=slice(s.mod_off, s.mod_off + s.n_mod * h))
            if s.skip_post:
                continue
            put(f"{p}.mlp.fc1", s, "w_fc1")
            if s.w_out is not None:                                                    # [Wo | W2] column windows
                put(f"{p}.attn.o_proj", s, "w_out", cols=slice(0, h))
                put(f"{p}.mlp.fc2", s, "w_out", cols=slice(h, None))
            else:
                put(f"{p}.attn.o_proj", s, "w_o")
                put(f"{p}.mlp.fc2", s, "w_fc2")
        return slots

    @staticmethod
    def _bound(owner, attr: str, idx: Optional[int]) -> torch.Tensor:
        t = getattr(owner, attr)
        return t if idx is None else t[idx]

    @staticmethod
    def _rebind(owner, attr: str, idx: Optional[int], t: torch.Tensor):
        if idx is not None:
            old = getattr(owner, attr)
            t = old[:idx] + (t,) + old[idx + 1:]
        setattr(owner, attr, t)

    def apply_lora(self, stack):
        """Merge a stack of LoRA adapters, a sequence of (lora.LoRA, scale), into the weights:
        W = round16(W_base + Σ round16(scale·up) @ round16(down)), one wgmma GEMM per weight with W_base as its
        residual.  The forward runs exactly the kernels it runs without adapters.

        A packed tensor the stack touches keeps its current tensor as the base, which is never written (it may be the
        caller's), and gets a live copy the forward reads.  Applying another stack re-merges from the bases in place,
        so captured CUDA graphs stay valid when only scales change; tensors the stack no longer touches go back to
        their base and their live copy is freed (an empty stack frees them all).  Binding a live copy or a base drops
        the captured graphs.  With FP8 on, the e4m3 copy of every weight whose 16-bit tensor changed is re-quantised in
        place, so it keeps its address too.  A merge that changes the adaLN or t / y / guidance embedder weights clears
        the modulation cache: call cache_modulation_params again before the next forward."""
        slots = self.lora_weight_slots()
        terms: Dict[str, list] = {}
        for lora, scale in stack:
            scale = float(scale)
            if not math.isfinite(scale):
                raise ValueError(f"LoRA {lora.name}: scale must be finite, got {scale}")
            for name, (up, down) in lora.targets.items():
                if name not in slots:
                    raise KeyError(f"LoRA {lora.name}: the model has no weight {name}")
                terms.setdefault(name, []).append((scale, up, down))
        touched = {}
        for name in terms:
            owner, attr, idx = slots[name][:3]
            touched[(id(owner), attr, idx)] = (owner, attr, idx)
        rebound, mod_changed = False, False
        mod_attrs = ("w_mod", "y0", "y2", "t0", "t2", "g0", "g2")        # what the modulation cache was built from
        changed = set(touched) | set(self._lora_live)
        for key in [k for k in self._lora_live if k not in touched]:
            owner, base, _ = self._lora_live.pop(key)
            self._rebind(owner, key[1], key[2], base)
            rebound, mod_changed = True, mod_changed or key[1] in mod_attrs
        for key, (owner, attr, idx) in touched.items():
            if key not in self._lora_live:
                base = self._bound(owner, attr, idx)
                self._lora_live[key] = (owner, base, torch.empty_like(base))
                self._rebind(owner, attr, idx, self._lora_live[key][2])
                rebound = True
            _, base, live = self._lora_live[key]
            live.copy_(base)
            mod_changed = mod_changed or attr in mod_attrs
        for name, ts in terms.items():
            owner, attr, idx, rows, cols = slots[name]
            _, base, live = self._lora_live[(id(owner), attr, idx)]
            up, down = self._lora_factors(ts)
            ops.gemm(up, down, out=live[rows, cols], res=base[rows, cols], w_n_major=True)
        packed = self._fp8_packed() if self._fp8 else {}
        for oid, attr, _ in changed:
            if (oid, attr) in packed:
                q, sc = self._fp8_w[(oid, attr)]
                ops.quantize_rows_e4m3(getattr(packed[(oid, attr)], attr), out=q, scale=sc)
        if rebound:
            self._shapes.drop_graphs()
        self._reset_step_cache()
        if any(attr == "w_x" for _, attr, _ in changed):
            self._fill_rows = 0                          # the conditioning term was computed from the old W_c
        if mod_changed:
            self.clear_modulation_params_cache()
            self._cur_t = None

    def _lora_factors(self, terms) -> Tuple[torch.Tensor, torch.Tensor]:
        """[round16(s1·up1) | round16(s2·up2) | ... | 0] and [round16(down1); round16(down2); ...; 0] on the device:
        the ranks concatenated and zero-padded to a multiple of 8 (the GEMM's K)"""
        r = sum(up.shape[1] for _, up, _ in terms)
        rp = -(-r // 8) * 8
        up = torch.zeros((terms[0][1].shape[0], rp), dtype=torch.float32)
        down = torch.zeros((rp, terms[0][2].shape[1]), dtype=torch.float32)
        o = 0
        for scale, u, d in terms:
            up[:, o:o + u.shape[1]] = u * scale
            down[o:o + u.shape[1]] = d
            o += u.shape[1]
        return up.to(self.dtype).to(self.device), down.to(self.dtype).to(self.device)

    # ------------------------------------------------------------------------------------------ workspace
    def _workspace(self, st: dict, B: int, N: int, T: int):
        """N: image-stream rows per sequence (target + reference tokens)"""
        if "ws" in st:
            return st["ws"]
        h, dt, dev = self.h, self.dtype, self.device
        S = N + T
        r = self.config.mlp_ratio

        def buf(*shape):
            return torch.empty(shape, dtype=dt, device=dev)

        ws = {
            "img": buf(B * N, h), "txt": buf(B * T, h),
            "m_img": buf(B * N, h), "m_txt": buf(B * T, h),
            "qkv": buf(B * S, 3 * h),
            "o_img": buf(B * N, h), "o_txt": buf(B * T, h),
            "hid_img": buf(B * N, r * h), "hid_txt": buf(B * T, r * h),
            "rows_in": buf(B * N, self.x_in), "rows_out": buf(B * N, self.w_final.shape[0]),
        }
        if self.attn2:                                 # MMDiT-X: attn2's packed q/k/v and its attention output
            ws["qkv2"] = buf(B * N, 3 * h)
            ws["o2"] = buf(B * N, h)
        if self.is_flux:
            ws["u"] = buf(B * S, h)
            ws["m_u"] = buf(B * S, h)
            ws["cat"] = buf(B * S, (1 + r) * h)
        st["ws"] = ws
        return ws

    def _workspace8(self, st: dict, B: int, N: int, T: int) -> dict:
        """e4m3 activation buffers and their per-row scales while FP8 is on (nothing otherwise): name -> (q, scale).
        "m_*" holds a stream's LayerNorm-modulate output and, after attention, its quantised attention output."""
        if not self._fp8:
            return {}
        if "ws8" in st:
            return st["ws8"]
        h, dev, r = self.h, self.device, self.config.mlp_ratio

        def buf(rows, cols):
            return (torch.empty((rows, cols), dtype=torch.float8_e4m3fn, device=dev),
                    torch.empty((rows,), dtype=torch.float32, device=dev))

        w8 = {"m_img": buf(B * N, h), "m_txt": buf(B * T, h), "hid_img": buf(B * N, r * h), "hid_txt": buf(B * T, r * h)}
        if self.is_flux:
            w8["m_u"] = buf(B * (N + T), h)
            w8["cat"] = buf(B * (N + T), (1 + r) * h)
        st["ws8"] = w8
        return w8

    def _rope_table(self, st: dict, T: int, hp: int, wp: int,
                    ref_grid: Optional[Tuple[int, int]] = None) -> torch.Tensor:
        """(S, d/2, 2) fp32 cos/sin; text tokens at position (0,0,0), image token (r, c) at (0, r, c)
        (reference mmdit.py:865-911).  ref_grid (hpr, wpr): Kontext reference token (r, c) at (1, r, c), after the
        target's.  Cached per input shape like the reference (:916-932)."""
        if "rope" in st:
            return st["rope"]
        axes = self.config.rope_axes_dim
        grids = [(0, hp, wp)] + ([(1, *ref_grid)] if ref_grid is not None else [])
        pos = torch.zeros((T + sum(a * b for _, a, b in grids), 3), dtype=torch.float32)
        row = T
        for axis0, gh, gw in grids:
            n = gh * gw
            pos[row:row + n, 0] = float(axis0)
            pos[row:row + n, 1] = torch.arange(gh, dtype=torch.float32)[:, None].expand(gh, gw).reshape(-1)
            pos[row:row + n, 2] = torch.arange(gw, dtype=torch.float32)[None, :].expand(gh, gw).reshape(-1)
            row += n
        parts = []
        for a, dim in enumerate(axes):
            scale = torch.arange(0, dim, 2, dtype=torch.float32) / dim
            omega = 1.0 / (10000.0 ** scale)
            parts.append(pos[:, a:a + 1] * omega[None, :])
        ang = torch.cat(parts, dim=-1)
        assert ang.shape[1] == self.d // 2, "sum(rope_axes_dim) must equal the head dim"
        st["rope"] = torch.stack([torch.cos(ang), torch.sin(ang)], dim=-1).contiguous().to(self.device)
        return st["rope"]

    # ------------------------------------------------------------------------------------------ forward
    def _qk_fused(self, s: _Stream, rope):
        """epilogue spec for the packed QKV GEMM: per-head QK-RMSNorm (+ RoPE) fused in (None: nothing to fuse)"""
        if s.q_norm is None and rope is None:
            return None
        return (self.heads, self.d, s.q_norm, s.k_norm, rope, 1e-6)

    # A covered linear's input is a 16-bit tensor or, with FP8 on, the (e4m3, row scales) pair in the buffers `x8`.
    def _ln_mod(self, x, s: _Stream, k: int, rows_per_batch, m, m8):
        """LN(x) * (1 + scale_k) + shift_k of stream s as the input of a covered linear"""
        shift, scale, eps = self._mod(s.mod_off, k), self._mod(s.mod_off, k + 1), self.config.layer_norm_eps
        if self._fp8:
            return ops.ln_modulate_fp8(x, shift, scale, rows_per_batch, eps, out=m8[0], out_scale=m8[1])
        return ops.ln_modulate(x, shift, scale, rows_per_batch, eps, out=m)

    def _lin_in(self, x, x8):
        """the 16-bit activation x as the input of a covered linear"""
        return ops.quantize_rows_e4m3(x, out=x8[0], scale=x8[1]) if self._fp8 else x

    def _linear(self, a, s: _Stream, attr: str, **epilogue):
        """covered linear `attr` of stream s on an input from _ln_mod / _lin_in"""
        if self._fp8:
            wq, w_scale = self._fp8_w[(id(s), attr)]
            return ops.gemm_fp8(a[0], a[1], wq, w_scale, **epilogue)
        return ops.gemm(a, getattr(s, attr), **epilogue)

    def _attn_stream_pre(self, s: _Stream, x, m, m8, rows_per_batch, S, row_off, qkv, rope):
        a = self._ln_mod(x, s, 0, rows_per_batch, m, m8)
        self._linear(a, s, "w_qkv", out=qkv, bias=s.b_qkv, rows_per_batch=rows_per_batch, out_batch_rows=S,
                     out_row_off=row_off, qk=self._qk_fused(s, rope))

    def _stream_post(self, s: _Stream, x, o, m, m8, hid, hid8, rows_per_batch, x_attn=None):
        """x += gate1 * o_proj(o); x += gate2 * fc2(gelu(fc1(LN(x)(1+scale2)+shift2)))  (mmdit.py:521-548).
        x_attn = (attn2 stream, its attention output): MMDiT-X's x += gate_msa2 * attn2.o_proj(o2) between the two."""
        for st, ot in [(s, o)] + ([x_attn] if x_attn is not None else []):
            self._linear(self._lin_in(ot, m8), st, "w_o", out=x, bias=st.b_o, gate=self._mod(st.mod_off, 2), res=x,
                         rows_per_batch=rows_per_batch, out_batch_rows=rows_per_batch)
        a = self._ln_mod(x, s, 3, rows_per_batch, m, m8)
        self._linear(a, s, "w_fc1", out=hid, bias=s.b_fc1, act=ACT_GELU_ERF)
        self._linear(self._lin_in(hid, hid8), s, "w_fc2", out=x, bias=s.b_fc2, gate=self._mod(s.mod_off, 5), res=x,
                     rows_per_batch=rows_per_batch, out_batch_rows=rows_per_batch)

    def _check_reference(self, reference, B: int, Cl: int):
        """raise ValueError, before any launch, for a Kontext reference latent this forward cannot take"""
        if not self.is_flux:
            raise ValueError("reference: Kontext reference tokens run on FLUX-shaped configs only, not on SD3-family "
                             "models")
        if reference.dim() != 4:
            raise ValueError(f"reference must be an NHWC latent (B, Hr, Wr, {Cl}), got rank {reference.dim()}")
        Br, Hr, Wr, Cr = reference.shape
        if Br != B:
            raise ValueError(f"reference has batch {Br}, the latent has batch {B}")
        if Cr != Cl:
            raise ValueError(f"reference has {Cr} channels, the latent has {Cl}")
        p = self.config.patch_size
        if Hr % p or Wr % p or Hr == 0 or Wr == 0:
            raise ValueError(f"reference latent height and width must be positive multiples of {p}, got {Hr}x{Wr}")

    def __call__(self, latent_image_embeddings: torch.Tensor, token_level_text_embeddings: torch.Tensor,
                 timestep=None, *, reference: Optional[torch.Tensor] = None, skip_layers=(),
                 skip_batch: int = 0) -> torch.Tensor:
        """latent (B, H, W, 16) NHWC, text (B, T, 1, 4096) or (B, T, 4096), timestep (B,) tensor / float
        (all entries equal, as in the reference which reads timestep[0], mmdit.py:445-447) -> (B, H, W, 16).
        reference (FLUX.1 Kontext, FLUX-shaped configs only): a 16-bit (B, Hr, Wr, 16) latent already in the
        process_in space, Hr and Wr even; its tokens join the image stream after the target's at RoPE positions
        (1, r, c), and the output covers the target alone.
        skip_layers / skip_batch (skip-layer guidance): the last skip_batch sequences skip the listed joint blocks,
        both of their streams passing through them unchanged."""
        c = self.config
        skip_layers = tuple(sorted(set(int(i) for i in skip_layers)))
        if skip_layers:
            if self.is_flux:
                raise ValueError("skip_layers: skip-layer guidance runs on SD3-family models only")
            if not all(0 <= i < c.depth_multimodal for i in skip_layers):
                raise ValueError(f"skip_layers {skip_layers} must be joint block indices in [0, {c.depth_multimodal})")
        skip_batch = int(skip_batch) if skip_layers else 0
        x = latent_image_embeddings
        if x.dim() != 4:
            raise ValueError(f"Input tensor must have rank 4, got {x.dim()}")
        B, H, W, Cl = x.shape
        if H % c.patch_size or W % c.patch_size:
            raise DkError("latent height/width must be divisible by the patch size")
        if reference is not None:
            self._check_reference(reference, B, Cl)
        if self.cond_channels:
            if reference is not None:
                raise ValueError("reference: a FLUX.1 Fill model takes no Kontext reference")
            Nx = (H // c.patch_size) * (W // c.patch_size)
            if self._fill_rows != Nx:
                raise ValueError(f"FLUX.1 Fill: the conditioning holds {self._fill_rows} tokens, the latent has {Nx}: "
                                 "call cache_fill_conditioning for this latent first")
        text = token_level_text_embeddings
        if text.dim() == 4:
            text = text.squeeze(2)
        T = text.shape[1]
        text = text.reshape(B * T, -1).to(dtype=self.dtype)
        if not text.is_contiguous():
            text = text.contiguous()
        x = x.to(dtype=self.dtype)
        if not x.is_contiguous():
            x = x.contiguous()
        if timestep is not None:
            tval = float(timestep.reshape(-1)[0]) if torch.is_tensor(timestep) else float(timestep)
            if tval != getattr(self, "_cur_t", None):
                self.select_timestep(tval)
        if skip_layers and not 0 < skip_batch < B:
            raise ValueError(f"skip_batch must be in (0, {B}) with skip_layers, got {skip_batch}")
        lead = self._mod_batch - self._mod_skip_batch        # a forward without the skip rows reads the leading rows
        if self._mod_cur is None or B not in (self._mod_batch, lead):
            raise DkError(f"modulation cache holds batch {self._mod_batch}, forward got batch {B}")
        key = (B, H, W, Cl, T, skip_layers, skip_batch)
        inputs = (x, text)
        if reference is not None:
            # the RoPE table, the workspaces and the graphs depend on the reference grid: part of the shape key
            key += (tuple(reference.shape[1:3]),)
            ref = reference.to(dtype=self.dtype)
            inputs += (ref if ref.is_contiguous() else ref.contiguous(),)
        state = self._shapes.state(key, self.max_cached_shapes)
        state["skip"] = (frozenset(skip_layers), skip_batch)
        state["ref_hw"] = tuple(reference.shape[1:3]) if reference is not None else None
        if self._step_cache is not None:
            return self._cached_forward(state, key, inputs, B, H, W, Cl, T)
        return self._shapes.run(state, self.use_cuda_graphs,
                                lambda xx, tt, *rr: self._forward_impl(state, xx, tt, B, H, W, Cl, T, *rr), *inputs)

    def _stream_rows(self, state, H, W) -> Tuple[int, int]:
        """(target tokens Nx, image-stream rows N = Nx + Kontext reference tokens) per sequence"""
        p, ref_hw = self.config.patch_size, state["ref_hw"]
        Nx = (H // p) * (W // p)
        return Nx, Nx + (0 if ref_hw is None else (ref_hw[0] // p) * (ref_hw[1] // p))

    def _geometry(self, state, B, H, W, T) -> dict:
        """buffers and sizes of one input shape that the forward pieces below share.  N is the image stream's length:
        the target's Nx tokens, then a Kontext reference's (none without one: N = Nx)."""
        c = self.config
        hp, wp = H // c.patch_size, W // c.patch_size
        Nx, N = self._stream_rows(state, H, W)
        ref_hw = state["ref_hw"]
        ref_grid = None if ref_hw is None else (ref_hw[0] // c.patch_size, ref_hw[1] // c.patch_size)
        g = {"B": B, "T": T, "N": N, "Nx": Nx, "S": N + T, "hp": hp, "wp": wp, "ws": self._workspace(state, B, N, T),
             "w8": self._workspace8(state, B, N, T).get, "state": state,
             "skip_layers": state["skip"][0], "skip_batch": state["skip"][1]}
        g["rope"] = (self._rope_table(state, T, hp, wp, ref_grid) if c.pos_embed_type == PositionalEncoding.PreSDPARope
                     else None)
        # joint sequence order: FLUX [text, image] (mmdit.py:594-606), SD3 [image, text] (:608-625)
        g["off_img"], g["off_txt"], g["split"] = (T, 0, T) if self.is_flux else (0, N, N)
        return g

    def _embed(self, g, x, text, ref=None):
        """input adapters (mmdit.py:195-206): text -> txt, latent -> img (and a Kontext reference -> its img rows)"""
        c, ws, state, N = self.config, g["ws"], g["state"], g["N"]
        ops.gemm(text, self.w_ctx, out=ws["txt"], bias=self.b_ctx)
        if ref is not None:
            # each sequence of img is [target Nx rows | reference N - Nx rows]; both embed through the output row remap
            B, Nx = g["B"], g["Nx"]
            rows_x, rows_r = ws["rows_in"][:B * Nx], ws["rows_in"][B * Nx:]
            ops.patchify(x, 0, out=rows_x)
            ops.gemm(rows_x, self.w_x, out=ws["img"], bias=self.b_x, rows_per_batch=Nx, out_batch_rows=N, out_row_off=0)
            ops.patchify(ref, 0, out=rows_r)
            ops.gemm(rows_r, self.w_x, out=ws["img"], bias=self.b_x, rows_per_batch=N - Nx, out_batch_rows=N,
                     out_row_off=Nx)
        elif self.cond_channels:
            # FLUX.1 Fill: the latent columns plus the per-call conditioning term, broadcast over the batch
            ops.patchify(x, 0, out=ws["rows_in"])
            ops.gemm(ws["rows_in"], self.w_x[:, :self.x_in], out=ws["img"], res=self._fill_cond, rows_per_batch=N,
                     out_batch_rows=N, res_batch_rows=0)
        elif c.patchify_via_reshape:
            ops.patchify(x, 0, out=ws["rows_in"])
            ops.gemm(ws["rows_in"], self.w_x, out=ws["img"], bias=self.b_x)
        else:
            ops.patchify(x, 1, out=ws["rows_in"])
            if "pos" not in state:
                state["pos"] = ops.pos_embed_crop(self.pos_table, c.max_latent_resolution, g["hp"], g["wp"])
            ops.gemm(ws["rows_in"], self.w_x, out=ws["img"], bias=self.b_x, res=state["pos"], rows_per_batch=N,
                     out_batch_rows=N, res_batch_rows=0)

    def _double_block(self, g, i: int):
        if i in g["skip_layers"]:
            g = self._leading(g, g["B"] - g["skip_batch"])
        ws, w8, B, N, T, S, rope = g["ws"], g["w8"], g["B"], g["N"], g["T"], g["S"], g["rope"]
        img, txt, qkv = ws["img"], ws["txt"], ws["qkv"]
        si, st = self.double[i]
        self._attn_stream_pre(si, img, ws["m_img"], w8("m_img"), N, S, g["off_img"], qkv, rope)
        self._attn_stream_pre(st, txt, ws["m_txt"], w8("m_txt"), T, S, g["off_txt"], qkv, rope)
        if self.is_flux:
            ops.attention(qkv, B, S, self.heads, self.d, ws["o_txt"], split=g["split"], out1=ws["o_img"])
        else:
            ops.attention(qkv, B, S, self.heads, self.d, ws["o_img"], split=g["split"], out1=ws["o_txt"])
        x_attn = None
        if i in self.attn2:                            # MMDiT-X: self-attention over the image tokens alone
            s2 = self.attn2[i]
            self._attn_stream_pre(s2, img, ws["m_img"], w8("m_img"), N, N, 0, ws["qkv2"], rope)
            ops.attention(ws["qkv2"], B, N, self.heads, self.d, ws["o2"])
            x_attn = (s2, ws["o2"])
        self._stream_post(si, img, ws["o_img"], ws["m_img"], w8("m_img"), ws["hid_img"], w8("hid_img"), N, x_attn)
        if not st.skip_post:
            self._stream_post(st, txt, ws["o_txt"], ws["m_txt"], w8("m_txt"), ws["hid_txt"], w8("hid_txt"), T)

    @staticmethod
    def _leading(g, nb: int) -> dict:
        """the geometry of the leading nb sequences alone: every batch-major buffer cut to its first nb sequences, so
        the trailing ones pass through untouched"""
        B = g["B"]

        def cut(t):
            return t[: nb * (t.shape[0] // B)]

        w8 = g["w8"]
        sub = dict(g, B=nb, ws={k: cut(t) for k, t in g["ws"].items()})
        sub["w8"] = lambda name: None if w8(name) is None else tuple(cut(t) for t in w8(name))
        return sub

    def _single_blocks(self, g):
        """FLUX: u = [text | image], every single-stream block, image rows of u back to img (nothing for SD3)"""
        if not self.is_flux:
            return
        ws, w8, B, N, T, S, rope, h = g["ws"], g["w8"], g["B"], g["N"], g["T"], g["S"], g["rope"], self.h
        img, txt, qkv = ws["img"], ws["txt"], ws["qkv"]
        u, m_u, cat = ws["u"], ws["m_u"], ws["cat"]
        ops.copy_rows(txt, u, B, T, h, S, 0, T, 0)                                     # u = [text | image] (:234-236)
        ops.copy_rows(img, u, B, N, h, S, T, N, 0)
        for s in self.single:                                                          # mmdit.py:693-751
            a = self._ln_mod(u, s, 0, S, m_u, w8("m_u"))
            self._linear(a, s, "w_qkv", out=qkv, bias=s.b_qkv, rows_per_batch=S, out_batch_rows=S,
                         qk=self._qk_fused(s, rope))
            ops.attention(qkv, B, S, self.heads, self.d, cat[:, :h])
            self._linear(a, s, "w_fc1", out=cat[:, h:], bias=s.b_fc1, act=ACT_GELU_ERF)
            self._linear(self._lin_in(cat, w8("cat")), s, "w_out", out=u, bias=s.b_o, gate=self._mod(s.mod_off, 2),
                         res=u, rows_per_batch=S, out_batch_rows=S)
        ops.copy_rows(u, img, B, N, h, N, 0, S, T)                                     # image part (:245-247)

    def _final_layer(self, g, H, W, Cl):
        """final layer (mmdit.py:780-796) on the target rows of img + unpatchify / unpack"""
        c, ws, B, N, Nx = self.config, g["ws"], g["B"], g["N"], g["Nx"]
        img, m_img, rows_out = ws["img"], ws["m_img"], ws["rows_out"]
        if Nx != N:
            # Kontext: the leading Nx rows of every N-row sequence (contiguous already for one sequence)
            if B > 1:
                img = ops.copy_rows(img, ws["o_img"], B, Nx, self.h, Nx, 0, N, 0)
            img, m_img, rows_out = img[:B * Nx], m_img[:B * Nx], rows_out[:B * Nx]
        ops.ln_modulate(img, self._mod(self.final_mod_off, 0), self._mod(self.final_mod_off, 1), Nx,
                        c.layer_norm_eps, out=m_img)
        ops.gemm(m_img, self.w_final, out=rows_out, bias=self.b_final)
        return ops.unpatchify(rows_out, B, H, W, Cl, 0 if c.patchify_via_reshape else 1)

    def _forward_impl(self, state, x, text, B, H, W, Cl, T, ref=None):
        g = self._geometry(state, B, H, W, T)
        self._embed(g, x, text, ref)
        for i in range(len(self.double)):
            self._double_block(g, i)
        self._single_blocks(g)
        return self._final_layer(g, H, W, Cl)

    # ------------------------------------------------------------------------------------------ step cache
    # The cached forward is three pieces per shape, each its own captured graph when graphs are on:
    #   head  embedders, e -> snap, block 0 (img = a), r0 = a - e and its per-sequence sums against r0prev;
    #   tail  a -> snap, the other blocks (img = f), R = f - a, r0prev = r0, final layer;
    #   skip  img = round16(a + R), final layer.
    # Between head and the rest the host reads the sums (one stream synchronise per step) and decides.
    def _step_cache_buffers(self, state: dict, B: int, N: int) -> dict:
        if "sc" in state:
            return state["sc"]
        h, dev = self.h, self.device

        def f32(*shape):
            return torch.empty(shape, dtype=torch.float32, device=dev)

        state["sc"] = {"snap": torch.empty((B * N, h), dtype=self.dtype, device=dev), "r0": f32(B * N, h),
                       "r0prev": torch.zeros((B * N, h), dtype=torch.float32, device=dev), "R": f32(B * N, h),
                       "sums": f32(B, 2), "ws": f32(B * 512),
                       "host": torch.empty((B, 2), dtype=torch.float32, pin_memory=True)}
        return state["sc"]

    def _head_impl(self, state, x, text, B, H, W, Cl, T, ref=None):
        g = self._geometry(state, B, H, W, T)
        sc, img, BN = state["sc"], g["ws"]["img"], B * g["N"]
        self._embed(g, x, text, ref)
        ops.copy_rows(img, sc["snap"], 1, BN, self.h, BN, 0, BN, 0)                 # e
        self._double_block(g, 0)
        return ops.residual_delta(img, sc["snap"], B, g["N"], r_out=sc["r0"], prev=sc["r0prev"], sums=sc["sums"],
                                  ws=sc["ws"])

    def _tail_impl(self, state, B, H, W, Cl, T):
        g = self._geometry(state, B, H, W, T)
        sc, img, BN = state["sc"], g["ws"]["img"], B * g["N"]
        ops.copy_rows(img, sc["snap"], 1, BN, self.h, BN, 0, BN, 0)                 # a
        for i in range(1, len(self.double)):
            self._double_block(g, i)
        self._single_blocks(g)
        ops.residual_delta(img, sc["snap"], B, g["N"], r_out=sc["R"])                 # R = f - a
        # r0prev = r0: a bit copy of the fp32 rows, viewed as twice as many 16-bit columns
        ops.copy_rows(sc["r0"].view(self.dtype), sc["r0prev"].view(self.dtype), 1, BN, 2 * self.h, BN, 0, BN, 0)
        return self._final_layer(g, H, W, Cl)

    def _skip_impl(self, state, B, H, W, Cl, T):
        g = self._geometry(state, B, H, W, T)
        ops.residual_apply(g["ws"]["img"], state["sc"]["R"], out=g["ws"]["img"])    # f = round16(a + R)
        return self._final_layer(g, H, W, Cl)

    def _cached_forward(self, state, key, inputs, B, H, W, Cl, T):
        policy = self._step_cache
        if key != self._step_cache_key:
            policy.reset()
            self._step_cache_key = key
        sc = self._step_cache_buffers(state, B, self._stream_rows(state, H, W)[1])
        graphs = self.use_cuda_graphs
        self._shapes.run(state, graphs, lambda xx, tt, *rr: self._head_impl(state, xx, tt, B, H, W, Cl, T, *rr),
                         *inputs, name="graph.head")
        sc["host"].copy_(sc["sums"], non_blocking=True)
        torch.cuda.current_stream(self.device).synchronize()
        part = self._skip_impl if policy.step(sc["host"].tolist()) else self._tail_impl
        return self._shapes.run(state, graphs, lambda: part(state, B, H, W, Cl, T), stateful=True, device=self.device,
                                name="graph.skip" if part == self._skip_impl else "graph.tail")
