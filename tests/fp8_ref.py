"""Test infrastructure for the FP8 linears (never imported by the product path): the row quantiser's rule in fp32
torch, and the MMDiT oracle with exactly the covered linears fake-quantised, so that a check of the FP8 path compares
like with like and no tolerance has to guess what e4m3 costs.
"""
import torch

from oracle.mmdit_ref import MMDiTRef, _r

E4M3_MAX = 448.0


def quantize_rows_e4m3(x: torch.Tensor):
    """x [..., cols] -> (q as fp32 holding e4m3 values, scale [...]): scale = amax|row| / 448 (1 for a zero row),
    q = e4m3_rn_satfinite(x / scale), all in fp32.  torch's float8_e4m3fn cast rounds to nearest even; the clamp to
    +-448 first is satfinite."""
    x = x.float()
    amax = x.abs().amax(dim=-1)
    scale = torch.where(amax > 0, amax / E4M3_MAX, torch.ones_like(amax))
    q = (x / scale[..., None]).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).float()
    return q, scale


def fake_quantize_rows(x: torch.Tensor) -> torch.Tensor:
    q, scale = quantize_rows_e4m3(x)
    return q * scale[..., None]


class FakeQuantMMDiTRef(MMDiTRef):
    """MMDiTRef whose covered linears (names from diffusionkit_b200.mmdit.fp8_covered_linears) see their input rows
    and weight rows fake-quantised.  FLUX single blocks quantise the [attn | GELU(fc1)] row and the [Wo | W2] row as
    one, as the engine's packed out projection does."""

    def __init__(self, cfg, params, covered, act_dtype=None):
        super().__init__(cfg, params, act_dtype)
        self.covered = set(covered)
        self._wq = {}

    def _w(self, name):
        if name not in self._wq:
            self._wq[name] = fake_quantize_rows(self.p[name])
        return self._wq[name]

    def _lin(self, x, prefix, bias=True):
        if prefix not in self.covered:
            return super()._lin(x, prefix, bias)
        y = fake_quantize_rows(x) @ self._w(prefix + ".weight").t()
        b = self.p.get(prefix + ".bias") if bias else None
        return _r(y if b is None else y + b.float(), self.dt)

    def _post_sdpa(self, x, o, m, mods, bn, parallel_mlp):
        if not parallel_mlp or bn + ".attn.o_proj" not in self.covered:
            return super()._post_sdpa(x, o, m, mods, bn, parallel_mlp)
        h1 = _r(self._gelu(self._lin(m, bn + ".mlp.fc1")), self.dt)
        key = bn + ".out"
        if key not in self._wq:
            self._wq[key] = fake_quantize_rows(torch.cat([self.p[bn + ".attn.o_proj.weight"].float(),
                                                          self.p[bn + ".mlp.fc2.weight"].float()], dim=1))
        y = fake_quantize_rows(torch.cat([o, h1], dim=-1)) @ self._wq[key].t() + self.p[bn + ".attn.o_proj.bias"].float()
        return _r(x + mods[2][:, None, :] * _r(y, self.dt), self.dt)
