"""Stored outputs of the reference's own code, for the tests that compare the project against it.

A test hands the reference-side part of its comparison to `recorded(name, compute)` as a function returning a dict of
arrays / tensors / strings.  The values come from tests/golden/reference_<name>.npz, so the test runs without the
reference checkout.  When the checkout is present the values are recomputed as well and must equal the stored ones
(DK_RECORD_REFERENCE=1 rewrites the file instead).  Float arrays above SAMPLE elements are stored as a fixed, seeded
sample of their elements plus their shape and L2 norm, which keeps every file far below 1 MB.
"""
import hashlib
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
SAMPLE = 4096


def _np(v):
    if isinstance(v, torch.Tensor):
        return v.detach().cpu().numpy()
    return np.asarray(v)


def digest(t) -> str:
    """exact identity of a tensor: sha256 of its shape and its float32 bytes"""
    a = np.ascontiguousarray(_np(t).astype(np.float32))
    return hashlib.sha256(repr(a.shape).encode() + a.tobytes()).hexdigest()


def _pack(values):
    out = {}
    for k, v in values.items():
        a = _np(v)
        if a.dtype.kind == "f" and a.size > SAMPLE:
            idx = np.sort(np.random.default_rng(0).choice(a.size, SAMPLE, replace=False))
            out[k + "@shape"] = np.asarray(a.shape, dtype=np.int64)
            out[k + "@idx"] = idx.astype(np.int64)
            out[k + "@val"] = a.reshape(-1)[idx].astype(np.float32)
            out[k + "@norm"] = np.asarray(np.linalg.norm(a.astype(np.float64)))
        else:
            out[k] = a.astype(np.float32) if a.dtype.kind == "f" else a
    return out


class Recorded:
    def __init__(self, packed):
        self.d = packed

    def __getitem__(self, k):
        return self.d[k]

    def close(self, k, got, atol, rtol):
        """got (tensor / array) == the stored reference value k within atol + rtol * |want| (element-wise on the stored
        elements; a sampled array also has to match shape and L2 norm)"""
        g = _np(got).astype(np.float64)
        if k + "@shape" in self.d:
            assert tuple(g.shape) == tuple(self.d[k + "@shape"]), (k, g.shape)
            want = self.d[k + "@val"].astype(np.float64)
            gv = g.reshape(-1)[self.d[k + "@idx"]]
            n = float(self.d[k + "@norm"])
            assert abs(np.linalg.norm(g) - n) <= atol * np.sqrt(g.size) + rtol * n, (k, np.linalg.norm(g), n)
        else:
            want = self.d[k].astype(np.float64)
            assert g.shape == want.shape, (k, g.shape, want.shape)
            gv = g
        err = np.abs(gv - want) - (atol + rtol * np.abs(want))
        assert err.max(initial=-1.0) <= 0, (k, float(np.abs(gv - want).max()))


def recorded(name, compute, available: bool) -> Recorded:
    path = os.path.join(HERE, f"reference_{name}.npz")
    if available:
        live = _pack(compute())
        if os.environ.get("DK_RECORD_REFERENCE") == "1" or not os.path.exists(path):
            np.savez_compressed(path, **live)
        else:
            stored = dict(np.load(path, allow_pickle=False))
            assert set(stored) == set(live), (name, sorted(set(stored) ^ set(live)))
            for k, v in live.items():
                if v.dtype.kind == "f":
                    assert np.allclose(v, stored[k], atol=1e-6, rtol=1e-5), (name, k)
                else:
                    assert np.array_equal(v, stored[k]), (name, k)
    return Recorded(dict(np.load(path, allow_pickle=False)))
