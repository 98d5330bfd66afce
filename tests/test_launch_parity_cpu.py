"""CPU checks of the launch census (tests/launch_parity.py): every op that reaches a dk_* entry point has a census
reference or a stated reason why no model path reaches it, and the GEMM reference reproduces dk_gemm's row remap,
broadcast residual, strided gate and column count (include/dkb200.h) against a plain loop."""
import torch

from diffusionkit_b200._lib import ACT_SILU
from tests import kernel_checks as kc
from tests import launch_parity as lp


def test_every_launching_op_has_a_reference():
    names = lp.launching_ops()
    assert "gemm" in names and "conv3x3_fused" in names and "gemm_fp8" not in names    # gemm_fp8 launches via gemm
    assert not [n for n in names if n not in lp.CHECKS], "ops without a census reference"
    assert not [n for n in names if n not in lp.WRITES and n not in ("pos_embed_crop", "image_pre", "image_post",
                                                                      "conv_up_weights")]
    assert set(lp.NOT_REACHED) <= set(names) and all(len(r) > 20 for r in lp.NOT_REACHED.values())
    assert set(lp.CHECKS) <= set(names), "census checks for ops that no longer launch"


def test_gemm_reference_addressing():
    """out[row(m), n] = res[rrow(m), n] + gate[m / rpb, n] * act(A W^T + bias) with a strided gate, a residual broadcast
    to every batch (res_batch_rows = 0) at a row offset, N below W's row count, and W given N-major"""
    g = torch.Generator().manual_seed(0)
    M, K, Nw, N, rpb, obr, off, roff = 12, 8, 24, 16, 4, 7, 2, 3
    A = torch.randn((M, K), generator=g)
    W = torch.randn((Nw, K), generator=g)
    bias = torch.randn((Nw,), generator=g)
    table = torch.randn((M // rpb, 5 * N), generator=g)
    gate = table[:, 2 * N:3 * N]                                           # row stride 5N, as MMDiT._mod views it
    res = torch.randn((roff + rpb, N), generator=g)
    got = kc.ref_gemm(A, W, bias, ACT_SILU, gate, res, rows_per_batch=rpb, res_batch_rows=0, res_row_off=roff, N=N)
    rows = kc.gemm_out_rows(M, rpb, obr, off, device="cpu")
    want = torch.empty((M, N))
    for m in range(M):
        b = m // rpb
        assert int(rows[m]) == b * obr + off + m % rpb
        for n in range(N):
            acc = sum(float(A[m, k]) * float(W[n, k]) for k in range(K)) + float(bias[n])
            acc = acc / (1.0 + pow(2.718281828459045, -acc))
            want[m, n] = float(res[roff + m % rpb, n]) + float(gate[b, n]) * acc
    assert torch.allclose(got, want, rtol=1e-5, atol=1e-5)
    nm = kc.ref_gemm(A, W.t().contiguous(), bias, ACT_SILU, gate, res, rows_per_batch=rpb, res_batch_rows=0,
                     res_row_off=roff, N=N, w_n_major=True)
    assert torch.allclose(nm, got, rtol=1e-6, atol=1e-6)
    # without rows_per_batch, the residual row is res_row_off + m and the whole product is one batch
    plain = kc.ref_gemm(A, W, None, 0, None, torch.randn((M + 1, Nw), generator=g)[:, :Nw], res_row_off=1)
    assert plain.shape == (M, Nw)
    assert torch.equal(kc.gemm_out_rows(M, 0, 0, 5, device="cpu"), torch.arange(M) + 5)


def test_references_of_the_layout_ops_invert():
    lat = torch.randn((2, 8, 12, 16))
    for order in (0, 1):
        rows = kc.ref_patchify(lat, order)
        assert torch.equal(kc.ref_unpatchify(rows, 2, 8, 12, 16, order), lat)
    w = torch.randn((8, 3, 3, 16)).to(torch.bfloat16)
    wp = kc.ref_conv_up_weights(w).float().reshape(4, 8, 4, 16)
    # phase (0, 0), tap (1, 1) sums ky, kx in {1, 2}; phase (1, 1), tap (0, 0) sums ky, kx in {0, 1}
    assert torch.allclose(wp[0, :, 3], w.float()[:, 1:, 1:].sum(dim=(1, 2)).to(torch.bfloat16).float())
    assert torch.allclose(wp[3, :, 0], w.float()[:, :2, :2].sum(dim=(1, 2)).to(torch.bfloat16).float())
