"""GPU: every accumulator width the wgmma kernels are instantiated for (csrc/wgmma.cuh).  The output width n_pad
= round16(N) rounds up to an instantiated width (64, 128, 208, 256 for the GEMM; 64, 128, 208, 224 for the fused
layer), the W rows beyond N come from the TMA zero fill and the epilogue skips the columns beyond n_pad.

- gr_linear_tc_planes against an fp64 product, for N on both sides of every width, with the three-product split and
  the single bf16 product, clusters of 1 and 2 CTAs and k-blocks of 32 and 64.
- the fused layer kernel against the unfused pair (generic aggregation into bf16 planes -> gr_linear_tc_planes) at
  D = 50, 120 and 200 with one and two instructions."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from gnn_rag_b200 import batching, ops
from gnn_rag_b200 import synthetic as S

DEV = "cuda"


@pytest.fixture
def tc_options():
    yield
    ops.set_option("tc_cluster", 1)                    # the documented defaults (linear_tc.cu)
    ops.set_option("tc_bk", 32)
    ops.ACT_BF16 = False


def _bf16(x):
    return x.to(torch.bfloat16).to(torch.float64)


@pytest.mark.parametrize("N", [8, 16, 50, 64, 100, 128, 200, 208, 224, 256])
@pytest.mark.parametrize("single", [False, True])
@pytest.mark.parametrize("cluster,bk", [(1, 32), (2, 32), (1, 64), (2, 64)])
def test_linear_tc_planes_every_width(N, single, cluster, bk, tc_options):
    ops.set_option("tc_cluster", cluster)
    ops.set_option("tc_bk", bk)
    ops.ACT_BF16 = single
    M, K = 1000, 336                                   # partial last 128-row tile, K not a multiple of 64
    rs = np.random.RandomState(N + 7 * bk + cluster)
    A = torch.from_numpy(rs.randn(M, K).astype(np.float32)).to(DEV)
    W = torch.from_numpy((rs.randn(N, K) / np.sqrt(K)).astype(np.float32)).to(DEV)
    bias = torch.from_numpy(rs.randn(N).astype(np.float32) * 0.1).to(DEV)
    wsc = torch.from_numpy(rs.randn(N).astype(np.float32)).to(DEV)
    a_hi = torch.zeros(M, K, dtype=torch.bfloat16, device=DEV)
    a_lo = torch.zeros(M, K, dtype=torch.bfloat16, device=DEV)
    ops.split_bf16(A, a_hi, a_lo)
    n16 = (N + 15) // 16 * 16
    out = torch.full((M, N), 7.0, device=DEV)
    c_hi = torch.full((M, n16 + 16), 3.0, dtype=torch.bfloat16, device=DEV)
    c_lo = torch.full((M, n16 + 16), 3.0, dtype=torch.bfloat16, device=DEV)
    dots = torch.full((2 * M,), 7.0, device=DEV)
    ops.linear_tc_planes(a_hi, a_lo, K, W, bias, out=out, out_planes=(c_hi, c_lo), w_score=wsc, dots=dots, relu=True,
                         single_ok=True)
    torch.cuda.synchronize()
    if single:
        want = _bf16(a_hi) @ _bf16(W).T          # one product A_hi W_hi
    else:
        want = A.double() @ W.double().T
    want = torch.relu(want + bias.double())
    scale = want.abs().max().item()
    assert (out.double() - want).abs().max().item() <= 2e-5 * scale
    planes = c_hi.double() + c_lo.double()
    assert (planes[:, :N] - out.double()).abs().max().item() <= 1e-5 * scale
    assert (c_hi[:, N:n16] == 0).all() and (c_lo[:, N:n16] == 0).all()       # pad columns written as zero
    assert (c_hi[:, n16:] == 3.0).all()                                         # nothing beyond round16(N)
    d_want = want @ wsc.double()
    d_got = (dots[:M] + dots[M:]).double()
    assert (d_got - d_want).abs().max().item() <= 1e-4 * d_want.abs().max().item() + 1e-5


@pytest.mark.parametrize("D", [50, 120, 200])
@pytest.mark.parametrize("I", [1, 2])
def test_fused_layer_every_width_matches_the_unfused_pair(D, I):
    B, N, E, R = 3, 700, 5000, 40
    pitch = (D + 15) // 16 * 16
    T = 2 * I + 1
    b = S.make_batch(23, B=B, N=N, E=E, num_entity=4000, num_relation=R, num_word=50, n_real="ragged")
    g = batching.stage_batch(b, torch.device(DEV), R + 1, False, False).graph
    assert ops.fused_layer_supported(N, D, pitch, I, D)
    rs = np.random.RandomState(D + I)
    M = B * N
    tab = torch.from_numpy(rs.randn(2 * (R + 1), D).astype(np.float32)).to(DEV)
    pn = ops.pad_table256(tab)
    ins = torch.from_numpy(rs.randn(B, I, D).astype(np.float32)).to(DEV)
    h = torch.from_numpy(rs.randn(M, D).astype(np.float32)).to(DEV)
    W = torch.from_numpy((rs.randn(D, T * D) / np.sqrt(D)).astype(np.float32)).to(DEV)
    bias = torch.from_numpy(rs.randn(D).astype(np.float32) * 0.1).to(DEV)
    wsc = torch.from_numpy(rs.randn(D).astype(np.float32)).to(DEV)
    prior = torch.softmax(torch.from_numpy(rs.randn(B, N).astype(np.float32)), 1).to(DEV)

    # unfused pair: [h | nb segments] planes with row pitch T * pitch, then the GEMM
    hi = torch.zeros(M, T * pitch, dtype=torch.bfloat16, device=DEV)
    lo = torch.zeros(M, T * pitch, dtype=torch.bfloat16, device=DEV)
    ops.split_bf16(h, hi, lo)
    ops.aggregate_dual(g, prior, tab[: R + 1], tab[R + 1:], ins, None, pitch, planes=(hi, lo), seg_pitch=pitch)
    want = torch.empty(M, D, device=DEV)
    wdots = torch.empty(2 * M, device=DEV)
    ops.linear_tc_planes(hi, lo, T * pitch, W, bias, out=want, w_score=wsc, dots=wdots, relu=True, k_seg=D,
                         k_seg_pitch=pitch)

    h_hi = torch.zeros(M, pitch, dtype=torch.bfloat16, device=DEV)
    h_lo = torch.zeros(M, pitch, dtype=torch.bfloat16, device=DEV)
    ops.split_bf16(h, h_hi, h_lo)
    out = torch.full((M, pitch), 7.0, device=DEV)[:, :D]          # TMA-store epilogue: 16-byte row pitch
    nhi = torch.zeros(M, pitch, dtype=torch.bfloat16, device=DEV)
    nlo = torch.zeros(M, pitch, dtype=torch.bfloat16, device=DEV)
    dots = torch.full((2 * M,), 7.0, device=DEV)
    ops.fused_layer(g, prior, pn[: R + 1], pn[R + 1:], ins, (h_hi, h_lo), pitch, W, bias, out=out,
                    out_planes=(nhi, nlo), w_score=wsc, dots=dots, relu=True)
    torch.cuda.synchronize()
    scale = want.abs().max().item()
    assert torch.isfinite(out).all()
    assert (out - want).abs().max().item() <= 2e-5 * scale
    got_p = nhi.float() + nlo.float()
    assert (got_p[:, :D] - out).abs().max().item() <= 1e-5 * scale
    assert (got_p[:, D:] == 0).all()
    d_got, d_want = dots[:M] + dots[M:], wdots[:M] + wdots[M:]
    assert (d_got - d_want).abs().max().item() <= 2e-5 * d_want.abs().max().item() + 1e-6
