"""GPU: the fused layer kernel (csrc/fused_layer.cu: aggregation produced straight into the wgmma GEMM's operand
stages) against the unfused pair it replaces (gr_aggregate_dual_abs -> gr_linear_tc_planes), through the C ABI.
The A operand is bit-identical by construction; the tensor core accumulates the k-blocks in a different order, so the
outputs agree to fp32 rounding (checked at 2e-5 of the output scale, the existing plane tolerance) -- and against the
reference goldens of the hot shape through the whole model (ops.FUSED_LAYER on / off)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import gnn_rag_b200 as G
from gnn_rag_b200 import batching, ops
from gnn_rag_b200 import synthetic as S

DEV = "cuda"


def _stage(batch, R1, normalized=False):
    return batching.stage_batch(batch, torch.device(DEV), R1, normalized, False)


def _unfused(g, prior, pf, pi, ins, h_hi, h_lo, W, bias, wsc, wt, wh, I, need_c=True):
    M = h_hi.shape[0]
    D = ins.shape[2]
    Kpad = 208 * (2 * I + 1)
    Kp = (Kpad + 63) // 64 * 64
    hi = torch.zeros(M, Kp, dtype=torch.bfloat16, device=DEV)
    lo = torch.zeros(M, Kp, dtype=torch.bfloat16, device=DEV)
    hi[:, :208] = h_hi[:, :208]
    lo[:, :208] = h_lo[:, :208]
    ops.aggregate_dual_abs(g, prior, pf, pi, ins, (hi, lo), 208, 208, wt, wh)
    out = torch.empty(M, D, device=DEV) if need_c else None
    nhi = torch.zeros(M, Kp, dtype=torch.bfloat16, device=DEV)
    nlo = torch.zeros(M, Kp, dtype=torch.bfloat16, device=DEV)
    dots = torch.empty(2 * M, device=DEV) if wsc is not None else None
    ops.linear_tc_planes(hi, lo, Kpad, W, bias, out=out, out_planes=(nhi, nlo), w_score=wsc, dots=dots, relu=True,
                         k_seg=D, k_seg_pitch=208)
    return out, nhi, nlo, dots


@pytest.mark.parametrize("B,N,E,normalized,I", [
    (3, 2000, 6000, False, 2),        # the hot shape, questions end inside tiles (2000 % 128 != 0)
    (5, 130, 900, True, 2),           # tiles span two questions, last tile partial, edge weights
    (2, 1000, 20000, False, 2),       # ~2600 in-edges per 128-row tile: the staging buffer overflows (slow path)
    (4, 700, 5000, False, 1),         # one instruction
])
def test_fused_layer_matches_the_unfused_pair(B, N, E, normalized, I):
    D, R = 200, 60
    b = S.make_batch(17, B=B, N=N, E=E, num_entity=5000, num_relation=R, num_word=50, n_real="ragged", powerlaw=True)
    db = _stage(b, R + 1, normalized)
    g = db.graph
    wt, wh = (g.w_t, g.w_h) if normalized else (None, None)
    assert ops.fused_layer_supported(N, D, 208, I, D)
    rs = np.random.RandomState(5)
    M = B * N
    tab = torch.from_numpy(rs.randn(2 * (R + 1), D).astype(np.float32)).to(DEV)
    pn = ops.pad_table256(tab)
    pf, pi = pn[: R + 1], pn[R + 1:]
    ins = torch.from_numpy(rs.randn(B, I, D).astype(np.float32)).to(DEV)
    h = torch.from_numpy(rs.randn(M, D).astype(np.float32)).to(DEV)
    h_hi = torch.zeros(M, 256, dtype=torch.bfloat16, device=DEV)
    h_lo = torch.zeros(M, 256, dtype=torch.bfloat16, device=DEV)
    ops.split_bf16(h, h_hi, h_lo)
    # columns beyond the segment pitch are NOT part of the h segment: the kernel must not read them
    h_hi[:, 208:] = float("nan")
    h_lo[:, 208:] = float("nan")
    W = torch.from_numpy((rs.randn(D, (2 * I + 1) * D) / np.sqrt(D)).astype(np.float32)).to(DEV)
    bias = torch.from_numpy(rs.randn(D).astype(np.float32) * 0.1).to(DEV)
    wsc = torch.from_numpy(rs.randn(D).astype(np.float32)).to(DEV)
    for kind in ("dense", "onehot"):
        prior = (torch.softmax(torch.from_numpy(rs.randn(B, N).astype(np.float32)), 1) if kind == "dense"
                 else torch.from_numpy(b[4].astype(np.float32))).to(DEV)
        want, whi, wlo, wdots = _unfused(g, prior, pf, pi, ins, h_hi, h_lo, W, bias, wsc, wt, wh, I)
        runs = []
        for _ in range(2):
            out = torch.full((M, D), 7.0, device=DEV)
            nhi = torch.zeros(M, 256, dtype=torch.bfloat16, device=DEV)
            nlo = torch.zeros(M, 256, dtype=torch.bfloat16, device=DEV)
            dots = torch.full((2 * M,), 7.0, device=DEV)
            ops.fused_layer(g, prior, pf, pi, ins, (h_hi, h_lo), 208, W, bias, out=out, out_planes=(nhi, nlo),
                            w_score=wsc, dots=dots, relu=True, w_t=wt, w_h=wh)
            torch.cuda.synchronize()
            runs.append((out, nhi, nlo, dots))
        for a, c in zip(runs[0], runs[1]):
            assert torch.equal(a, c)                                   # run-to-run bit identical
        out, nhi, nlo, dots = runs[0]
        scale = want.abs().max().item()
        assert torch.isfinite(out).all()
        assert (out - want).abs().max().item() <= 2e-5 * scale, (kind, (out - want).abs().max().item(), scale)
        got_p = nhi[:, :208].float() + nlo[:, :208].float()
        want_p = whi[:, :208].float() + wlo[:, :208].float()
        assert (got_p - want_p).abs().max().item() <= 2e-5 * scale
        assert (got_p[:, 200:] == 0).all() and (nhi[:, 208:] == 0).all()     # pad columns zero, nothing beyond written
        d_got = dots[:M] + dots[M:]
        d_want = wdots[:M] + wdots[M:]
        assert (d_got - d_want).abs().max().item() <= 2e-5 * d_want.abs().max().item() + 1e-6
        assert ((want == 0) & (out != 0)).sum().item() <= 1e-4 * want.numel()   # relu zeros stay zeros (up to rounding)


def test_fused_layer_without_fp32_output_and_status_codes():
    B, N, D, R, I = 2, 256, 200, 30, 2
    b = S.make_batch(3, B=B, N=N, E=1500, num_entity=3000, num_relation=R, num_word=50)
    g = _stage(b, R + 1).graph
    rs = np.random.RandomState(1)
    M = B * N
    pn = ops.pad_table256(torch.from_numpy(rs.randn(2 * (R + 1), D).astype(np.float32)).to(DEV))
    ins = torch.from_numpy(rs.randn(B, I, D).astype(np.float32)).to(DEV)
    h = torch.from_numpy(rs.randn(M, D).astype(np.float32)).to(DEV)
    h_hi = torch.zeros(M, 208, dtype=torch.bfloat16, device=DEV)
    h_lo = torch.zeros(M, 208, dtype=torch.bfloat16, device=DEV)
    ops.split_bf16(h, h_hi, h_lo)
    W = torch.from_numpy((rs.randn(D, 5 * D) / 14).astype(np.float32)).to(DEV)
    prior = torch.softmax(torch.from_numpy(rs.randn(B, N).astype(np.float32)), 1).to(DEV)
    want, whi, wlo, _ = _unfused(g, prior, pn[: R + 1], pn[R + 1:], ins, h_hi, h_lo, W, None, None, None, None, I)
    nhi = torch.zeros(M, 208, dtype=torch.bfloat16, device=DEV)
    nlo = torch.zeros(M, 208, dtype=torch.bfloat16, device=DEV)
    ops.fused_layer(g, prior, pn[: R + 1], pn[R + 1:], ins, (h_hi, h_lo), 208, W, None, out=None,
                    out_planes=(nhi, nlo), relu=True)
    got = nhi.float() + nlo.float()
    ref = whi[:, :208].float() + wlo[:, :208].float()
    assert (got - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()
    assert not ops.fused_layer_supported(64, D, 208, I, D)        # N < one tile
    assert not ops.fused_layer_supported(N, D, 208, 3, D)         # three instructions: operand slots do not fit
    with pytest.raises(Exception):
        ops.fused_layer(g, prior, pn[: R + 1], pn[R + 1:], ins[:, :1].repeat(1, 3, 1), (h_hi, h_lo), 208,
                        torch.zeros(D, 7 * D, device=DEV), None, out=None, out_planes=(nhi, nlo))


def test_model_forward_fused_equals_unfused_on_the_hot_shape():
    args = S.model_args("ReaRev", entity_dim=200, word_dim=64, num_iter=2, num_ins=2, num_gnn=3, use_cuda=True)
    torch.manual_seed(0)
    m = G.ReaRev(dict(args), 4000, 40, 60).eval()
    b = S.make_batch(9, B=4, N=600, E=3000, num_entity=4000, num_relation=40, num_word=60)
    outs = {}
    min_rows = ops.FUSED_MIN_ROWS
    ops.FUSED_MIN_ROWS = 0                                       # the test batch is smaller than one tile per SM
    for flag in (False, True):
        ops.FUSED_LAYER = flag
        try:
            n0 = ops.STATS.launches
            loss, pred, dist, _ = m(b)
            outs[flag] = (float(loss), dist.clone(), ops.STATS.launches - n0)
        finally:
            ops.FUSED_LAYER = True
    ops.FUSED_MIN_ROWS = min_rows
    assert outs[True][2] != outs[False][2]                        # fewer launches: the fused kernel really ran
    a, r = outs[True][1], outs[False][1]
    assert (a - r).abs().max().item() <= 1e-5 * r.max().item()
    assert abs(outs[True][0] - outs[False][0]) <= 1e-5 * abs(outs[False][0])
