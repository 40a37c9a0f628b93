"""GPU: the dense-prior layer with its neighbour segments in the K-order layout -- gr_aggregate_dual_abs_ex with
GR_AGG_K_ORDER, then gr_linear_tc_planes with GR_LINEAR_K_GROUPED | GR_LINEAR_K_ORDER_PLANES, the pair ops.dense_layer
runs -- held bit for bit to what it replaces:
  * the pair against gr_fused_layer: fp32 h, both output planes and the score dots, on NaN-prefilled outputs and with
    NaN in every plane column the aggregation does not write;
  * the aggregation against the segment-layout aggregation, permuted by the column map, in every agg_abs_ws mode; the
    columns before the region and past it keep their contents;
  * the GEMM against the grouped-order GEMM on the same A operand permuted on the host into the K-order layout, at
    D = 200 and at the other widths the grouped order admits (full and 16-column last groups, one and three
    instructions).
Each of these walks the same k16 steps in the same order on the same operand bits, so equality is exact."""
import math

import numpy as np
import pytest
import torch

from gnn_rag_b200 import batching, ops
from gnn_rag_b200 import synthetic as S

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16 = torch.bfloat16
NAN = float("nan")


def _t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


def _bits(x):
    return x.view(torch.int16 if x.dtype == BF16 else torch.int32)


def korder_index(P, I):
    """(dst, src): plane column dst of the K-order layout holds column src of the segment layout (neighbours only)."""
    nb0, Gf = ops.k_order_nb0(P), P // 32
    dst, src = [], []
    for d in range(2):
        for j in range(I):
            u, s = d * I + j, 1 + 2 * j + d
            for c in range(P):
                dst.append(nb0 + ((c >> 5) * 64 * I + 32 * u + (c & 31) if c < 32 * Gf else Gf * 64 * I + 16 * u + c - 32 * Gf))
                src.append(s * P + c)
    return torch.tensor(dst, device=DEV), torch.tensor(src, device=DEV)


@pytest.fixture
def options():
    yield ops.set_option
    ops.set_option("tc_cluster", 1)
    ops.set_option("agg_abs_ws", 2)


def _graph(B, N, E, normalized, R=60):
    b = S.make_batch(17, B=B, N=N, E=E, num_entity=5000, num_relation=R, num_word=50, n_real="ragged", powerlaw=True)
    g = batching.stage_batch(b, torch.device(DEV), R + 1, normalized, False).graph
    return b, g, ((g.w_t, g.w_h) if normalized else (None, None))


@pytest.mark.parametrize("B,N,E,normalized,I", [
    (3, 2000, 6000, False, 2),        # M = 6000: 47 tiles (fewer than SMs), the last one partial
    (5, 130, 900, True, 2),           # tiles span two questions, normalized_gnn edge weights
    (2, 1000, 20000, False, 2),       # ~2600 in-edges per tile: hub rows past the staging capacity
    (4, 700, 5000, False, 1),         # one instruction (T = 3)
    (32, 2000, 6000, False, 2),       # 500 tiles: several per persistent CTA
])
def test_k_order_pair_equals_fused_layer_bit_for_bit(B, N, E, normalized, I, options):
    D, P, R = 200, 208, 60
    b, g, (wt, wh) = _graph(B, N, E, normalized, R)
    assert ops.fused_layer_supported(N, D, P, I, D)
    rs = np.random.RandomState(5)
    M, T = B * N, 2 * I + 1
    tiles = math.ceil(M / 128)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert (tiles < sms) if B <= 5 else (tiles >= 3 * sms)
    pn = ops.pad_table256(_t(rs.randn(2 * (R + 1), D)))
    pf, pi = pn[: R + 1], pn[R + 1:]
    ins = _t(rs.randn(B, I, D))
    Kp = (T * P + 63) // 64 * 64
    planes = [torch.zeros(M, Kp, dtype=BF16, device=DEV) for _ in range(2)]
    ops.split_bf16(_t(rs.randn(M, D)), planes[0], planes[1])
    for p in planes:
        p[:, P:] = NAN                       # 208 .. 223 are never written and must never be read; the region is written
    h_hi, h_lo = (p[:, :256].clone() for p in planes)
    W = _t(rs.randn(D, T * D) / np.sqrt(D))
    bias = _t(rs.randn(D) * 0.1)
    wsc = _t(rs.randn(D))

    def outputs():
        return (torch.full((M, D), NAN, device=DEV), torch.full((M, 256), NAN, dtype=BF16, device=DEV),
                torch.full((M, 256), NAN, dtype=BF16, device=DEV), torch.full((2 * M,), NAN, device=DEV))

    for kind in ("dense", "onehot"):
        prior = (torch.softmax(_t(rs.randn(B, N)), 1) if kind == "dense" else _t(b[4].astype(np.float32)))
        want = outputs()
        ops.fused_layer(g, prior, pf, pi, ins, (h_hi, h_lo), P, W, bias, out=want[0], out_planes=want[1:3],
                        w_score=wsc, dots=want[3], relu=True, w_t=wt, w_h=wh)
        assert torch.isfinite(want[0]).all() and torch.isfinite(want[3]).all()
        for cs in (1, 2):
            options("tc_cluster", cs)
            got = outputs()
            ops.dense_layer(g, prior, pf, pi, ins, tuple(planes), P, W, bias, out=got[0], out_planes=got[1:3],
                            w_score=wsc, dots=got[3], w_t=wt, w_h=wh)
            torch.cuda.synchronize()
            for name, a, c in zip(("h", "hi", "lo", "dots"), got, want):
                assert torch.equal(_bits(a), _bits(c)), (kind, cs, name, int((_bits(a) != _bits(c)).sum()))
            assert torch.isnan(planes[0][:, P:ops.k_order_nb0(P)].float()).all()     # the gap stays unwritten


@pytest.mark.parametrize("mode", [0, 1, 2, 3])
@pytest.mark.parametrize("B,N,E,normalized,I", [
    (16, 73, 2000, True, 2),          # 72-row tiles holding three questions' rows, edge weights
    (2, 1000, 20000, False, 2),       # hub rows past the staging capacity of every variant
    (4, 700, 5000, False, 1),
])
def test_k_order_aggregation_is_the_segment_layout_permuted(B, N, E, normalized, I, mode, options):
    D, P, R = 200, 208, 60
    b, g, (wt, wh) = _graph(B, N, E, normalized, R)
    rs = np.random.RandomState(9)
    M, T = B * N, 2 * I + 1
    pn = ops.pad_table256(_t(rs.randn(2 * (R + 1), D)))
    pf, pi = pn[: R + 1], pn[R + 1:]
    ins = _t(rs.randn(B, I, D))
    ins[0, 0, :7] = 0.0                                    # exact zeros in the instructions: exact zeros out
    prior = torch.softmax(_t(rs.randn(B, N)), 1)
    prior[0, : N // 2] = 0.0                              # rows whose in-edges all carry c == 0
    Kp = 1088 if I == 2 else 640 + 64
    dst, src = korder_index(P, I)
    options("agg_abs_ws", mode)
    sentinel = torch.from_numpy(rs.randint(-2 ** 15, 2 ** 15, size=(M, Kp)).astype(np.int16)).to(DEV).view(BF16)
    seg_planes = [sentinel.clone() for _ in range(2)]
    ko_planes = [sentinel.clone() for _ in range(2)]
    ops.aggregate_dual_abs(g, prior, pf, pi, ins, tuple(seg_planes), P, P, wt, wh)
    ops.aggregate_dual_abs(g, prior, pf, pi, ins, tuple(ko_planes), ops.k_order_nb0(P), P, wt, wh, k_order=True)
    torch.cuda.synchronize()
    end = ops.k_order_nb0(P) + 2 * I * P
    for sp, kp in zip(seg_planes, ko_planes):
        assert torch.equal(_bits(kp[:, dst]), _bits(sp[:, src]))
        assert torch.equal(_bits(kp[:, :ops.k_order_nb0(P)]), _bits(sentinel[:, :ops.k_order_nb0(P)]))
        assert torch.equal(_bits(kp[:, end:]), _bits(sentinel[:, end:]))
    assert (seg_planes[0][:, P:T * P].float() != 0).any()   # the kernel wrote something


# pitches 208 and 144: a 16-column last group; 224, 160 and 64: none.  D = 200 at the model's I <= 2
@pytest.mark.parametrize("D,I", [(200, 1), (200, 2)] + [(D, I) for D in (224, 136, 160, 50) for I in (1, 2, 3)])
@pytest.mark.parametrize("M", [1000, 20000])
def test_k_order_gemm_equals_grouped_gemm_on_permuted_planes(M, D, I, options):
    rs = np.random.RandomState(D + I)
    P, T = (D + 15) // 16 * 16, 2 * I + 1
    K = T * P
    Kp = (K + 63) // 64 * 64
    Kk = (ops.k_order_nb0(P) + 2 * I * P + 63) // 64 * 64
    A = np.zeros((M, K), np.float32)
    A.reshape(M, T, P)[:, :, :D] = rs.randn(M, T, D)
    seg_planes = [torch.full((M, Kp), NAN, dtype=BF16, device=DEV) for _ in range(2)]
    ops.split_bf16(_t(A), seg_planes[0], seg_planes[1])
    dst, src = korder_index(P, I)
    ko_planes = [torch.full((M, Kk), NAN, dtype=BF16, device=DEV) for _ in range(2)]
    for sp, kp in zip(seg_planes, ko_planes):
        kp[:, :P] = sp[:, :P]
        kp[:, dst] = sp[:, src]
    W = _t(rs.randn(D, T * D) / np.sqrt(T * D))
    bias = _t(rs.randn(D) * 0.1)
    wsc = _t(rs.randn(D))
    runs = {}
    for k_order, cs in ((False, 1), (True, 1), (True, 2)):
        options("tc_cluster", cs)
        out = torch.full((M, D), NAN, device=DEV)
        oh, ol = (torch.full((M, 256), NAN, dtype=BF16, device=DEV) for _ in range(2))
        dots = torch.full((2 * M,), NAN, device=DEV)
        pl = ko_planes if k_order else seg_planes
        ops.linear_tc_planes(pl[0], pl[1], K, W, bias, out=out, out_planes=(oh, ol), w_score=wsc, dots=dots, relu=True,
                             k_seg=D, k_seg_pitch=P, k_grouped=True, k_order=k_order)
        torch.cuda.synchronize()
        runs[(k_order, cs)] = (out, oh, ol, dots)
    assert torch.isfinite(runs[(False, 1)][0]).all()
    for key in ((True, 1), (True, 2)):
        for name, a, c in zip(("h", "hi", "lo", "dots"), runs[key], runs[(False, 1)]):
            assert torch.equal(_bits(a), _bits(c)), (key, name, int((_bits(a) != _bits(c)).sum()))
