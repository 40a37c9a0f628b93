"""GPU: the dense-prior layer as the pair gr_aggregate_dual_abs -> gr_linear_tc_planes in grouped K order
(GR_LINEAR_K_GROUPED) against gr_fused_layer, bit for bit.  Both build the same A operand and walk the same k-blocks
in the same order with the same W planes, so every output element sees the same sequence of tensor-core
accumulations: fp32 h, both output planes and the score dots must be equal as bit patterns, on NaN-prefilled outputs.

gr_aggregate_dual_abs specialises D = 200 (pitch 208), so that is the width at which the pair can be held to the fused
kernel; it is also the only width at which the model runs either.  At the other widths (a full last column group, a
half one, one and three instructions) the grouped-order GEMM is held to float64 and to the segment-order GEMM on the
same planes.  At model level the reference goldens of the hot shape run with ops.DENSE_WIDE_AS_PAIR on and off: same
pred_dist, loss, pred and ranked candidates, and both within the existing parity bounds."""
import math

import numpy as np
import pytest
import torch

from gnn_rag_b200 import batching, evaluate, ops
from gnn_rag_b200 import synthetic as S

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16 = torch.bfloat16
NAN = float("nan")


def _t(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


def _bits(x):
    return x.view(torch.int16 if x.dtype == BF16 else torch.int32)


@pytest.fixture
def cluster_option():
    yield lambda cs: ops.set_option("tc_cluster", cs)
    ops.set_option("tc_cluster", 1)


@pytest.mark.parametrize("B,N,E,normalized,I", [
    (3, 2000, 6000, False, 2),        # M = 6000: 47 tiles (fewer than SMs), the last one partial
    (5, 130, 900, True, 2),           # tiles span two questions, normalized_gnn edge weights
    (2, 1000, 20000, False, 2),       # ~2600 in-edges per tile: hub rows past the fused kernel's staging capacity
    (4, 700, 5000, False, 1),         # one instruction (T = 3)
    (32, 2000, 6000, False, 2),       # 500 tiles: several per persistent CTA
])
def test_grouped_pair_equals_fused_layer_bit_for_bit(B, N, E, normalized, I, cluster_option):
    D, P, R = 200, 208, 60
    b = S.make_batch(17, B=B, N=N, E=E, num_entity=5000, num_relation=R, num_word=50, n_real="ragged", powerlaw=True)
    g = batching.stage_batch(b, torch.device(DEV), R + 1, normalized, False).graph
    wt, wh = (g.w_t, g.w_h) if normalized else (None, None)
    assert ops.fused_layer_supported(N, D, P, I, D)
    rs = np.random.RandomState(5)
    M, T = B * N, 2 * I + 1
    tiles = math.ceil(M / 128)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert (tiles < sms) if B <= 5 else (tiles >= 3 * sms)
    pn = ops.pad_table256(_t(rs.randn(2 * (R + 1), D)))
    pf, pi = pn[: R + 1], pn[R + 1:]
    ins = _t(rs.randn(B, I, D))
    h = _t(rs.randn(M, D))
    Kp = (T * P + 63) // 64 * 64
    planes = [torch.zeros(M, Kp, dtype=BF16, device=DEV) for _ in range(2)]
    ops.split_bf16(h, planes[0], planes[1])
    for p in planes:
        p[:, P:] = NAN                       # the neighbour segments are written by the aggregation, the tail never read
    h_hi, h_lo = (p[:, :256].clone() for p in planes)                    # the fused kernel's input: h, NaN beyond the pitch
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
        assert (want[3][M:] == 0).all()
        for cs in (1, 2):
            cluster_option(cs)
            got = outputs()
            ops.aggregate_dual_abs(g, prior, pf, pi, ins, tuple(planes), P, P, wt, wh)
            ops.linear_tc_planes(planes[0], planes[1], T * P, W, bias, out=got[0], out_planes=got[1:3], w_score=wsc,
                                 dots=got[3], relu=True, k_seg=D, k_seg_pitch=P, k_grouped=True)
            torch.cuda.synchronize()
            for name, a, c in zip(("h", "hi", "lo", "dots"), got, want):
                assert torch.equal(_bits(a), _bits(c)), (kind, cs, name, int((_bits(a) != _bits(c)).sum()))
            assert torch.equal(_bits(got[3][:M]), _bits(want[3][:M])) and torch.equal(got[3][M:], want[3][M:])
        # the segment-order GEMM on the same planes is the same sum in another order: close, and not the yardstick
        seg = torch.empty(M, D, device=DEV)
        ops.linear_tc_planes(planes[0], planes[1], T * P, W, bias, out=seg, relu=True, k_seg=D, k_seg_pitch=P)
        assert (seg - want[0]).abs().max().item() <= 2e-5 * want[0].abs().max().item()


@pytest.mark.parametrize("I", [1, 3])
@pytest.mark.parametrize("D", [224, 136, 160, 50])    # pitches 224 and 160: full last group; 144 and 64: 16-column last group / two groups
@pytest.mark.parametrize("M", [1000, 20000])          # a partial last tile; more tiles than SMs
def test_grouped_gemm_vs_fp64_and_segment_order(M, D, I, cluster_option):
    rs = np.random.RandomState(D + I)
    P, T = (D + 15) // 16 * 16, 2 * I + 1
    K = T * P
    Kp = (K + 63) // 64 * 64
    A = np.zeros((M, K), np.float32)
    A.reshape(M, T, P)[:, :, :D] = rs.randn(M, T, D)
    planes = [torch.full((M, Kp), NAN, dtype=BF16, device=DEV) for _ in range(2)]
    ops.split_bf16(_t(A), planes[0], planes[1])
    W = _t(rs.randn(D, T * D) / np.sqrt(T * D))
    bias = _t(rs.randn(D) * 0.1)
    wsc = _t(rs.randn(D))
    a64 = (planes[0][:, :K].double() + planes[1][:, :K].double()).view(M, T, P)[:, :, :D].reshape(M, T * D)
    want = torch.relu(a64 @ W.double().t() + bias.double())
    scale = (a64.abs() @ W.double().abs().t() + bias.double().abs()).max().item()
    runs = {}
    for grouped, cs in ((True, 1), (True, 2), (False, 1)):
        cluster_option(cs)
        out = torch.full((M, D), NAN, device=DEV)
        dots = torch.full((2 * M,), NAN, device=DEV)
        ops.linear_tc_planes(planes[0], planes[1], K, W, bias, out=out, w_score=wsc, dots=dots, relu=True, k_seg=D,
                             k_seg_pitch=P, k_grouped=grouped)
        torch.cuda.synchronize()
        assert (out.double() - want).abs().max().item() <= 2e-5 * scale, (grouped, cs)
        d64 = want @ wsc.double()
        assert (dots[:M].double() + dots[M:].double() - d64).abs().max().item() <= 1e-4 * scale * wsc.abs().sum().item()
        runs[(grouped, cs)] = (out, dots)
    for a, c in zip(runs[(True, 1)], runs[(True, 2)]):
        assert torch.equal(_bits(a), _bits(c))               # the cluster size does not enter the accumulation order


def test_grouped_flag_is_refused_where_the_k_map_does_not_apply():
    M, D, P = 256, 200, 208
    hi = torch.zeros(M, 4 * P, dtype=BF16, device=DEV)
    out = torch.empty(M, D, device=DEV)
    with pytest.raises(Exception, match="odd number of segments"):
        ops.linear_tc_planes(hi, hi, 4 * P, torch.zeros(D, 4 * D, device=DEV), None, out=out, k_seg=D, k_seg_pitch=P,
                             k_grouped=True)
    ops.set_option("tc_bk", 64)
    try:
        with pytest.raises(Exception, match="32-column k-blocks"):
            ops.linear_tc_planes(hi, hi, 3 * P, torch.zeros(D, 3 * D, device=DEV), None, out=out, k_seg=D,
                                 k_seg_pitch=P, k_grouped=True)
    finally:
        ops.set_option("tc_bk", 32)


@pytest.mark.parametrize("name", ["cfg2_full", "d200_rand", "d200_sharp", "d200_norm"])
def test_model_same_results_with_the_pair_and_with_the_fused_kernel(name):
    from test_hot_goldens_gpu import Hot, _check_dist
    import rank_check
    h = Hot(name)
    m = h.model()
    full = name == "cfg2_full"
    # d200_rand and d200_norm have fewer than 128 nodes per question: neither form of the dense layer takes them
    dense = ops.fused_layer_supported(h.batch[0].shape[1], 200, 208, h.args["num_ins"], 200)
    assert dense or name in ("d200_rand", "d200_norm")
    res = {}
    min_rows = ops.FUSED_MIN_ROWS
    ops.FUSED_MIN_ROWS = 0                                   # the d200 goldens are smaller than one tile per SM
    try:
        for pair in (True, False):
            ops.DENSE_WIDE_AS_PAIR = pair
            ops.STATS.reset()
            ops.STATS.time_ops = True
            try:
                loss, pred, dist, _ = m(h.batch[:7])
                torch.cuda.synchronize()
            finally:
                ops.STATS.time_ops = False
            classes = {e[2] for e in ops.STATS.op_events}
            assert ("fused_layer" in classes) == (dense and not pair)   # the switch selects the kernels that run
            rel = _check_dist(dist, h.out["pred_dist"], "%s pair=%d" % (name, pair), logits=full)
            assert abs(float(loss) - float(h.out["loss"])) < 1e-3 * max(1.0, abs(float(h.out["loss"])))
            got, _ = evaluate.retrieve(dist, m.last_batch, h.vocab["num_entity"], h.args["eps"])
            rank_check.report("hot/%s pair=%d" % (name, pair),
                              rank_check.compare(got, h.ref_lists(), h.out["pred_dist"],
                                                 **({"margin": max(2e-5, 2 * rel)} if full else {})))
            res[pair] = (dist.clone(), loss.clone(), pred.clone(), [(r.ent.tolist(), r.prob.tolist()) for r in got])
    finally:
        ops.DENSE_WIDE_AS_PAIR = True
        ops.FUSED_MIN_ROWS = min_rows
        ops.STATS.reset()
    for a, c in zip(res[True][:3], res[False][:3]):
        assert torch.equal(a, c)
    assert res[True][3] == res[False][3]                     # ranked candidate lists: same ids in the same order
