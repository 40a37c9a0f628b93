"""CPU: the restatements of tests/retrieval_ref.py pinned to the oracle, to networkx and to the training path's own
host metrics; the host-side candidate cut of training (autograd_path._retrieved_sets_host) against the reference's cut
at the (1-eps)/N boundary and for eps >= 1; the torch behaviour that cut depends on; the construction the GPU tests use
to separate the ranking kernel's parallel scan from its sequential loop; and the shape rule and refusals of
ops.rank_candidates / gr_rank_candidates."""
import math

import networkx as nx
import numpy as np
import pytest
import torch

from gnn_rag_b200 import autograd_path, ops
from oracle import kgqa_oracle as O
import retrieval_ref as R
import test_graphed_train_host as HT
from test_entry_refusals_host import INVALID, WORKSPACE, call

f32 = np.float32


def _random_rank_case(rs, B, N, eps):
    pad = 50
    le = rs.randint(0, 60, size=(B, N))
    le[rs.rand(B, N) < 0.15] = pad
    qe = rs.choice(np.array([0.0, 0.0, 0.0, 1.0, 1.5, 0.5, 2.0, -1.0], f32), size=(B, N))
    p = rs.choice(np.array([0.0, -0.0, 1e-45, -1e-3, 0.25, 0.25, 0.125], f32), size=(B, N))
    p = np.where(rs.rand(B, N) < 0.5, (rs.rand(B, N) / N).astype(f32), p).astype(f32)
    return le, qe, p, pad


# ---- the ranking restatement ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("eps", [0.5, 0.95, 1.0, 1.5])
def test_rank_matches_the_oracle(eps):
    rs = np.random.RandomState(int(eps * 100))
    for N in (1, 7, 130):
        le, qe, p, pad = _random_rank_case(rs, 6, N, eps)
        want = O.rank_candidates(le, qe.astype(np.float64), p, pad, eps)
        got = R.rank(le, qe, p, pad, eps)
        assert got == want
        assert [cand[:cut] for cand, cut in R.rank_full(le, qe, p, pad, eps)] == got


def test_rank_keeps_python_sorted_order_for_signed_zeros_and_negatives():
    p = np.array([[0.0, -0.0, -0.5, 0.25, -0.0, 0.0, -1e-45, 1e-45]], f32)
    got = R.rank_full(np.arange(8)[None], np.zeros((1, 8)), p, -1, 1.5)[0][0]
    assert [n for n, _, _ in got] == [3, 7, 0, 1, 4, 5, 6]      # -0.5 < (1 - 1.5) / 8


# ---- the exactness construction of the GPU tests ------------------------------------------------------------------------

def _kernel_scan_count(values, eps):
    """rank_kernel's parallel eps-mass cut, emulated in float64: an inclusive Hillis-Steele scan per 32-lane warp, the
    preceding warps' sums added in order onto the carry of the previous 512-item chunk."""
    total = len(values)
    carry = 0.0
    for base in range(0, total, 512):
        v = [values[i] if i < total else 0.0 for i in range(base, base + 512)]
        x = list(v)
        for o in (1, 2, 4, 8, 16):
            x = [x[t] + x[t - o] if t % 32 >= o else x[t] for t in range(512)]
        wsum = [x[w * 32 + 31] for w in range(16)]
        cums = []
        for t in range(512):
            off = carry
            for w in range(t // 32):
                off += wsum[w]
            cums.append(off + x[t])
        for t in range(512):
            if base + t < total and cums[t] > eps:
                return base + t + 1
        carry = cums[511]
    return total


def _sequential_count(values, eps):
    tp = 0.0
    for i, v in enumerate(values):
        tp += v
        if tp > eps:
            return i + 1
    return len(values)


def test_the_scan_and_the_sequential_sum_differ_only_past_53_bits():
    """eps = 1 - 2^-40, N = 16 384: (1-eps)/N = 2^-54 and the host's bound is 79 bits.  2^-1 .. 2^-40 sum exactly to
    eps; three more terms of 2^-54 are each a half-ulp tie of the running sum, so the sequential sum never exceeds eps
    (all 43 kept), while the second warp pairs two of them into 2^-53 and crosses at the 42nd.  At 53 bits
    (eps = 1 - 2^-18, N = 1024) the same construction gives the same count either way."""
    for k, m, bits, seq, par in [(40, 14, 79, 43, 42), (18, 10, 53, 19, 19)]:
        eps, N = 1 - 2.0 ** -k, 2 ** m
        ip = (1 - eps) / N
        assert ip == 2.0 ** -(k + m) and 24 + (1 - math.frexp(ip)[1]) + 1 == bits
        vals = [2.0 ** -i for i in range(1, k + 1)] + [ip] * 3
        assert all(float(f32(v)) == v for v in vals)
        assert (_sequential_count(vals, eps), _kernel_scan_count(vals, eps)) == (seq, par)
        p = np.zeros((1, N), f32)
        p[0, :len(vals)] = vals
        assert R.rank_full(np.arange(N)[None], np.zeros((1, N)), p, -1, eps)[0][1] == seq


# ---- the host-side cut of training ------------------------------------------------------------------------------------

def _host_cut(p, le, qe, pad, eps):
    t = torch.from_numpy
    order, count = autograd_path._retrieved_sets_host(t(np.asarray(p, f32)), t(np.asarray(le, np.int64)),
                                                      (t(np.asarray(qe, f32)) > 0).float(), pad, eps)
    return [order[b, :int(c)].tolist() for b, c in enumerate(count.tolist())]


def _ref_cut(p, le, qe, pad, eps):
    return [[n for n, _, _ in r] for r in R.rank(le, (np.asarray(qe) > 0).astype(f32), p, pad, eps)]


def test_torch_rounds_the_python_bound_to_fp32():
    """What the host cut has to work around: an fp32 tensor compared with a Python float compares in fp32.  At
    eps = 0.95, N = 2000 the bound 2.500000000000002e-05 rounds down to an fp32 value below it, which such a compare
    keeps and the reference's float64 compare drops; the hit threshold 1e-10 likewise rounds to fp32."""
    ip = (1 - 0.95) / 2000
    lo = f32(ip)
    assert float(lo) < ip
    assert bool((torch.tensor([lo]) >= ip).item()) and not float(lo) >= ip
    assert bool((torch.tensor([lo]).double() < ip).item())
    th = f32(1e-10)
    assert float(th) > 1e-10 and not bool((torch.tensor([th]) > 1e-10).item())


def test_host_cut_at_the_ignore_prob_boundary():
    N = 2000
    ip = (1 - 0.95) / N
    rs = np.random.RandomState(0)
    p = np.zeros((3, N), f32)
    p[:, :50] = ((0.5 + rs.rand(3, 50)) * 0.015).astype(f32)
    p[0, 300:310] = f32(ip)                                   # below the float64 bound: dropped
    p[1, 300:310] = np.nextafter(f32(ip), f32(1))             # above it: kept
    p[2, 300:310] = np.nextafter(f32(ip), f32(0))
    le = np.arange(3 * N).reshape(3, N)
    qe = np.zeros((3, N), f32)
    want = _ref_cut(p, le, qe, -1, 0.95)
    assert _host_cut(p, le, qe, -1, 0.95) == want
    assert [300 in w for w in want] == [False, True, False]


@pytest.mark.parametrize("eps", [0.5, 0.95, 1.0, 1.5])
def test_host_cut_matches_the_reference_cut(eps):
    rs = np.random.RandomState(3)
    for N in (1, 9, 257):
        le, qe, p, pad = _random_rank_case(rs, 8, N, eps)
        assert _host_cut(p, le, qe, pad, eps) == _ref_cut(p, le, qe, pad, eps)


# ---- the train-time metrics restatement -------------------------------------------------------------------------------

def _metrics_np_on_ref_cut(pd, ad, sd, le, pad, eps):
    B, N = pd.shape
    cand_idx = np.zeros((B, N), np.int64)
    cand_count = np.zeros(B, np.int64)
    for b, r in enumerate(R.rank(le, (sd > 0).astype(f32), pd, pad, eps)):
        cand_idx[b, :len(r)] = [n for n, _, _ in r]
        cand_count[b] = len(r)
    return HT.metrics_np(pd, ad, sd, le, cand_idx, cand_count, pad)


def _check_metrics(pd, ad, sd, le, pad, eps=0.95):
    h1, f1 = R.train_metrics(pd, ad, sd, le, pad, eps)
    h1n, f1n = _metrics_np_on_ref_cut(pd, ad, sd, le, pad, eps)
    assert h1.tobytes() == h1n.tobytes() and f1.tobytes() == f1n.tobytes(), (h1, h1n, f1, f1n)
    t = torch.from_numpy
    h1e, f1e = autograd_path.eval_metric(type("M", (), dict(num_entity=pad, eps=eps)), t(pd), t(ad), t(sd),
                                         t(le.astype(np.int64)))
    assert h1e.numpy().tobytes() == h1.tobytes() and f1e.numpy().tobytes() == f1.tobytes()
    return h1.tolist(), f1.tolist()


def test_train_metrics_on_the_edge_batch():
    pd, ad, sd, le, pad = HT.edge_batch()
    h1, f1 = _check_metrics(pd, ad, sd, le, pad)
    assert h1 == HT.EDGE_H1
    assert f1[1] == 0.0 and f1[2] == 1.0 and f1[3] == 0.0 and f1[6] == 1.0
    for b in range(len(h1)):
        _check_metrics(pd[b:b + 1], ad[b:b + 1], sd[b:b + 1], le[b:b + 1], pad)


@pytest.mark.parametrize("seed", [0, 1])
def test_train_metrics_on_random_batches(seed):
    rs = np.random.RandomState(seed)
    B, N, pad = 16, 120, 500
    le = rs.randint(0, 60, size=(B, N)).astype(np.int64)
    le[rs.rand(B, N) < 0.2] = pad
    sd = (rs.rand(B, N) < 0.03).astype(f32)
    ad = ((rs.rand(B, N) < 0.1) * rs.rand(B, N)).astype(f32)
    logits = rs.randn(B, N) * 2 + 3 * (ad > 0)
    pd = np.exp(logits - logits.max(1, keepdims=True))
    h1, _ = _check_metrics((pd / pd.sum(1, keepdims=True)).astype(f32), ad, sd, le, pad)
    assert 0 < sum(h1)


def test_train_metrics_hit_threshold_and_nan():
    th = f32(1e-10)
    pd = np.full((4, 6), 0.1, f32)
    pd[:, 2] = 0.5
    ad = np.zeros((4, 6), f32)
    ad[:3, 2] = [th, np.nextafter(th, f32(1)), 1.0]
    pd[2, 4] = np.nan                                         # the NaN is the top-1, with no answer mass
    pd[3, 1] = np.nan
    ad[3, 1] = 1.0                                            # ... with answer mass
    h1, _ = R.train_metrics(pd, ad, np.zeros((4, 6), f32), np.arange(24).reshape(4, 6), -1, 0.95)
    assert h1.tolist() == [0.0, 1.0, 0.0, 1.0]


# ---- the shortest-path restatement -------------------------------------------------------------------------------------

def _nx_path_nodes(heads, tails, N, sources, targets):
    g = nx.Graph()
    g.add_nodes_from(range(N))
    g.add_edges_from(zip(heads, tails))
    nodes, pair = set(), np.full((len(sources), len(targets)), -1, np.int32)
    for i, s in enumerate(sources):
        for j, t in enumerate(targets):
            if nx.has_path(g, s, t):
                pair[i, j] = nx.shortest_path_length(g, s, t)
                for path in nx.all_shortest_paths(g, s, t):
                    nodes.update(path)
    return pair, sorted(nodes)


@pytest.mark.parametrize("seed", range(6))
def test_path_nodes_match_the_oracle_and_networkx(seed):
    rs = np.random.RandomState(seed)
    N = int(rs.randint(1, 40))
    E = int(rs.randint(0, 2 * N))
    heads = rs.randint(0, N, size=E).tolist() + [0]           # a self-loop; repeats give parallel edges
    tails = rs.randint(0, N, size=E).tolist() + [0]
    sources = rs.randint(0, N, size=int(rs.randint(1, 4))).tolist()
    targets = rs.randint(0, N, size=int(rs.randint(1, 6))).tolist() + sources[:1]
    ds, dt, pair, nodes = R.path_nodes(heads, tails, N, sources, targets)
    want_nodes, want_pd = O.shortest_path_nodes(heads, tails, N, sources, targets)
    assert nodes == want_nodes
    assert pair.tolist() == [[want_pd.get((s, t), -1) for t in targets] for s in sources]
    nx_pair, nx_nodes = _nx_path_nodes(heads, tails, N, sources, targets)
    assert nodes == nx_nodes and np.array_equal(pair, nx_pair)
    g = nx.Graph()
    g.add_nodes_from(range(N))
    g.add_edges_from(zip(heads, tails))
    for roots, d in ((sources, ds), (targets, dt)):
        for r, row in zip(roots, d):
            lengths = nx.single_source_shortest_path_length(g, r)
            assert row.tolist() == [lengths.get(v, -1) for v in range(N)]


# ---- ops.rank_candidates / gr_rank_candidates refusals -----------------------------------------------------------------

RANK = dict(pad_id=7, eps=0.95, B=2, N=3, workspace_bytes=48, stream=None)


@pytest.mark.parametrize("over,status,msg", [
    (dict(dist=None), INVALID, "invalid argument: null pointer"),
    (dict(cand_total=None), INVALID, "invalid argument: null pointer"),
    (dict(B=0), INVALID, "invalid argument: bad shape"),
    (dict(N=0), INVALID, "invalid argument: bad shape"),
    (dict(N=-1), INVALID, "invalid argument: bad shape"),
    (dict(workspace_bytes=47), WORKSPACE, "workspace too small"),
    (dict(workspace=None), WORKSPACE, "workspace too small")])
def test_entry_point_refusals(over, status, msg):
    assert call("gr_rank_candidates", dict(RANK, **over)) == (status, "gr_rank_candidates: " + msg)


def test_shape_rule():
    for B, N in [(1, 1), (0, 3), (2, 0), (64, 2000)]:
        assert ops.rank_candidates_ok(B, N) == (B > 0 and N > 0)


@pytest.mark.parametrize("dist,le,qe", [
    ((2, 3), (2, 4), (2, 3)), ((2, 3), (2, 3), (3, 3)), ((2, 3), (6,), (2, 3)), ((6,), (6,), (6,)),
    ((0, 3), (0, 3), (0, 3)), ((2, 0), (2, 0), (2, 0)), ((2, 3, 1), (2, 3, 1), (2, 3, 1))])
def test_wrapper_refuses_mismatched_shapes(dist, le, qe):
    with pytest.raises(RuntimeError, match="rank_candidates: .* must be"):
        ops.rank_candidates(torch.zeros(dist), torch.zeros(le, dtype=torch.int64), torch.zeros(qe), 7, 0.95)


def test_wrapper_refuses_cpu_tensors():
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.rank_candidates(torch.zeros(2, 3), torch.zeros(2, 3, dtype=torch.int64), torch.zeros(2, 3), 7, 0.95)
