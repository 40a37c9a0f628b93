"""The kernels that produce the retrieval output, held bit for bit to the exact restatements of tests/retrieval_ref.py at
their edge shapes: gr_rank_candidates (csrc/rank.cu: the ordered candidate lists and the eps-mass cut),
gr_train_metrics (the train-time hit@1 and F1, now against a restatement with its own cut rather than the ranking
kernel) and gr_shortest_path_nodes (csrc/paths.cu: the seed -> candidate path node sets and hop distances).

Every case compares the whole output: the ranking's ordered indices, counts and totals with the zero fill past the
total; h1 and f1 as bytes; on_path, pair_dist with its -1 fill past the counts, and the BFS distance arrays."""
import math

import numpy as np
import pytest
import torch

from gnn_rag_b200 import batching, evaluate, ops, synthetic as S
from golden_io import Golden
import retrieval_ref as R
import test_training_path as TP

pytestmark = pytest.mark.gpu
DEV = "cuda"
f32 = np.float32


def _t(a, dtype):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, dtype)


# ---- gr_rank_candidates -----------------------------------------------------------------------------------------------

def check_rank(p, le, qe, pad, eps):
    """Rank on the device and compare everything with retrieval_ref.rank_full; returns the reference's
    [(survivors in order, cut), ...]."""
    p, le, qe = np.asarray(p, f32), np.asarray(le, np.int64), np.asarray(qe, f32)
    ci, cc, ct = ops.rank_candidates(_t(p, torch.float32), _t(le, torch.int64), _t(qe, torch.float32), pad, eps)
    ci, cc, ct = ci.cpu().numpy(), cc.cpu().numpy(), ct.cpu().numpy()
    want = R.rank_full(le, qe, p, pad, eps)
    for b, (cand, cut) in enumerate(want):
        total = len(cand)
        assert (int(ct[b]), int(cc[b])) == (total, cut), (b, "total, count", int(ct[b]), int(cc[b]), total, cut)
        assert ci[b, :total].tolist() == [n for n, _, _ in cand], b
        assert not ci[b, total:].any(), b                       # the documented zero fill past cand_total
    return want


def _question(rs, N, n_surv, eps, pad, mass=None, levels=None):
    """One question of N nodes of which exactly n_surv survive the seed / pad / (1-eps)/N filters, placed at random
    local indices.  The survivors' probabilities are (1 + U)/N, or one of ``levels`` distinct values (many exact ties),
    scaled to total ``mass``; the others are seeds and pads with large p, and nodes just below (1-eps)/N."""
    p = np.zeros(N, f32)
    le = rs.randint(0, pad, size=N).astype(np.int64)
    qe = np.zeros(N, f32)
    perm = rs.permutation(N)
    surv, rest = perm[:n_surv], perm[n_surv:]
    v = (1.0 + (rs.randint(0, levels, size=n_surv) / levels if levels else rs.rand(n_surv))) / N
    if mass is not None and n_surv:
        v = v * (mass / v.sum())
    p[surv] = v.astype(f32)
    ip = (1 - eps) / N
    assert n_surv == 0 or float(p[surv].min()) >= ip
    k = len(rest)
    seeds, pads, small = rest[: k // 3], rest[k // 3: 2 * k // 3], rest[2 * k // 3:]
    qe[seeds] = 1.0
    p[seeds] = 0.5
    le[pads] = pad
    p[pads] = 0.5
    p[small] = np.nextafter(f32(ip), f32(0)) if float(f32(ip)) >= ip else f32(ip)
    return p, le, qe


@pytest.mark.parametrize("n_surv", [0, 1, 31, 511, 512, 513, 4095, 4096, 4097, 9000])
def test_rank_survivor_counts(n_surv):
    """Around the warp, the 512-thread chunk and the 4096-key shared-memory sort boundaries: a cut inside the list, a
    list whose mass never reaches eps, and a list of exact ties."""
    rs = np.random.RandomState(n_surv)
    N, eps, pad = n_surv + 300, 0.9, 10 ** 6
    rows = [_question(rs, N, n_surv, eps, pad, mass=1.0), _question(rs, N, n_surv, eps, pad, mass=0.5),
            _question(rs, N, n_surv, eps, pad, levels=5)]
    want = check_rank(*(np.stack(x) for x in zip(*rows)), pad, eps)
    assert [len(c) for c, _ in want] == [n_surv] * 3
    if n_surv > 1:
        assert want[0][1] < n_surv and want[1][1] == n_surv


def test_rank_single_node_questions():
    p = np.array([[1.0], [1.0], [1.0], [0.01]], f32)
    le = np.array([[3], [3], [9], [3]])
    qe = np.array([[0.0], [1.0], [0.0], [0.0]], f32)
    want = check_rank(p, le, qe, 9, 0.95)                     # kept, seed, pad, below (1-eps)/N
    assert [c for _, c in want] == [1, 0, 0, 0]


def test_rank_real_shape_and_cfg5_question():
    """B = 64, N = 2000 (cfg2) with seeds and pads, and one question of N = 100 000 (cfg5) through the global sort."""
    rs = np.random.RandomState(1)
    B, N, pad = 64, 2000, S.WEBQSP_NUM_ENTITY
    logits = rs.randn(B, N) * rs.choice([0.3, 1.0, 3.0, 8.0], size=(B, 1))
    p = np.exp(logits - logits.max(1, keepdims=True))
    p = (p / p.sum(1, keepdims=True)).astype(f32)
    le = rs.randint(0, pad, size=(B, N))
    le[:, 1500:] = pad
    p[:, 1500:] = 0.0
    qe = np.zeros((B, N), f32)
    qe[np.arange(B), rs.randint(0, 1500, size=B)] = 1.0
    check_rank(p, le, qe, pad, 0.95)
    N = 100_000
    p = np.exp(rs.randn(1, N) * 2.0)
    p = (p / p.sum()).astype(f32)
    p[0, ::11] = p[0, 5]                                      # exact ties all along the list
    want = check_rank(p, rs.randint(0, pad, size=(1, N)), np.zeros((1, N), f32), pad, 0.95)
    assert len(want[0][0]) > 50_000


@pytest.mark.parametrize("where", ["first_chunk", "later_chunk", "tie", "last_survivor", "never"])
def test_rank_cut_position(where):
    """eps set to an exact prefix sum of the sorted survivors, so the cut falls where wanted: in the first 512-item
    chunk, in a later one (the scan's carry between chunks), on an item tied with the next (the stable index order
    decides who is in), on the last survivor, and never."""
    rs = np.random.RandomState(7)
    N, pad = 1500, 10 ** 6
    n_surv = 600 if where in ("last_survivor", "never") else 1200
    p, le, qe = _question(rs, N, n_surv, 0.999, pad, levels=64)      # survivors >= 1/N, the small ones < 0.001/N
    order = R.rank_full(le[None], qe[None], p[None], pad, 0.999)[0][0]
    probs = [x[2] for x in order]
    k = dict(first_chunk=100, later_chunk=700, tie=None, last_survivor=n_surv - 1, never=None)[where]
    if where == "tie":
        k = next(i for i in range(300, n_surv - 1) if probs[i] == probs[i + 1] and probs[i - 1] != probs[i])
    eps = 0.0
    for x in probs[:k] if k is not None else probs:
        eps += x
    assert 0.0 < eps < 1.0
    want = check_rank(p[None], le[None], qe[None], pad, eps)
    assert want[0][1] == (k + 1 if k is not None else n_surv)
    if where == "tie":                                        # the tied pair straddles the cut, in local-index order
        assert order[k][0] < order[k + 1][0]


def test_rank_ignore_prob_boundary():
    """p exactly at (1-eps)/N where that is an fp32 value (eps = 0.5, N = 1024: kept, the float below is not), and at
    its fp32 neighbours where it is not (eps = 0.95, N = 2000: the float64 compare drops the lower one)."""
    rs = np.random.RandomState(3)
    N = 1024
    ip = (1 - 0.5) / N
    assert float(f32(ip)) == ip
    p = np.full((2, N), 0.0, f32)
    p[:, :40] = ((0.5 + rs.rand(2, 40)) * 0.01).astype(f32)
    p[0, 100:120] = f32(ip)
    p[1, 100:120] = np.nextafter(f32(ip), f32(0))
    want = check_rank(p, np.arange(2 * N).reshape(2, N), np.zeros((2, N), f32), -1, 0.5)
    assert [len(c) for c, _ in want] == [60, 40]
    N = 2000
    ip = (1 - 0.95) / N
    lo = f32(ip)
    assert float(lo) < ip
    hi = np.nextafter(lo, f32(1))
    p = np.full((2, N), 0.0, f32)
    p[:, :30] = ((0.5 + rs.rand(2, 30)) * 0.02).astype(f32)
    p[0, 500:510] = lo
    p[1, 500:510] = hi
    want = check_rank(p, np.arange(2 * N).reshape(2, N), np.zeros((2, N), f32), -1, 0.95)
    assert [len(c) for c, _ in want] == [30, 40]


def test_rank_seed_values_and_pads():
    """The seed test is int(s) == 1 (the reference's LongTensor cast): 1.0 and 1.5 are seeds, 0.5, 2.0, -1.0 and 0.0
    are not.  Pads, an all-pad question and an all-seed question."""
    rs = np.random.RandomState(4)
    B, N, pad = 4, 600, 777
    p = rs.rand(B, N).astype(f32) / N * 2
    le = rs.randint(0, 700, size=(B, N))
    qe = rs.choice(np.array([1.0, 1.5, 0.5, 2.0, -1.0, 0.0], f32), size=(B, N))
    le[:2, ::5] = pad
    le[2] = pad
    qe[3] = rs.choice(np.array([1.0, 1.5], f32), size=N)
    want = check_rank(p, le, qe, pad, 0.95)
    assert len(want[0][0]) > 0 and len(want[2][0]) == 0 and len(want[3][0]) == 0


def test_rank_ties_across_the_shared_memory_boundary():
    rs = np.random.RandomState(5)
    N, pad = 6000, 10 ** 6
    rows = [_question(rs, N, n, 0.95, pad, levels=3) for n in (4090, 4100, 5500)]
    check_rank(*(np.stack(x) for x in zip(*rows)), pad, 0.95)


def _bits(eps, N):
    """The host's exactness bound (gr_rank_candidates): bits of a partial sum of fp32 terms >= (1-eps)/N."""
    return 24 + (1 - math.frexp((1 - eps) / N)[1]) + 1


@pytest.mark.parametrize("k,m,bits", [(18, 10, 53), (19, 10, 54), (40, 14, 79)])
def test_rank_exactness_boundary(k, m, bits):
    """eps = 1 - 2^-k, N = 2^m, so (1-eps)/N = 2^-(k+m): the parallel fp64 scan at bits = 53, the sequential loop past
    it.  The terms 2^-1 .. 2^-k sum exactly to eps; then terms equal to (1-eps)/N, then full-mantissa fp32 values.
    At k = 40 the tiny terms are half-ulp ties of the running sum: added in order each one rounds away and all are
    kept, while a warp's tree would pair them first and cross eps one item early."""
    eps, N = 1 - 2.0 ** -k, 2 ** m
    assert _bits(eps, N) == bits
    ip = 2.0 ** -(k + m)
    p = np.zeros((1, N), f32)
    p[0, :k] = 2.0 ** -np.arange(1, k + 1)
    p[0, k:k + 3] = ip
    if bits < 79:
        rs = np.random.RandomState(k)
        p[0, 100:140] = (ip * (1 + rs.rand(40)) * 2 ** rs.randint(0, 8, 40)).astype(f32)
    want = check_rank(p, np.arange(N)[None], np.zeros((1, N), f32), -1, eps)
    if bits == 79:
        assert (len(want[0][0]), want[0][1]) == (k + 3, k + 3)


@pytest.mark.parametrize("eps", [1.0, 1.5])
def test_rank_sequential_fallback_signed_zeros_negatives_subnormals(eps):
    """eps >= 1: (1-eps)/N <= 0, so zeros, -0.0, subnormals and (for eps > 1) small negative values survive and the
    order is the whole output.  -0.0 ranks level with +0.0 in index order, negative values below them."""
    rs = np.random.RandomState(6)
    N = 64
    sub = np.array([1e-45, 3e-42, 1e-39], f32)
    vals = np.concatenate([np.array([0.0, -0.0, 0.0, -0.0, -1e-3, -1e-5, -0.25, -1e-45, 2.0, 0.75, 0.75], f32), sub,
                           -sub, (rs.rand(N - 17) * 0.1).astype(f32)])
    assert len(vals) == N
    p = np.stack([rs.permutation(vals), rs.permutation(vals), np.where(vals > 0.5, f32(0.1), vals)]).astype(f32)
    want = check_rank(p, np.arange(3 * N).reshape(3, N), np.zeros((3, N), f32), -1, eps)
    assert all(len(c) > N // 2 for c, _ in want)
    neg = [x for c, _ in want for x in c if x[2] < 0]
    assert bool(neg) == (eps > 1.0)


def test_rank_kept_probability_above_one():
    """A kept p > 1 takes the sequential loop; with eps < 1 the first item crosses."""
    p = np.array([[0.2, 3.0, 0.1, 1.5, 0.3], [0.2, 0.4, 1.0000001, 0.1, 0.0]], f32)
    want = check_rank(p, np.arange(10).reshape(2, 5), np.zeros((2, 5), f32), -1, 0.95)
    assert [c for _, c in want] == [1, 1]


# ---- gr_train_metrics -------------------------------------------------------------------------------------------------

def check_metrics(pd, ad, sd, le, pad, eps=0.95, f1_rows=None):
    """h1 and f1 of the device (ranking + metrics kernels) against retrieval_ref.train_metrics, as bytes; f1 only on
    ``f1_rows`` when given.  Returns the reference's (h1, f1)."""
    pd, ad, sd, le = np.asarray(pd, f32), np.asarray(ad, f32), np.asarray(sd, f32), np.asarray(le, np.int64)
    pd_t, ad_t, sd_t, le_t = _t(pd, torch.float32), _t(ad, torch.float32), _t(sd, torch.float32), _t(le, torch.int64)
    ci, cc, _ = ops.rank_candidates(pd_t, le_t, (sd_t > 0).float(), pad, eps)
    h1, f1 = ops.train_metrics(pd_t, ad_t, sd_t, le_t, ci, cc, pad)
    h1w, f1w = R.train_metrics(pd, ad, sd, le, pad, eps)
    assert h1.cpu().numpy().tobytes() == h1w.tobytes(), (h1.cpu().numpy(), h1w)
    rows = slice(None) if f1_rows is None else f1_rows
    assert f1.cpu().numpy()[rows].tobytes() == f1w[rows].tobytes(), (f1.cpu().numpy()[rows], f1w[rows])
    return h1w, f1w


@pytest.mark.parametrize("name", TP.CASES)
def test_train_metrics_on_the_goldens(name):
    g = Golden(name)
    t = np.load(TP.os.path.join(TP.GOLDEN_DIR, "train", name + ".npz"))
    b = g.batch
    h1, _ = check_metrics(t["pred_dist"], t["answer_dist"], b[4], b[0], g.num_entity, g.args["eps"])
    assert h1.tolist() == t["h1"].tolist()


def test_train_metrics_on_a_cfg2_sized_batch():
    c = S.CONFIGS["cfg2"]
    rs = np.random.RandomState(0)
    b = S.make_batch(1, B=c["B"], N=c["N"], E=c["E"], with_weights=False, multi_seed=True)
    ans = np.asarray(b[6], dtype=f32)
    logits = rs.randn(c["B"], c["N"]) * rs.choice([0.3, 3.0], size=(c["B"], 1)) + 4.0 * (ans > 0)
    pd = np.exp(logits - logits.max(1, keepdims=True))
    h1, f1 = check_metrics(pd / pd.sum(1, keepdims=True), ans, b[4], b[0], S.WEBQSP_NUM_ENTITY)
    assert h1.sum() > 0 and f1.sum() > 0


def test_train_metrics_more_answers_than_shared_memory_holds():
    """More than 2048 answers (matched from global memory), with repeated entity ids."""
    B, N, pad = 2, 5000, 10 ** 6
    rs = np.random.RandomState(5)
    le = rs.randint(0, 3000, size=(B, N))
    ad = (rs.rand(B, N) < np.array([[0.6], [0.45]])).astype(f32)
    sd = np.zeros((B, N), f32)
    sd[:, :3] = 1.0
    pd = rs.rand(B, N).astype(f32) + 3.0 * ad
    pd[:, 10:20] += 50.0 * ad[:, 10:20]
    pd /= pd.sum(1, keepdims=True)
    _, f1 = check_metrics(pd, ad, sd, le, pad)
    assert (ad * (sd == 0)).sum(1).min() > 2048 and f1.min() > 0


def test_train_metrics_answer_mass_at_the_hit_threshold():
    """Answer mass at the top-1 of fp32(1e-10) (no hit: the compare is in fp32), the float above it (a hit) and the
    float below it."""
    th = f32(1e-10)
    B, N = 3, 40
    pd = np.full((B, N), 0.01, f32)
    pd[:, 7] = 0.5
    ad = np.zeros((B, N), f32)
    ad[:, 7] = [th, np.nextafter(th, f32(1)), np.nextafter(th, f32(0))]
    ad[:, 20] = 0.3
    h1, _ = check_metrics(pd, ad, np.zeros((B, N), f32), np.arange(B * N).reshape(B, N), -1)
    assert h1.tolist() == [0.0, 1.0, 0.0]


def test_train_metrics_nan_and_all_equal_rows():
    """NaN counts as maximal for hit@1 (torch.argmax): a NaN before the finite maximum, after it, two NaNs, and an
    all-equal row (the first index).  F1 is not compared where a NaN is the hit: the ranking excludes NaN."""
    B, N = 5, 300
    pd = np.full((B, N), 0.002, f32)
    ad = np.zeros((B, N), f32)
    pd[:, 50] = 0.4
    ad[:, 50] = 1.0                                           # the finite maximum is an answer
    pd[0, 10] = np.nan                                        # NaN before it, no answer there: no hit
    pd[1, 200] = np.nan                                       # NaN after it, no answer there: no hit
    pd[2, [30, 250]] = np.nan
    ad[2, 250] = 1.0                                          # answer at the second NaN only: no hit
    pd[3, 260] = np.nan
    ad[3, 260] = 1.0                                          # answer at the NaN: a hit
    pd[4] = 1.0 / N
    ad[4, 0] = 1.0                                            # all equal: the first index, an answer
    h1, _ = check_metrics(pd, ad, np.zeros((B, N), f32), np.arange(B * N).reshape(B, N), -1, f1_rows=[0, 1, 2, 4])
    assert h1.tolist() == [0.0, 0.0, 0.0, 1.0, 1.0]


def test_train_metrics_no_candidates_and_no_answers():
    """Hit questions whose every candidate is a seed or pad (c = 0), with and without an answer left; questions with
    no answers, with and without candidates."""
    B, N, pad = 4, 257, 9999
    pd = np.zeros((B, N), f32)
    ad = np.zeros((B, N), f32)
    sd = np.zeros((B, N), f32)
    le = np.tile(np.arange(N), (B, 1))
    sd[:2, 0] = 1.0
    pd[:2, 0] = 0.9                                           # the top-1 is the seed, which carries answer mass
    ad[:2, 0] = 1.0
    le[:2, 1:] = pad
    le[1, 5] = 5
    ad[1, 5] = 1.0                                            # an answer below (1-eps)/N: c = 0, one answer
    le[2:, 100:] = pad
    pd[2:, 3] = 0.9
    ad[2:, 3] = 1.0
    sd[2:, 3] = 1.0                                           # hit on a seed; no answers left
    pd[3, 4] = 0.05                                           # ... and one candidate
    h1, f1 = check_metrics(pd, ad, sd, le, pad)
    assert h1.tolist() == [1.0] * 4 and f1.tolist() == [1.0, 0.0, 1.0, 0.0]


@pytest.mark.parametrize("B,N", [(3, 1), (4, 257), (1000, 257)])
def test_train_metrics_shapes(B, N):
    rs = np.random.RandomState(B + N)
    pad = 500
    le = rs.randint(0, 300, size=(B, N))
    le[rs.rand(B, N) < 0.1] = pad
    sd = (rs.rand(B, N) < 0.02).astype(f32)
    ad = ((rs.rand(B, N) < 0.1) * rs.rand(B, N)).astype(f32)
    if N == 1:
        ad[:, 0] = 1.0
    logits = rs.randn(B, N) * 2 + 3 * (ad > 0)
    pd = np.exp(logits - logits.max(1, keepdims=True))
    h1, _ = check_metrics(pd / pd.sum(1, keepdims=True), ad, sd, le, pad)
    assert h1.sum() > 0


# ---- gr_shortest_path_nodes -------------------------------------------------------------------------------------------

def check_paths(graphs, N, sources, targets, S_, T_, seed=0):
    """graphs: per question (heads, tails) local node lists; sources / targets: per question lists of at most S_ / T_
    local indices.  The slots past the counts hold other valid node indices, which must not matter."""
    rs = np.random.RandomState(seed)
    B = len(graphs)
    heads = np.concatenate([np.asarray(h, np.int64) + b * N for b, (h, _) in enumerate(graphs)])
    tails = np.concatenate([np.asarray(t, np.int64) + b * N for b, (_, t) in enumerate(graphs)])
    g = ops.csr_build(_t(heads, torch.int64), _t(np.zeros_like(heads), torch.int64), _t(tails, torch.int64), B, N, 1)
    g.check_status()
    src = rs.randint(0, N, size=(B, S_)).astype(np.int32)
    tgt = rs.randint(0, N, size=(B, T_)).astype(np.int32)
    for b in range(B):
        src[b, :len(sources[b])] = sources[b]
        tgt[b, :len(targets[b])] = targets[b]
    scnt = np.array([len(s) for s in sources], np.int32)
    tcnt = np.array([len(t) for t in targets], np.int32)
    on, pair, dist = ops.shortest_path_nodes(g, _t(src, torch.int32), _t(scnt, torch.int32), _t(tgt, torch.int32),
                                             _t(tcnt, torch.int32), return_distances=True)
    on, pair, dist = on.cpu().numpy(), pair.cpu().numpy(), dist.cpu().numpy()
    out = []
    for b, (h, t) in enumerate(graphs):
        ns, nt = len(sources[b]), len(targets[b])
        ds, dt, pd, nodes = R.path_nodes(h, t, N, sources[b], targets[b])
        assert set(np.unique(on[b]).tolist()) <= {0, 1}
        assert np.nonzero(on[b])[0].tolist() == nodes, b
        want_pair = np.full((S_, T_), -1, np.int32)
        want_pair[:ns, :nt] = pd
        assert np.array_equal(pair[b], want_pair), b
        assert np.array_equal(dist[b, :ns], ds), b
        assert np.array_equal(dist[b, S_:S_ + nt], dt), b
        out.append((pd, nodes))
    return out


def _random_graph(rs, nodes, n_extra):
    """A random spanning tree over ``nodes`` plus n_extra random edges, every edge in a random direction."""
    nodes = np.asarray(nodes)
    parent = nodes[[rs.randint(0, i) for i in range(1, len(nodes))]]
    h = np.concatenate([nodes[1:], rs.choice(nodes, n_extra)])
    t = np.concatenate([parent, rs.choice(nodes, n_extra)])
    flip = rs.rand(len(h)) < 0.5
    return np.where(flip, t, h), np.where(flip, h, t)


def test_paths_ragged_counts_disconnected_pairs_duplicates():
    """N = 513 (past one 512-thread stride): two components per question, so some pairs are disconnected; a source
    equal to a target, duplicate targets, parallel edges and self-loops; ragged source / target counts, down to 0."""
    rs = np.random.RandomState(1)
    N = 513
    graphs, sources, targets = [], [], []
    for b in range(4):
        h1, t1 = _random_graph(rs, np.arange(0, 300), 60)
        h2, t2 = _random_graph(rs, np.arange(300, 510), 30)
        h = np.concatenate([h1, h2, h1[:20], [4, 4, 400, 512]])     # parallel edges, self-loops (512 is isolated)
        t = np.concatenate([t1, t2, t1[:20], [4, 4, 400, 512]])
        graphs.append((h, t))
    sources = [[0, 350, 7], [12], [5, 301], []]
    targets = [[7, 200, 200, 420, 511], [12, 500], [], [3, 4, 5]]
    out = check_paths(graphs, N, sources, targets, 3, 5)
    pd0 = out[0][0]
    assert pd0[0, 3] == -1 and pd0[1, 3] > 0 and pd0[2, 0] == 0 and pd0[0, 4] == -1


def test_paths_long_chain():
    """A chain of 5 000 nodes with edges in random directions: the BFS level loop runs N - 1 levels."""
    rs = np.random.RandomState(2)
    N = 5000
    h, t = np.arange(N - 1), np.arange(1, N)
    flip = rs.rand(N - 1) < 0.5
    out = check_paths([(np.where(flip, t, h), np.where(flip, h, t))], N, [[0, 2500]], [[N - 1, 1, 2500]], 2, 3)
    assert out[0][0][0, 0] == N - 1 and len(out[0][1]) == N


def test_paths_single_node_questions():
    check_paths([([0], [0]), ([0], [0])], 1, [[0], []], [[0], [0]], 1, 1)


def test_paths_twenty_thousand_nodes_and_a_hub():
    """N = 20 000 (40 thread strides) with a hub of 3 000 edges and isolated nodes among the targets."""
    rs = np.random.RandomState(3)
    N = 20_000
    h, t = _random_graph(rs, np.arange(0, N - 10), 2000)
    hub = rs.randint(0, N - 10, size=3000)
    h = np.concatenate([h, np.full(3000, 17), np.arange(5000, 5400)])
    t = np.concatenate([t, hub, np.arange(5001, 5401)])
    out = check_paths([(h, t)], N, [[17, 123]], [[N - 1, 5400, 999, 17]], 2, 4)
    assert out[0][0][0, 0] == -1 and out[0][0][0, 3] == 0


def test_path_node_sets_on_retrieved_candidates():
    """evaluate.path_node_sets end to end on evaluate.retrieve's lists for 8 questions: ragged candidate counts, several
    seeds per question."""
    B, N = 8, 300
    b = S.make_batch(11, B=B, N=N, E=900, num_entity=1000, num_relation=20, num_word=50, multi_seed=True,
                     with_weights=False)
    db = batching.stage_batch(b, torch.device(DEV), 21, False, False)
    rs = np.random.RandomState(4)
    logits = rs.randn(B, N) * np.array([0.2, 1, 2, 4, 8, 16, 30, 60])[:, None]
    pd = np.exp(logits - logits.max(1, keepdims=True))
    retrieved, _ = evaluate.retrieve(_t(pd / pd.sum(1, keepdims=True), torch.float32), db, 1000, 0.95)
    nodes, pair = evaluate.path_node_sets(db, retrieved)
    T = pair.shape[2]
    assert T == 32 and min(len(r) for r in retrieved) < T
    heads, tails, bids = b[2][0], b[2][2], b[2][3]
    for q in range(B):
        sel = bids == q
        srcs = np.nonzero(b[1][q])[0].tolist()
        tgts = retrieved[q].idx[:T].tolist()
        _ds, _dt, pdq, want = R.path_nodes(heads[sel] - q * N, tails[sel] - q * N, N, srcs, tgts)
        assert nodes[q] == want, q
        assert np.array_equal(pair[q, :len(srcs), :len(tgts)], pdq), q
        assert (pair[q, len(srcs):] == -1).all() and (pair[q, :, len(tgts):] == -1).all(), q
