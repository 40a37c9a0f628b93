"""The rule-path kernels (csrc/rule_paths.cu) held bit for bit to the exact restatements of tests/rule_adj_ref.py at
the places where they branch: gr_rule_adj_build (one-thread rows of <= 16 merged entries, CTA rows sorted in shared
memory up to 2 048 entries and in the global workspace beyond, the F > 8 gate of the CTA kernel, deduplication,
relabelling and self-loops), gr_rule_level_count (the int64 scan at one chunk, past it and past 1 024 chunks, a total
above 2^32, the ranges of the jobs finishing at a level), gr_rule_level_emit (zero-count runs, one entry owning every
child, totals around the grid cap), gr_rule_paths_write (more paths than the grid has threads, rule lengths 0-4 mixed)
and the walks through ops.rule_walks, paths.apply_rules and paths.reasoning_paths.

Caller-owned outputs start at a sentinel and the tests check that nothing outside the documented extent changes.  The
level entry points run on inputs laid out inside larger buffers whose margins hold in-range values, so a kernel that
used a wrong index would give a wrong answer, not a fault."""
import numpy as np
import pytest
import torch

import rule_adj_ref as A
import rule_paths_ref as R
from gnn_rag_b200 import _lib, ops, paths

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENT = -123456789          # int32 / int64 sentinel
SLACK = 8                  # sentinel entries past every documented extent


def _dev(a, dtype=torch.int32):
    return torch.as_tensor(np.ascontiguousarray(np.asarray(a, dtype=np.int64))).to(DEV, dtype)


def _full(n, dtype=torch.int32, value=SENT):
    return torch.full((n,), value, dtype=dtype, device=DEV)


def _p(t):
    return ops._p(t)


def grid_cap():
    """Threads of the largest grid the level and path kernels launch: 16 CTAs of 256 threads per SM."""
    return 16 * 256 * torch.cuda.get_device_properties(DEV).multi_processor_count


# ---- gr_rule_adj_build -------------------------------------------------------------------------------------------------

def csr_of(h, l, t, B, N):
    l = np.asarray(l, dtype=np.int64)
    return ops.csr_build(_dev(h, torch.int64), _dev(l, torch.int64), _dev(t, torch.int64), B, N,
                         int(l.max()) + 1 if len(l) else 1)


def adj_raw(g):
    """gr_rule_adj_build into sentinel-filled outputs SLACK entries longer than documented -> numpy arrays."""
    Nt, F = g.B * g.N, g.F
    out = dict(rowptr=_full(Nt + 1 + SLACK), len=_full(Nt + SLACK), nbr=_full(2 * F + SLACK), lab=_full(2 * F + SLACK))
    ws, nbytes = ops._workspace(DEV, "gr_rule_adj_workspace_bytes", F)
    ops._launch("gr_rule_adj_build", _p(g.rowptr_t), _p(g.src_t), _p(g.rel_t), _p(g.fact_t), _p(g.rowptr_h),
                _p(g.src_h), _p(g.rel_h), _p(g.fact_h), Nt, F, _p(out["rowptr"]), _p(out["len"]), _p(out["nbr"]),
                _p(out["lab"]), _p(ws), nbytes)
    return {k: v.cpu().numpy() for k, v in out.items()}


def check_adj(got, want, F, sentinel=True):
    """rowptr in full, len, and nbr / lab on [rowptr[u], rowptr[u] + len[u]); with ``sentinel`` nothing past Nt + 1,
    Nt and 2F was written.  Row capacity past len[u] is unspecified."""
    Nt = want["Nt"]
    rp, ln = got["rowptr"][: Nt + 1].astype(np.int64), got["len"][:Nt]
    assert np.array_equal(rp, want["rowptr"])
    assert np.array_equal(ln, want["len"])
    assert (rp[:-1] + ln <= rp[1:]).all()
    used = A.used_slots(want)
    assert np.array_equal(got["nbr"][used], want["nbr"])
    assert np.array_equal(got["lab"][used], want["lab"])
    if sentinel:
        assert (got["rowptr"][Nt + 1:] == SENT).all() and (got["len"][Nt:] == SENT).all()
        assert (got["nbr"][2 * F:] == SENT).all() and (got["lab"][2 * F:] == SENT).all()


def check_build(h, l, t, B, N):
    """Both the raw entry point and ops.rule_adjacency against rule_adj_ref.adjacency."""
    want = A.adjacency(h, l, t, B, N)
    g = csr_of(h, l, t, B, N)
    check_adj(adj_raw(g), want, len(h))
    adj = ops.rule_adjacency(g)
    check_adj({k: getattr(adj, k).cpu().numpy() for k in ("rowptr", "len", "nbr", "lab")}, want, len(h),
              sentinel=False)
    return want


def row_triples(length, how, seed, filler=40, n_lab=5):
    """Triples whose node 0 has a merged row of exactly ``length`` entries, plus ``filler`` triples among the other
    nodes.  'distinct': one triple per neighbour, in reversed order; 'repeated': one neighbour met ``length`` times in
    either direction with changing labels, so the row collapses to one entry with the last triple's label; 'mixed':
    about length / 3 neighbours met 1-5 times each, shuffled.  Labels repeat inside the row."""
    rs = np.random.RandomState(seed)
    if how == "distinct":
        nbrs = 1 + np.arange(length)[::-1]
    elif how == "repeated":
        nbrs = np.ones(length, dtype=np.int64)
    else:
        nbrs = 1 + rs.randint(max(length // 3, 1), size=length)
    fwd = rs.rand(length) < 0.5
    h, t = np.where(fwd, 0, nbrs), np.where(fwd, nbrs, 0)
    Nt = int(nbrs.max(initial=0)) + 4                        # the last rows are isolated
    fh, ft = 1 + rs.randint(Nt - 3, size=filler), 1 + rs.randint(Nt - 3, size=filler)
    h, t = np.concatenate([h, fh]), np.concatenate([t, ft])
    l = rs.randint(n_lab, size=len(h))
    if how == "mixed":
        idx = rs.permutation(len(h))
        h, l, t = h[idx], l[idx], t[idx]
    return h, l, t, Nt


ROW_LENGTHS = [0, 1, 15, 16, 17, 2047, 2048, 2049, 4097]


@pytest.mark.parametrize("how", ["distinct", "repeated", "mixed"])
@pytest.mark.parametrize("length", ROW_LENGTHS)
def test_adj_row_lengths(length, how):
    """Merged rows at the register / CTA boundary (16 / 17) and the shared-memory / workspace boundary (2 048 / 2 049)."""
    h, l, t, Nt = row_triples(length, how, seed=length)
    want = check_build(h, l, t, 1, Nt)
    assert want["rowptr"][1] == length
    if how == "repeated" and length:
        assert A.row(want, 0) == [(1, int(l[np.flatnonzero((h == 0) | (t == 0))[-1]]))]


@pytest.mark.parametrize("how", ["distinct", "mixed"])
def test_adj_one_row_holds_every_triple(how):
    h, l, t, Nt = row_triples(5000, how, seed=5, filler=0)
    want = check_build(h, l, t, 1, Nt)
    assert want["rowptr"][1] == len(h) == want["rowptr"][-1] // 2


@pytest.mark.parametrize("loops", [8, 9, 1025])
def test_adj_self_loops_alone(loops):
    """Every triple a self-loop on node 0: 2 * loops entries, one neighbour with the last loop's label.  8 loops: 16
    entries, the register path, and F = 8 leaves the CTA kernel unlaunched; 9: 18 entries on the CTA path with F = 9;
    1 025: 2 050 entries, sorted in the workspace."""
    l = np.random.RandomState(loops).randint(3, size=loops)
    want = check_build(np.zeros(loops, np.int64), l, np.zeros(loops, np.int64), 1, 2)
    assert want["rowptr"].tolist() == [0, 2 * loops, 2 * loops] and A.row(want, 0) == [(0, int(l[-1]))]


@pytest.mark.parametrize("loops,others", [(3, 2), (4, 8), (4, 9), (7, 30), (500, 1000), (600, 900)])
def test_adj_self_loops_mixed_with_edges(loops, others):
    """Loops on node 0 among edges to other nodes (some repeated), in shuffled order: 16 and 17 entries with F = 12 and
    13, a 2 000-entry shared-memory row and a 2 100-entry workspace row."""
    rs = np.random.RandomState(loops + others)
    nb = 1 + rs.randint(max(others * 2 // 3, 1), size=others)
    fwd = rs.rand(others) < 0.5
    h = np.concatenate([np.zeros(loops, np.int64), np.where(fwd, 0, nb)])
    t = np.concatenate([np.zeros(loops, np.int64), np.where(fwd, nb, 0)])
    l = rs.randint(4, size=len(h))
    idx = rs.permutation(len(h))
    want = check_build(h[idx], l[idx], t[idx], 1, int(nb.max()) + 2)
    assert want["rowptr"][1] == 2 * loops + others


def test_adj_large_ids_and_labels():
    """Node ids above 65 535, label ids 0 and above 65 535 repeated inside a 2 100-entry and a 40-entry row."""
    rs = np.random.RandomState(12)
    N = 70000
    hub, small = N - 10, N - 20
    nb = 65536 + rs.randint(4000, size=2100)
    nb2 = 65536 + rs.randint(4000, size=40)
    h = np.concatenate([np.full(2100, hub), nb2, [N - 1]])
    t = np.concatenate([nb, np.full(40, small), [N - 1]])
    l = np.array([0, 3, 65536, 70001])[rs.randint(4, size=len(h))]
    want = check_build(h, l, t, 1, N)
    assert want["len"][hub] > 16 and want["len"][small] > 16


def test_adj_batches_like_reasoning_paths():
    """B questions in one padded batch (question b owns rows b*N ..): rows of degree 0 past each question's entities,
    an empty question, a batch with N = 1 (self-loops only) and one with no triples at all."""
    rs = np.random.RandomState(13)
    N, sizes = 40, [(30, 90), (5, 3), (0, 0), (40, 400), (12, 17)]
    h, l, t = [], [], []
    for b, (n_ent, n_tri) in enumerate(sizes):
        if n_ent:
            h.append(b * N + rs.randint(n_ent, size=n_tri))
            t.append(b * N + rs.randint(n_ent, size=n_tri))
            l.append(rs.randint(6, size=n_tri))
    h, l, t = np.concatenate(h), np.concatenate(l), np.concatenate(t)
    h[:200:7] = t[:200:7] = 3 * N                              # a hub in question 3
    check_build(h, l, t, len(sizes), N)
    loops = np.array([0, 2, 2, 3, 3, 3])
    check_build(loops, rs.randint(3, size=6), loops, 5, 1)
    want = check_build(np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.int64), 3, 5)
    assert not want["rowptr"].any() and not want["len"].any()


# ---- gr_rule_level_count -----------------------------------------------------------------------------------------------

def dev_adjacency(adj):
    """The restated adjacency on the device, rows at rowptr.  Capacity slots past len hold label 0 (a label the rules
    ask for) and neighbour 0, so a kernel that read them would count or emit wrong entries."""
    cap = max(int(adj["rowptr"][-1]), 1)
    nbr, lab = np.zeros(cap, np.int64), np.zeros(cap, np.int64)
    used = A.used_slots(adj)
    nbr[used], lab[used] = adj["nbr"], adj["lab"]
    return ops.RuleAdjacency(_dev(adj["rowptr"]), _dev(adj["len"]), _dev(nbr), _dev(lab))


def count_raw(dadj, rule_off, rule_len, rule_lab, level, node, job):
    """gr_rule_level_count into sentinel-filled outputs -> numpy (seg_begin, off, res_begin, res_count)."""
    n, J = len(node), len(rule_len)
    seg, off = _full(n + SLACK), _full(n + 1 + SLACK, torch.int64)
    rb, rc = _full(J + SLACK), _full(J + SLACK)
    d_off, d_len, d_lab = _dev(rule_off), _dev(rule_len), _dev(np.append(rule_lab, -1))
    d_node, d_job = _dev(node), _dev(job)
    ws, nbytes = ops._workspace(DEV, "gr_rule_level_workspace_bytes", n)
    ops._launch("gr_rule_level_count", _p(dadj.rowptr), _p(dadj.len), _p(dadj.lab), _p(d_off), _p(d_len), _p(d_lab),
                J, level, _p(d_node), _p(d_job), n, _p(seg), _p(off), _p(rb), _p(rc), _p(ws), nbytes)
    return dict(seg_begin=seg.cpu().numpy(), off=off.cpu().numpy(), res_begin=rb.cpu().numpy(),
                res_count=rc.cpu().numpy())


def check_count(got, want, J):
    """child_off[0..n] exact, seg_begin where the count is non-zero, the finishing jobs' ranges; nothing past n / n + 1
    written, and res_begin / res_count of every other job untouched."""
    n = len(want["count"])
    assert np.array_equal(got["off"][: n + 1], want["off"])
    assert (got["off"][n + 1:] == SENT).all()
    nz = want["count"] > 0
    assert np.array_equal(got["seg_begin"][:n][nz], want["seg_begin"][nz])
    assert (got["seg_begin"][n:] == SENT).all()
    fin = want["fin"]
    assert np.array_equal(got["res_begin"][fin], want["res_begin"])
    assert np.array_equal(got["res_count"][fin], want["res_count"])
    rest = np.setdiff1d(np.arange(J + SLACK), fin)
    assert (got["res_begin"][rest] == SENT).all() and (got["res_count"][rest] == SENT).all()


def random_jobs(J, rs, n_lab, max_len=4):
    """J rules of length 0..max_len over labels [0, n_lab), with -1 (a label the graph lacks) at the first position of
    some and at a middle position of others."""
    rule_len = rs.randint(max_len + 1, size=J)
    rule_off = np.zeros(J, np.int64)
    np.cumsum(rule_len[:-1], out=rule_off[1:])
    rule_lab = rs.randint(n_lab, size=int(rule_len.sum()))
    for j in np.flatnonzero(rule_len)[::7]:
        rule_lab[rule_off[j] + (rule_len[j] // 2 if j % 2 else 0)] = -1
    return rule_off, rule_len, rule_lab


@pytest.fixture(scope="module")
def count_graph():
    """3 000 nodes, 20 000 triples over 6 labels and a 3 000-triple hub: segments of 0 to hundreds of entries."""
    rs = np.random.RandomState(21)
    Nt, F = 3000, 20000
    h, t, l = rs.randint(Nt, size=F), rs.randint(Nt, size=F), rs.randint(6, size=F)
    h[:3000] = 7
    adj = A.adjacency(h, l, t, 1, Nt)
    return adj, dev_adjacency(adj)


FRONTIERS = [0, 1, 1023, 1024, 1025, 1048575, 1048576, 2100000]


@pytest.mark.parametrize("n", FRONTIERS)
def test_count_scan_frontiers(count_graph, n):
    """n + 1 scanned entries: one 1 024-entry chunk (n = 1 023), one past it, and 1 024 / 1 025 / 2 051 chunks, where
    the scan of the chunk sums carries across its 1 024-thread passes."""
    adj, dadj = count_graph
    rs = np.random.RandomState(n % 997)
    J = 300
    rule_off, rule_len, rule_lab = random_jobs(J, rs, 6)
    job = np.sort(rs.randint(J, size=n))
    node = rs.randint(adj["Nt"], size=n)
    node[:: 5] = 7                                             # the hub
    want = A.level_count(adj, rule_off, rule_len, rule_lab, 1, node, job)
    if n > 1000:
        assert want["count"].max() > 100 and (want["count"] == 0).sum() > n // 10
    check_count(count_raw(dadj, rule_off, rule_len, rule_lab, 1, node, job), want, J)


def test_count_total_above_2_32_is_exact_and_emit_refuses_it():
    """65 537 entries on a hub of 65 536 neighbours with one label: 4 295 032 832 children, just above 2^32."""
    k = 65536
    h, t, l = np.zeros(k, np.int64), 1 + np.arange(k), np.zeros(k, np.int64)
    adj = A.adjacency(h, l, t, 1, k + 1)
    dadj = dev_adjacency(adj)
    n = k + 1
    node, job = np.zeros(n, np.int64), np.zeros(n, np.int64)
    rule = (np.zeros(1, np.int64), np.array([2]), np.zeros(2, np.int64))
    want = A.level_count(adj, *rule, 0, node, job)
    assert want["off"][-1] == n * k == 4295032832 > 2 ** 32
    check_count(count_raw(dadj, *rule, 0, node, job), want, 1)
    d_job, seg, off = _dev(job), _dev(want["seg_begin"]), _dev(want["off"], torch.int64)
    outs = [_full(SLACK) for _ in range(3)]
    with pytest.raises(_lib.GrError, match="4295032832"):
        ops._launch("gr_rule_level_emit", _p(dadj.nbr), _p(d_job), _p(seg), _p(off), n, int(want["off"][-1]),
                    *(_p(o) for o in outs))
    assert all((o.cpu().numpy() == SENT).all() for o in outs)


@pytest.fixture(scope="module")
def walk_graph():
    rs = np.random.RandomState(22)
    Nt, F = 400, 1500
    h, t, l = rs.randint(Nt, size=F), rs.randint(Nt, size=F), rs.randint(5, size=F)
    h[::50] = t[1::50] = 11                                    # self-loops
    adj = A.adjacency(h, l, t, 1, Nt)
    return adj, dev_adjacency(adj)


@pytest.mark.parametrize("J", [0, 1, 255, 256, 257, 5000])
def test_count_every_level_of_jobs_finishing_at_levels_0_to_4(walk_graph, J):
    """Every level's frontier of an expansion whose jobs (rule lengths 0-4 interleaved, absent labels, starts -1 with
    empty rules and dropped starts -1 with non-empty ones) finish at different levels: one job-range thread per job,
    J around one 256-thread block and many blocks."""
    adj, dadj = walk_graph
    rs = np.random.RandomState(J)
    rule_off, rule_len, rule_lab = random_jobs(J, rs, 5)
    start = rs.randint(adj["Nt"], size=J)
    start[4::9] = -1
    x = A.expand(adj, start, rule_off, rule_len, rule_lab)
    if J == 0:
        got = count_raw(dadj, rule_off, rule_len, rule_lab, 0, np.zeros(0, np.int64), np.zeros(0, np.int64))
        check_count(got, A.level_count(adj, rule_off, rule_len, rule_lab, 0, [], []), 0)
        return
    for level, lv in enumerate(x["levels"]):
        check_count(count_raw(dadj, rule_off, rule_len, rule_lab, level, lv["node"], lv["job"]), lv, J)
    if J >= 256:
        assert len(x["levels"]) == 5 and (x["res_count"] == 0).sum() > 0 and x["res_count"].max() > 1
        assert ((start == -1) & (rule_len == 0)).any() and ((start == -1) & (rule_len > 0)).any()


# ---- gr_rule_level_emit ------------------------------------------------------------------------------------------------

def emit_raw(nbr, seg_begin, off, job):
    """gr_rule_level_emit into sentinel-filled outputs.  nbr sits between margins as long as the largest count, and
    seg_begin / job are followed by SLACK zeros: a child given a wrong parent reads in-range values."""
    off = np.asarray(off, np.int64)
    n, total = len(job), int(off[-1])
    M = int(np.diff(off).max(initial=0)) + SLACK
    nbr_buf = _dev(np.concatenate([np.full(M, -5), nbr, np.full(M, -5)]))
    seg_d = _dev(np.concatenate([seg_begin, np.zeros(SLACK, np.int64)]))
    job_d = _dev(np.concatenate([job, np.zeros(SLACK, np.int64)]))
    off_d = _dev(off, torch.int64)
    outs = [_full(total + SLACK) for _ in range(3)]
    ops._launch("gr_rule_level_emit", _p(nbr_buf[M:]), _p(job_d), _p(seg_d), _p(off_d), n, total, *(_p(o) for o in outs))
    return [o.cpu().numpy() for o in outs]


def emit_case(kind, total, rs):
    """Per-entry counts: 'runs' = counts 1-5 with zero runs first (500), last (500) and in the middle (3 000 and
    single zeros); 'single' = one entry owns every child; 'spread' = random counts summing to ``total``; 'none' =
    every count 0."""
    if kind == "runs":
        cnt = rs.randint(1, 6, size=20000)
        cnt[:500] = cnt[-500:] = cnt[5000:8000] = 0
        cnt[rs.randint(20000, size=300)] = 0
    elif kind == "single":
        cnt = np.zeros(3000, np.int64)
        cnt[1234] = total
    elif kind == "spread":
        cuts = np.sort(rs.randint(total + 1, size=99999))
        cuts[:100] = 0                                         # a zero-count run first
        cnt = np.diff(np.concatenate([[0], cuts, [total]]))
    else:
        cnt = np.zeros(1000, np.int64)
    n = len(cnt)
    size = int(cnt.max()) + 1000
    nbr = rs.randint(0, 2 ** 31 - 1, size=size)
    seg = rs.randint(0, size - cnt + 1)                        # a zero-count entry's seg_begin is never read
    off = np.zeros(n + 1, np.int64)
    np.cumsum(cnt, out=off[1:])
    job = np.sort(rs.randint(50, size=n))
    return nbr, seg, off, job


EMIT_CASES = [("runs", None), ("single", 1), ("single", "cap-1"), ("single", "cap+1"), ("spread", "cap-1"),
              ("spread", "cap+1"), ("none", 0)]


@pytest.mark.parametrize("case", range(len(EMIT_CASES)), ids=["%s_%s" % c for c in EMIT_CASES])
def test_emit_children(case):
    """Zero-count entries first, last and in runs; totals 0, 1 and one less and one more than the grid cap's
    threads."""
    kind, total = EMIT_CASES[case]
    if isinstance(total, str):
        total = grid_cap() + (1 if total.endswith("+1") else -1)
    nbr, seg, off, job = emit_case(kind, total, np.random.RandomState(case))
    total = int(off[-1])
    if kind != "runs":
        assert total == EMIT_CASES[case][1] or total in (grid_cap() - 1, grid_cap() + 1)
    got = emit_raw(nbr, seg, off, job)
    want = A.level_emit(nbr, seg, off, job)
    for g, w in zip(got, want):
        assert np.array_equal(g[:total], w)
        assert (g[total:] == SENT).all()


# ---- gr_rule_paths_write and the walks ---------------------------------------------------------------------------------

STAR = 800


def write_graph():
    """An 800-leaf star (centre 0, label 0) and a 30-node ring with chords (labels 1, 2) -> (h, l, t, Nt)."""
    ring = STAR + 1 + np.arange(30)
    h = np.concatenate([np.zeros(STAR, np.int64), ring, ring[:27:3]])
    t = np.concatenate([1 + np.arange(STAR), np.roll(ring, -1), ring[5::3]])
    l = np.concatenate([np.zeros(STAR, np.int64), 1 + np.arange(30) % 2, np.full(9, 2)])
    return h, l, t, STAR + 31


# (start, rule): rule lengths 0-4 mixed, jobs without paths between jobs with many
WRITE_JOBS = [(0, [0, 0, 0]), (STAR + 1, [7]), (3, []), (0, [0]), (-1, [0]), (0, [0, 0]), (STAR + 5, [1, 2, 1, 2]),
              (-1, []), (STAR + 2, [2, 2]), (1, [0, 0, 0, 0]), (STAR + 9, [1, 1])]


def write_expected():
    h, l, t, Nt = write_graph()
    adj = A.adjacency(h, l, t, 1, Nt)
    lab2id = {x: x for x in range(8)}
    return (h, l, t, Nt), adj, A.encode_jobs(lab2id, [s for s, _ in WRITE_JOBS], [r for _, r in WRITE_JOBS])


def test_write_star_closed_form_and_mixed_jobs():
    """gr_rule_paths_write on the restated levels: P above the grid cap (the star job alone gives 640 000 paths).  The
    levels sit in one buffer at a stride of the largest level + 2 with zero margins, and the pointer arrays start one
    pointer early, so every index a wrong parent link can produce reads inside the buffer."""
    _, adj, jobs = write_expected()
    start, rule_off, rule_len, rule_lab = jobs
    x = A.expand(adj, start, rule_off, rule_len, rule_lab)
    i = np.arange(STAR * STAR)
    star = np.stack([0 * i, 1 + i // STAR, 0 * i, 1 + i % STAR], 1).reshape(-1)
    assert np.array_equal(x["paths"][: len(star)], star)             # job 0, in closed form
    counts = x["counts"]
    P = int(counts.sum())
    assert P > grid_cap() and (counts == 0).sum() >= 2 and counts[2] == counts[7] == 1
    levels = x["levels"]
    S = max(len(lv["node"]) for lv in levels) + 2
    nb = np.zeros((len(levels) + 1) * S + 1, np.int64)
    pb = np.zeros_like(nb)
    for k, lv in enumerate(levels):
        base = 1 + (k + 1) * S
        nb[base: base + len(lv["node"])] = lv["node"]
        pb[base: base + len(lv["parent"])] = lv["parent"]
    dn, dp = _dev(nb), _dev(pb)
    lv_node = torch.tensor([dn.data_ptr() + 4 * (1 + k * S) for k in range(len(levels) + 1)], dtype=torch.int64,
                           device=DEV)
    lv_parent = torch.tensor([dp.data_ptr() + 4 * (1 + k * S) for k in range(len(levels) + 1)], dtype=torch.int64,
                             device=DEV)
    path_off = np.zeros(len(counts) + 1, np.int64)
    np.cumsum(counts, out=path_off[1:])
    E = int(x["elem_off"][-1])
    out = _full(E + SLACK)
    args = [_dev(rule_len), _dev(x["res_begin"]), _dev(path_off, torch.int64), _dev(x["elem_off"][:-1], torch.int64)]
    ops._launch("gr_rule_paths_write", _p(lv_node[1:]), _p(lv_parent[1:]), *(_p(a) for a in args), len(counts), P,
                _p(out))
    got = out.cpu().numpy()
    assert np.array_equal(got[:E], x["paths"])
    assert (got[E:] == SENT).all()


def check_walks(adj_dev, adj, start, rule_off, rule_len, rule_lab):
    x = A.expand(adj, start, rule_off, rule_len, rule_lab)
    got, counts, elem_off = ops.rule_walks(adj_dev, start, rule_off, rule_len, rule_lab)
    assert np.array_equal(counts, x["counts"])
    assert np.array_equal(elem_off, x["elem_off"][:-1])
    assert np.array_equal(got.cpu().numpy(), x["paths"])
    return x


def test_walks_mixed_jobs_over_the_grid_cap():
    """The same jobs end to end through ops.rule_adjacency and ops.rule_walks."""
    (h, l, t, Nt), adj, jobs = write_expected()
    x = check_walks(ops.rule_adjacency(csr_of(h, l, t, 1, Nt)), adj, *jobs)
    assert int(x["counts"].sum()) > grid_cap()


def string_triples(h, l, t):
    return [("n%d" % a, "l%d" % r, "n%d" % b) for a, r, b in zip(h.tolist(), l.tolist(), t.tolist())]


def shape_rules(n_lab):
    """One- and two-step rules from the hub, three-step rules from a leaf, the empty rule, a label the graph lacks and
    an unstripped label."""
    one = [["l%d" % x] for x in range(n_lab)]
    two = [["l%d" % x, "l%d" % ((x + 1) % n_lab)] for x in range(n_lab)]
    return one, two + [["l0", "l0", "l1"], ["l2", "l1", "l0"]], [[], ["l%d" % n_lab], [" l0"], ["l0", "lx", "l0"]]


@pytest.mark.parametrize("how", ["distinct", "repeated", "mixed"])
@pytest.mark.parametrize("length", [1, 16, 17, 2048, 2049, 4097])
def test_walks_on_adjacency_shapes(length, how):
    """paths.apply_rules on the adjacency shapes against the restated expansion, and against networkx where the
    walks are few."""
    h, l, t, Nt = row_triples(length, how, seed=length + 1)
    tri = string_triples(h, l, t)
    one, more, edge = shape_rules(5)
    g = paths.build_graph(tri)
    hub_jobs = (["n0", "n1", "absent"], one + edge + (more[:5] if length <= 2049 else more[:2]))
    leaf_jobs = (["n%d" % v for v in np.unique(np.concatenate([h, t]))[1:4]], more)
    for sources, rules in (hub_jobs, leaf_jobs):
        got = paths.apply_rules(g, rules, sources)
        assert got == A.apply_rules(tri, rules, sources)
        if length <= 17:
            assert got == R.apply_rules(R.build_graph(tri), rules, sources)


def test_walks_reasoning_paths_batch_of_shapes():
    """paths.reasoning_paths over a batch of the shapes (a 2 049-entry hub, 16- and 17-entry rows, self-loops, an empty
    question) against the restated expansion per question."""
    qs = []
    for length, how in [(17, "mixed"), (2049, "distinct"), (16, "repeated"), (0, "distinct")]:
        h, l, t, _ = row_triples(length, how, seed=length + 2)
        qs.append(string_triples(h, l, t))
    qs.append(string_triples(np.zeros(9, np.int64), np.arange(9) % 2, np.zeros(9, np.int64)))
    qs.append([])
    one, more, edge = shape_rules(5)
    questions = [dict(graph=tri, q_entity=["n0", "n1", "absent"], predicted_paths=one + edge + more[:3], cand=None)
                 for tri in qs]
    for q, r in zip(questions, paths.reasoning_paths(questions)):
        want = A.apply_rules(q["graph"], q["predicted_paths"], q["q_entity"])
        assert r.rule_paths == want
        assert r.with_rules == [paths.path_to_string(p) for p in want] and r.without_rules == []


def test_walks_batch_without_triples():
    questions = [dict(graph=[], q_entity=["a", "b"], predicted_paths=[[], ["r"]], cand=None)] * 3
    for r in paths.reasoning_paths(questions):
        assert r.rule_paths == [[], []]
