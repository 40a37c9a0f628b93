"""The index kernels that build every batch, held bit for bit to the exact restatements of tests/index_ref.py at the
places where they branch: gr_csr_build (csrc/csr_build.cu: the register / shared-memory / global row sorts, the
multi-chunk scan, live counts over a stale capacity tail, clamping), the relation index of the deterministic backward
kernels with gr_csr_row_of, gr_gather_f32, gr_fact_weights (csrc/split.cu: the hash table's probe chains and wrap,
inexact 1/count, refusals) and gr_graft_stage (csrc/graft.cu: pairing, slot order, live counts, every status bit).

Where the C entry point takes its outputs from the caller, they start at a sentinel and the test checks that nothing
past the documented extent changes.  A capacity tail past a live count always holds in-range ids, so a kernel that
read it would give a wrong answer, not a fault."""
import numpy as np
import pytest
import torch

from gnn_rag_b200 import ops
import index_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENT = -123456789          # int32 sentinel
FSENT = -7.0               # fp32 sentinel: never a weight
SLACK = 8                  # sentinel entries past every documented extent
INT32_MAX = 2 ** 31 - 1


def _dev(a, dtype=torch.int64):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV, dtype)


def _nfacts(live):
    return None if live is None else torch.tensor([live], dtype=torch.int32, device=DEV)


# ---- gr_csr_build ------------------------------------------------------------------------------------------------------

def csr_raw(h, r, t, Nt, R1, live=None, dtype=torch.int64):
    """gr_csr_build into sentinel-filled buffers SLACK entries longer than documented -> numpy arrays.  The fact slots
    [0, pad4(F)) start at fact 0 instead: the fill kernel reads a fact id from each of them, so a placement that left
    one unwritten reads an in-range fact and gives a wrong answer rather than a fault."""
    h, r, t = _dev(h, dtype), _dev(r, dtype), _dev(t, dtype)
    F = h.numel()
    full = lambda n: torch.full((n,), SENT, dtype=torch.int32, device=DEV)      # noqa: E731
    out = {k: full(Nt + 1 + SLACK) for k in ("rowptr_t", "rowptr_h")}
    out.update({k: full(R.pad4(F) + SLACK) for k in ("src_t", "rel_t", "fact_t", "src_h", "rel_h", "fact_h")})
    out["fact_t"][: R.pad4(F)] = 0
    out["fact_h"][: R.pad4(F)] = 0
    out["status"] = full(1)
    ws, nbytes = ops._workspace(h.device, "gr_csr_build_workspace_bytes", F, Nt)
    p = {k: ops._p(v) for k, v in out.items()}
    ops._launch("gr_csr_build", ops._p(h), ops._p(r), ops._p(t), h.element_size(), F, Nt, R1,
                p["rowptr_t"], p["src_t"], p["rel_t"], p["fact_t"], p["rowptr_h"], p["src_h"], p["rel_h"], p["fact_h"],
                p["status"], ops._p(_nfacts(live)), ops._p(ws), nbytes)
    return {k: v.cpu().numpy() for k, v in out.items()}


def check_csr(got, want, F, Nt, sentinel=True):
    """``got`` (numpy arrays of a build) equals ``want`` (index_ref.csr) on every specified entry: rowptr, the live
    fact slots, src / rel over pad4(F) (pads zero); with ``sentinel`` nothing past those extents was written."""
    L, Fp = want["live"], R.pad4(F)
    assert int(got["status"][0]) == want["status"]
    for d in "th":
        assert np.array_equal(got["rowptr_" + d][: Nt + 1], want["rowptr_" + d]), d
        assert np.array_equal(got["fact_" + d][:L], want["fact_" + d]), d
        assert np.array_equal(got["src_" + d][:Fp], want["src_" + d]), d
        assert np.array_equal(got["rel_" + d][:Fp], want["rel_" + d]), d
        if sentinel:
            assert (got["rowptr_" + d][Nt + 1:] == SENT).all(), d
            for k in ("src_", "rel_", "fact_"):
                assert (got[k + d][Fp:] == SENT).all(), k + d


def graph_arrays(g):
    """The arrays of an ops.CsrGraph as numpy (status included)."""
    keys = ("rowptr_t", "src_t", "rel_t", "fact_t", "rowptr_h", "src_h", "rel_h", "fact_h", "status")
    return {k: getattr(g, k).cpu().numpy() for k in keys}


def degree_graph(degrees, rows_per_degree, order, seed, filler=0):
    """Facts whose tail rows have exactly the given degrees (``rows_per_degree`` rows each, plus ``filler`` facts over
    rows of degree 3 to spread the rest over many CTAs); the head rows are a random relabelling of the tail rows, so
    both directions see the same degrees.  ``order``: 'reverse' lists the facts by descending row and reversed inside
    each row, 'random' in a random permutation; either way every row has to be reordered."""
    rs = np.random.RandomState(seed)
    tails = [np.full(d, row) for row, d in enumerate(d for d in degrees for _ in range(rows_per_degree(d)))]
    n_rows = len(tails)
    tails.append(n_rows + np.arange(filler) // 3)
    t = np.concatenate(tails).astype(np.int64)
    Nt = int(t.max()) + 2 if len(t) else 2
    h = rs.permutation(Nt)[t]
    r = rs.randint(0, 37, len(t))
    if order == "reverse":
        idx = np.lexsort((-np.arange(len(t)), -t))
    else:
        idx = rs.permutation(len(t))
    return h[idx], r[idx], t[idx], Nt


ROW_DEGREES = [0, 1, 2, 15, 16, 17, 4095, 4096, 4097, 8193]


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64], ids=["i32", "i64"])
@pytest.mark.parametrize("order", ["reverse", "random"])
def test_csr_row_sort_degrees(order, dtype):
    """Rows at and around the register sort (16/17) and the shared-memory sort (4096/4097), and rows of 8193 facts
    sorted in place in global memory."""
    h, r, t, Nt = degree_graph(ROW_DEGREES, lambda d: 256 if d <= 17 else 2, order, seed=3, filler=60000)
    want = R.csr(h, r, t, Nt, 37)
    for d in ROW_DEGREES:                              # the construction hits every degree in both directions
        assert d in np.diff(want["rowptr_t"]) and d in np.diff(want["rowptr_h"])
    check_csr(csr_raw(h, r, t, Nt, 37, dtype=dtype), want, len(h), Nt)
    g = ops.csr_build(_dev(h, dtype), _dev(r, dtype), _dev(t, dtype), 1, Nt, 37)
    check_csr(graph_arrays(g), want, len(h), Nt, sentinel=False)


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64], ids=["i32", "i64"])
@pytest.mark.parametrize("order", ["reverse", "random"])
def test_csr_one_row_holds_every_fact(order, dtype):
    rs = np.random.RandomState(4)
    F, Nt = 20000, 50
    t = np.full(F, 17)
    h = np.full(F, 3) if order == "reverse" else rs.randint(0, Nt, F)
    r = rs.randint(0, 5, F)
    idx = np.arange(F)[::-1] if order == "reverse" else rs.permutation(F)
    h, r, t = h[idx], r[idx], t[idx]
    check_csr(csr_raw(h, r, t, Nt, 5, dtype=dtype), R.csr(h, r, t, Nt, 5), F, Nt)


def _spread_facts(Nt, F, seed):
    """F facts with heads and tails uniform over [0, Nt), plus one on the last row in both directions."""
    rs = np.random.RandomState(seed)
    h, t, r = rs.randint(0, Nt, F), rs.randint(0, Nt, F), rs.randint(0, 11, F)
    h[F // 2] = t[F // 3] = Nt - 1
    return h, r, t


@pytest.mark.parametrize("Nt", [2046, 2047, 2048, 2049])
def test_csr_scan_around_one_chunk(Nt):
    """Nt + 1 counters at one 2048-entry scan chunk -1, 0, +1 and +2."""
    h, r, t = _spread_facts(Nt, 3 * Nt, Nt)
    check_csr(csr_raw(h, r, t, Nt, 11), R.csr(h, r, t, Nt, 11), len(h), Nt)


LARGE_NT = [2 ** 21 - 1, 2 ** 21, 3_000_000]


@pytest.fixture(scope="module")
def large_builds():
    """One build per large Nt (B = 1): 1 024 and 1 025 scan chunks, and ~1 465 with edges on rows past 2^21, where
    the scan of the chunk sums runs a second pass."""
    out = {}
    for Nt in LARGE_NT:
        h, r, t = _spread_facts(Nt, 400_000, Nt % 1000)
        assert (t >= 2 ** 21).sum() > 0 or Nt <= 2 ** 21
        out[Nt] = (csr_raw(h, r, t, Nt, 11), R.csr(h, r, t, Nt, 11), len(h))
    return out


@pytest.mark.parametrize("Nt", LARGE_NT)
def test_csr_scan_large(large_builds, Nt):
    got, want, F = large_builds[Nt]
    check_csr(got, want, F, Nt)


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64], ids=["i32", "i64"])
@pytest.mark.parametrize("F,Nt", [(0, 5), (1, 7), (5000, 1)], ids=["F0", "F1", "N1"])
def test_csr_edge_sizes(F, Nt, dtype):
    h, r, t = _spread_facts(Nt, F, 9) if F else (np.zeros(0, np.int64),) * 3
    check_csr(csr_raw(h, r, t, Nt, 11, dtype=dtype), R.csr(h, r, t, Nt, 11), F, Nt)


def stale_capacity(F, Nt, R1, seed):
    """A capacity-F fact buffer: every slot in range, the tail different facts from an 'earlier batch'."""
    rs = np.random.RandomState(seed)
    h, t, r = rs.randint(0, Nt, F), rs.randint(0, Nt, F), rs.randint(0, R1, F)
    h[: F // 3] = 0                                   # a hub over the register / shared-memory thresholds
    return h, r, t


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64], ids=["i32", "i64"])
@pytest.mark.parametrize("live", [0, 1, 3001, 6001, 6002, 6003, 10 ** 6, -1, -(2 ** 31)])
def test_csr_live_counts(live, dtype):
    """Only the live prefix of a capacity buffer counts; the result equals the build of the prefix alone, with zero pad
    slots [live, pad4(F))."""
    F, Nt, R1 = 6002, 40, 9
    h, r, t = stale_capacity(F, Nt, R1, seed=live % 1000)
    want = R.csr(h, r, t, Nt, R1, live=live)
    L = want["live"]
    prefix = R.csr(h[:L], r[:L], t[:L], Nt, R1)
    assert want["status"] == 0
    assert all(np.array_equal(want["fact_" + d], prefix["fact_" + d]) for d in "th")
    check_csr(csr_raw(h, r, t, Nt, R1, live=live, dtype=dtype), want, F, Nt)
    g = ops.csr_build(_dev(h, dtype), _dev(r, dtype), _dev(t, dtype), 2, Nt // 2, R1, nfacts=_nfacts(live))
    check_csr(graph_arrays(g), want, F, Nt, sentinel=False)


@pytest.mark.parametrize("dtype", [torch.int32, torch.int64], ids=["i32", "i64"])
def test_csr_out_of_range_ids_clamp(dtype):
    F, Nt, R1 = 300, 50, 6
    rs = np.random.RandomState(11)
    h, t, r = rs.randint(0, Nt, F), rs.randint(0, Nt, F), rs.randint(0, R1, F)
    h[[3, 40]], t[[7, 41]], r[[9, 42]] = [-1, Nt], [Nt, -5], [R1, -2]
    cases = [(h, r, t)]
    if dtype == torch.int64:
        h2, t2, r2 = h.copy(), t.copy(), r.copy()
        h2[100], t2[101], r2[102] = 2 ** 31 + 5, -(2 ** 33), 2 ** 40
        cases.append((h2, r2, t2))
    for hh, rr, tt in cases:
        want = R.csr(hh, rr, tt, Nt, R1)
        assert want["status"] == 1
        check_csr(csr_raw(hh, rr, tt, Nt, R1, dtype=dtype), want, F, Nt)


# ---- relation index, row_of and gather ---------------------------------------------------------------------------------

def self_loop_batch(B, N, F, R1, seed):
    """Random facts plus one self-loop per node (relation R1 - 1: a relation row of B*N entries) and a relation 0 of
    5 000 facts, in random order."""
    rs = np.random.RandomState(seed)
    Nt = B * N
    h, t, r = rs.randint(0, Nt, F), rs.randint(0, Nt, F), rs.randint(1, R1 - 1, F)
    r[:5000] = 0
    h, t, r = np.concatenate([h, np.arange(Nt)]), np.concatenate([t, np.arange(Nt)]), np.concatenate([r, np.full(Nt, R1 - 1)])
    idx = rs.permutation(len(h))
    return h[idx], r[idx], t[idx]


@pytest.mark.parametrize("live", [None, 21000, 29000], ids=["all", "live21000", "live29000"])
def test_csr_relation_index_and_row_of(live):
    """ops.csr_relation_index over both CSRs: relation rows past 4 096 (relation 0) and past 8 192 (the self-loops),
    with and without a live count over a stale tail."""
    B, N, R1 = 3, 3000, 23
    h, r, t = self_loop_batch(B, N, 20000, R1, seed=5)
    F = len(h)
    want = R.csr(h, r, t, B * N, R1, live=live)
    L = want["live"]
    g = ops.csr_build(_dev(h), _dev(r), _dev(t), B, N, R1, nfacts=_nfacts(live))
    check_csr(graph_arrays(g), want, F, B * N, sentinel=False)
    for direction, d in (("fwd", "t"), ("inv", "h")):
        ptr, slot = R.relation_index(want["rel_" + d], R1, live=L)
        if live is None:
            assert np.diff(ptr)[0] > 4096 and np.diff(ptr)[-1] > 8192
        rix_ptr, rix_slot, row_of = ops.csr_relation_index(g, direction)
        assert np.array_equal(rix_ptr[: R1 + 1].cpu().numpy(), ptr), direction
        assert np.array_equal(rix_slot[:L].cpu().numpy(), slot), direction
        assert np.array_equal(row_of[:L].cpu().numpy(), R.row_of(want["rowptr_" + d])), direction


def test_gather_f32_on_live_slots():
    F, Nt, R1, live = 6002, 40, 9, 4500
    h, r, t = stale_capacity(F, Nt, R1, seed=8)
    vals = np.random.RandomState(8).standard_normal(F).astype(np.float32)
    want = R.csr(h, r, t, Nt, R1, live=live)
    g = ops.csr_build(_dev(h), _dev(r), _dev(t), 1, Nt, R1, nfacts=_nfacts(live))
    v = _dev(vals, torch.float32)
    for d in "th":
        out = ops.gather_f32(v, getattr(g, "fact_" + d)).cpu().numpy()
        assert np.array_equal(out[:live].view(np.int32), vals[want["fact_" + d]].view(np.int32)), d


# ---- gr_fact_weights ---------------------------------------------------------------------------------------------------

def weights_raw(h, r, Nt, dtype):
    """gr_fact_weights into sentinel-filled outputs SLACK entries longer than F -> (w, wr, status)."""
    h, r = _dev(h, dtype), _dev(r, dtype)
    F = h.numel()
    w, wr = (torch.full((F + SLACK,), FSENT, device=DEV) for _ in range(2))
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    ws, nbytes = ops._workspace(h.device, "gr_fact_weights_workspace_bytes", F, Nt)
    ops._launch("gr_fact_weights", ops._p(h), ops._p(r), h.element_size(), F, int(Nt), ops._p(w), ops._p(wr),
                ops._p(status), ops._p(ws), nbytes)
    return w.cpu().numpy(), wr.cpu().numpy(), int(status.item())


def check_weights(h, r, Nt, dtype):
    w, wr, st = weights_raw(h, r, Nt, dtype)
    ww, wwr, wst = R.fact_weights(h, r, Nt)
    F = len(ww)
    assert st == wst
    assert np.array_equal(w[:F].view(np.int32), ww.view(np.int32))
    assert np.array_equal(wr[:F].view(np.int32), wwr.view(np.int32))
    assert (w[F:] == FSENT).all() and (wr[F:] == FSENT).all()
    g = ops.fact_weights(_dev(h, dtype), _dev(r, dtype), Nt)             # the wrapper: same bits
    assert np.array_equal(g[0].cpu().numpy().view(np.int32), ww.view(np.int32))
    assert np.array_equal(g[1].cpu().numpy().view(np.int32), wwr.view(np.int32))
    assert int(g[2].item()) == wst
    return ww, wwr


DTYPES = pytest.mark.parametrize("dtype", [torch.int32, torch.int64], ids=["i32", "i64"])


@DTYPES
@pytest.mark.parametrize("F", [1, 511, 512, 513])
def test_fact_weights_table_size_boundary(F, dtype):
    """F = 512 is the last count with a 1 024-slot table, 513 the first with 2 048."""
    rs = np.random.RandomState(F)
    h, r = rs.randint(0, 60, F), rs.randint(0, 4, F)
    check_weights(h, r, 60, dtype)


@DTYPES
@pytest.mark.parametrize("count", [3, 7, 70000])
def test_fact_weights_one_key(count, dtype):
    """Every fact on one (head, rel) key: 1/3, 1/7 and 1/70 000 are inexact in fp32 and must be rounded once."""
    h, r = np.full(count, 5), np.full(count, 2)
    ww, wwr = check_weights(h, r, 9, dtype)
    assert ww[0] == wwr[0] == np.float32(1.0 / count) and float(ww[0]) != 1.0 / count


@DTYPES
def test_fact_weights_all_keys_distinct(dtype):
    h, r = np.divmod(np.random.RandomState(1).permutation(6000), 60)
    ww, wwr = check_weights(h, r, 100, dtype)
    assert (wwr == 1).all() and (ww == np.float32(1 / 60)).all()


@DTYPES
@pytest.mark.parametrize("T,slot,n_keys", [(1024, 17, 300), (1024, 1023, 160), (2048, 2047, 400), (2048, 5, 400)],
                         ids=["chain1024", "wrap1024", "wrap2048", "chain2048"])
def test_fact_weights_probe_chains(T, slot, n_keys, dtype):
    """n_keys keys with one home slot: a probe chain of n_keys slots, wrapping past T - 1 to slot 0 when the home slot
    is the last.  Keys repeat 1, 2 or 3 times, in random order, so F puts the table at exactly T slots."""
    h, r = R.colliding_keys(n_keys, slot, T, 64, 16384)
    reps = 1 + np.arange(n_keys) % (3 if T == 1024 and n_keys < 200 else 2)
    h, r = np.repeat(h, reps), np.repeat(r, reps)
    assert R.table_size(len(h)) == T
    idx = np.random.RandomState(slot).permutation(len(h))
    ww, wwr = check_weights(h[idx], r[idx], 64, dtype)
    assert set(np.unique(wwr).tolist()) >= {1.0, 0.5}


@DTYPES
def test_fact_weights_refusals(dtype):
    """rel = INT_MAX is a key; INT_MAX + 1 (int64 only), a negative relation and a head outside [0, Nt) are refused:
    weight 0, counted nowhere, status 1."""
    h = np.array([0, 0, 0, 1, -1, 2, 7, 1, 1, 0], dtype=np.int64)
    r = np.array([5, 5, INT32_MAX, INT32_MAX, 0, -1, 0, INT32_MAX, 0, INT32_MAX], dtype=np.int64)
    if dtype == torch.int64:
        r[5] = INT32_MAX + 1
    ww, wwr = check_weights(h, r, 7, dtype)
    assert ww[4] == ww[5] == ww[6] == 0 and wwr[3] == 0.5
    ok = np.array([0, 1, 2, 3, 7, 8, 9])
    check_weights(h[ok], r[ok], 7, dtype)                 # the status is clear without the refused facts


# ---- gr_graft_stage ----------------------------------------------------------------------------------------------------

def graft_lists(B, N, M, R1, filled, seed, permute_tails=True):
    """Random graft lists: for every question the slots in ``filled[b]`` (a count or an index array) get a head and a
    tail, in random order; the tail list in an independent order.  kb_fact_rel rows hold relations in [0, R1) with the
    pad relation R1 - 1 on unlisted slots."""
    rs = np.random.RandomState(seed)
    e2f, f2e = [[], [], []], [[], [], []]
    kfr = np.full((B, M), R1 - 1, dtype=np.int64)
    for b in range(B):
        fs = filled[b] if isinstance(filled[b], np.ndarray) else rs.choice(M, filled[b], replace=False)
        kfr[b, fs] = rs.randint(0, R1 - 1, len(fs))
        hd, tl = rs.randint(0, N, len(fs)), rs.randint(0, N, len(fs))
        for lst, vals in ((e2f, (np.full(len(fs), b), fs, hd)), (f2e, (np.full(len(fs), b), tl, fs))):
            for k in range(3):
                lst[k].append(vals[k])
    e2f = [np.concatenate(x).astype(np.int64) for x in e2f]
    f2e = [np.concatenate(x).astype(np.int64) for x in f2e]
    i = rs.permutation(len(e2f[0]))
    e2f = [x[i] for x in e2f]
    j = rs.permutation(len(f2e[0])) if permute_tails else i
    f2e = [x[j] for x in f2e]
    return e2f, f2e, kfr


def check_stage(e2f, f2e, kfr, B, N, R1, live=None):
    """ops.graft_stage against index_ref.graft_stage: the staged facts up to nfacts, nfacts, the exact status word and
    the CSRs over the staged facts (gg.graph) against index_ref.csr."""
    M = kfr.shape[1]
    lv = None if live is None else torch.tensor(live, dtype=torch.int32, device=DEV)
    gg = ops.graft_stage([_dev(x) for x in e2f], [_dev(x) for x in f2e], _dev(kfr), B, N, R1, live=lv)
    want = R.graft_stage(e2f, f2e, kfr, B, N, M, R1, live)
    nf = int(gg.nfacts.item())
    assert nf == want["nfacts"] and int(gg.status.item()) == want["status"]
    for k in ("heads", "rels", "tails", "slot_of"):
        assert np.array_equal(getattr(gg, k)[:nf].cpu().numpy(), want[k]), k
    F0 = len(e2f[0])
    pad = lambda a: np.concatenate([a, np.zeros(F0 - len(a), np.int64)])      # noqa: E731  stale part: never read
    staged = R.csr(pad(want["heads"]), pad(want["rels"]), pad(want["tails"]), B * N, R1, live=nf)
    check_csr(graph_arrays(gg.graph), staged, F0, B * N, sentinel=False)
    return gg, want


def test_graft_stage_one_slot():
    e2f, f2e, kfr = graft_lists(1, 3, 1, 4, [1], seed=1)
    gg, want = check_stage(e2f, f2e, kfr, 1, 3, 4)
    assert want["nfacts"] == 1 and want["status"] == 0
    e2f, f2e, kfr = graft_lists(1, 3, 1, 4, [0], seed=1)
    _, want = check_stage(e2f, f2e, kfr, 1, 3, 4)
    assert want["nfacts"] == 0


def test_graft_stage_large_max_fact_few_facts():
    check_stage(*graft_lists(3, 50, 5000, 30, [3, 1, 2], seed=2), 3, 50, 30)


def test_graft_stage_empty_questions():
    _, want = check_stage(*graft_lists(5, 40, 60, 12, [20, 0, 35, 0, 0], seed=3), 5, 40, 12)
    assert want["nfacts"] == 55


@pytest.mark.parametrize("permute_tails", [False, True], ids=["same_order", "tails_permuted"])
def test_graft_stage_every_slot_filled(permute_tails):
    """Every slot paired, the last one included (nfacts is pos + flag of the last slot)."""
    B, M = 3, 50
    e2f, f2e, kfr = graft_lists(B, 30, M, 12, [np.arange(M)] * B, seed=4, permute_tails=permute_tails)
    _, want = check_stage(e2f, f2e, kfr, B, 30, 12)
    assert want["nfacts"] == B * M


def test_graft_stage_hub_rows():
    """Many facts on one head and one tail node: the staged CSR rows cross the 16 and 4 096 sort thresholds."""
    B, N, M, R1 = 2, 20, 6000, 9
    e2f, f2e, kfr = graft_lists(B, N, M, R1, [5000, 300], seed=5)
    e2f[2][: 9 * len(e2f[2]) // 10] = 3
    f2e[1][: 9 * len(f2e[1]) // 10] = 7
    check_stage(e2f, f2e, kfr, B, N, R1)


@pytest.mark.parametrize("live", [(0, 0), (1, 1), (120, 150), (300, 300), (300, 260), (400, 10 ** 6), (-1, 5)])
def test_graft_stage_live_counts_over_stale_tails(live):
    """Both lists are capacity buffers: past the live counts they hold in-range entries for slots the live part does
    not list, so reading them would pair or unpair slots that are not there."""
    B, N, M, R1 = 4, 30, 100, 10
    e2f, f2e, kfr = graft_lists(B, N, M, R1, [75, 75, 75, 75], seed=6, permute_tails=False)
    gg, want = check_stage(e2f, f2e, kfr, B, N, R1, live=live)
    lh, lt = (min(max(x, 0), 300) for x in live)
    if lh == lt:
        assert want["status"] == 0 and want["nfacts"] == lh
    rix_ptr, rix_fact = gg.fact_relation_index(R1)        # GraftNet's fact relation index over the live staged facts
    ptr, pos = R.relation_index(want["rels"], R1)
    assert np.array_equal(rix_ptr[: R1 + 1].cpu().numpy(), ptr)
    assert np.array_equal(rix_fact[: want["nfacts"]].cpu().numpy(), pos)


def test_graft_stage_live_head_count_below_capacity():
    """nfacts is the number of paired slots, here far below the head list's capacity."""
    B, N, M, R1 = 2, 30, 400, 10
    e2f, f2e, kfr = graft_lists(B, N, M, R1, [300, 300], seed=7, permute_tails=False)
    _, want = check_stage(e2f, f2e, kfr, B, N, R1, live=(40, 600))
    assert want["nfacts"] == 40 and want["status"] == R.UNPAIRED


def _status_case(bit):
    B, N, M, R1 = 2, 10, 8, 5
    e2f, f2e, kfr = graft_lists(B, N, M, R1, [5, 4], seed=8)
    e2f, f2e = [list(x) for x in e2f], [list(x) for x in f2e]
    free = [f for f in range(M) if f not in set(np.asarray(e2f[1])[np.asarray(e2f[0]) == 1].tolist())][0]
    if bit == R.BAD_ID:            # out-of-range b, f or node in either list, for slots not otherwise listed
        for lst, row in ((e2f, (B, 0, 1)), (e2f, (0, M, 1)), (f2e, (1, N, free)), (f2e, (-1, 0, 0))):
            for k in range(3):
                lst[k].append(row[k])
    elif bit == R.BAD_REL:         # the fact is kept, with relation 0
        kfr[e2f[0][0], e2f[1][0]] = R1
        kfr[e2f[0][1], e2f[1][1]] = -3
    elif bit == R.DUP_SLOT:        # a slot listed twice with the same node, in each list
        for lst in (e2f, f2e):
            for k in range(3):
                lst[k].append(lst[k][0])
    elif bit == R.UNPAIRED:        # a head without a tail
        for k, v in enumerate((1, free, 2)):
            e2f[k].append(v)
    return [np.array(x) for x in e2f], [np.array(x) for x in f2e], kfr, B, N, R1


@pytest.mark.parametrize("bit", [R.BAD_ID, R.BAD_REL, R.DUP_SLOT, R.UNPAIRED], ids=["bad_id", "bad_rel", "dup", "unpaired"])
def test_graft_stage_status_bit_alone(bit):
    e2f, f2e, kfr, B, N, R1 = _status_case(bit)
    gg, want = check_stage(e2f, f2e, kfr, B, N, R1)
    assert want["status"] == bit and int(gg.status.item()) == bit
    if bit == R.BAD_REL:
        assert (want["rels"] == 0).sum() >= 2 and want["nfacts"] == 9
    if bit in (R.BAD_ID, R.UNPAIRED):
        assert want["nfacts"] == 9
