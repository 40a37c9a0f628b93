"""The restatements of tests/index_ref.py pinned without a GPU: the CSR against a stable numpy argsort (the np_csr helper
of test_parity_gpu.py) and scipy.sparse, the weights against the loader oracle (oracle/loader_oracle.build_fact_mat)
and the reference's recorded weight lists, the graft staging against the sparse entity2fact / fact2entity matrices of
oracle/graft_oracle.forward on the graft goldens, and the splitmix64 finaliser against its published values."""
import os

import numpy as np
import pytest
from scipy.sparse import coo_matrix

import index_ref as R
import test_graftnet_host as graftnet_goldens
from loader_fixture import CASES, FakeLoader, live_cases
from test_parity_gpu import np_csr

LOADER_GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loader")


def _facts(seed, F, Nt, R1, hub=False):
    rs = np.random.RandomState(seed)
    h, r, t = rs.randint(0, Nt, F), rs.randint(0, R1, F), rs.randint(0, Nt, F)
    if hub and F:
        t[rs.rand(F) < 0.3] = Nt // 2
        h[rs.rand(F) < 0.2] = 0
    return h, r, t


# ---- csr ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("seed,F,Nt,R1,hub", [(0, 0, 5, 3, False), (1, 1, 1, 1, False), (2, 200, 50, 7, False),
                                              (3, 5000, 300, 40, True), (4, 20000, 1, 3, False)])
def test_csr_matches_stable_argsort_and_scipy(seed, F, Nt, R1, hub):
    h, r, t = _facts(seed, F, Nt, R1, hub)
    c = R.csr(h, r, t, Nt, R1)
    assert c["status"] == 0 and c["live"] == F
    for d, key, other in (("t", t, h), ("h", h, t)):
        rp, src, rel, order = np_csr(key, other, r, Nt)
        assert np.array_equal(c["rowptr_" + d], rp)
        assert np.array_equal(c["fact_" + d], order)
        assert np.array_equal(c["src_" + d][:F], src) and np.array_equal(c["rel_" + d][:F], rel)
        assert not c["src_" + d][F:].any() and not c["rel_" + d][F:].any() and len(c["src_" + d]) == R.pad4(F)
        # scipy: (destination, fact index) -> CSR; inside a row its column indices are the fact ids in order
        m = coo_matrix((np.ones(F), (key, np.arange(F))), shape=(Nt, max(F, 1))).tocsr()
        m.sort_indices()
        assert np.array_equal(c["rowptr_" + d], m.indptr)
        assert np.array_equal(c["fact_" + d], m.indices)


@pytest.mark.parametrize("live", [-3, 0, 1, 50, 99, 100, 250])
def test_csr_live_prefix_and_clamping(live):
    Nt, R1, F = 30, 5, 100
    h, r, t = _facts(5, F, Nt, R1)
    c = R.csr(h, r, t, Nt, R1, live=live)
    L = min(max(live, 0), F)
    p = R.csr(h[:L], r[:L], t[:L], Nt, R1)
    assert c["live"] == L
    for k in p:
        if k.startswith(("src", "rel")):
            assert np.array_equal(c[k][:L], p[k][:L]) and not c[k][L:].any() and len(c[k]) == R.pad4(F), k
        elif k != "live":
            assert np.array_equal(c[k], p[k]), k
    # out-of-range ids past the live count do not count; inside it they clamp and set the status
    h2 = h.copy()
    h2[L:] = -7
    assert R.csr(h2, r, t, Nt, R1, live=live)["status"] == 0
    if L:
        h2[L - 1], r2 = Nt, r.copy()
        r2[0] = R1
        c2 = R.csr(h2, r2, t, Nt, R1, live=live)
        assert c2["status"] == 1
        slot = int(np.flatnonzero(c2["fact_t"] == L - 1)[0])
        assert c2["src_t"][slot] == Nt - 1
        assert c2["rel_h"][int(np.flatnonzero(c2["fact_h"] == 0)[0])] == R1 - 1


def test_relation_index_and_row_of():
    rs = np.random.RandomState(7)
    rel = rs.randint(0, 9, 1000)
    for live in (None, 0, 1, 500, 1000, 5000):
        ptr, slot = R.relation_index(rel, 9, live)
        L = 1000 if live is None else min(live, 1000)
        assert ptr[-1] == L and len(slot) == L
        assert np.array_equal(np.sort(slot), np.arange(L))
        keys = rel[slot]
        assert (np.diff(keys) >= 0).all()
        assert all((np.diff(slot[keys == k]) > 0).all() for k in range(9))
        assert all((rel[slot[ptr[k]:ptr[k + 1]]] == k).all() for k in range(9))
    rowptr = np.array([0, 0, 3, 3, 4, 8])
    assert R.row_of(rowptr).tolist() == [1, 1, 1, 3, 4, 4, 4, 4]


# ---- fact weights ------------------------------------------------------------------------------------------------------

def _loader_cases():
    return dict(CASES, **live_cases())


@pytest.mark.parametrize("name", sorted(_loader_cases()))
def test_fact_weights_match_loader_oracle_and_reference(name):
    """loader_oracle.build_fact_mat's weight lists (two Counter passes, dataset_load.py:509-517) and the ones recorded
    from the reference, rounded to fp32, against index_ref.fact_weights -- dropout and empty questions included."""
    from oracle import loader_oracle
    kw, ids, dropout, seed = _loader_cases()[name]
    ld = FakeLoader(**kw)
    np.random.seed(seed)
    heads, rels, _t, _b, _f, wl, wrl = loader_oracle.build_fact_mat(ld, ids, dropout)
    Nt = len(ids) * ld.max_local_entity
    w, wr, st = R.fact_weights(heads, rels, Nt)
    assert st == 0
    assert np.array_equal(w, np.asarray(wl, dtype=np.float64).astype(np.float32))
    assert np.array_equal(wr, np.asarray(wrl, dtype=np.float64).astype(np.float32))
    gold = np.load(os.path.join(LOADER_GOLD, "fact_mat_%s.npz" % name))
    assert np.array_equal(w, gold["weight_list"].astype(np.float32))
    assert np.array_equal(wr, gold["weight_rel_list"].astype(np.float32))


def test_fact_weights_refusals_and_rounding():
    h = np.array([0, 0, 0, 1, -1, 2, 2, 1, 1], dtype=np.int64)
    r = np.array([5, 5, 5, 2 ** 31 - 1, 0, 2 ** 31, -1, 2 ** 31 - 1, 0], dtype=np.int64)
    w, wr, st = R.fact_weights(h, r, 3)
    assert st == 1
    assert w.tolist() == [np.float32(1 / 3)] * 3 + [np.float32(1 / 3), 0, 0, 0, np.float32(1 / 3), np.float32(1 / 3)]
    assert wr.tolist() == [np.float32(1 / 3)] * 3 + [0.5, 0, 0, 0, 0.5, 1.0]
    assert R.fact_weights(h[:4], r[:4], 3)[2] == 0
    w7 = R.fact_weights(np.zeros(7, np.int64), np.zeros(7, np.int64), 1)[0]
    assert w7[0] == np.float32(1 / 7) and float(w7[0]) != 1 / 7            # inexact in fp32, rounded once


def test_mix64_published_values_and_table_arithmetic():
    # splitmix64 seeded with 0: its outputs are mix64(k * 0x9E3779B97F4A7C15), k = 1, 2, 3
    gamma = 0x9E3779B97F4A7C15
    want = [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F]
    assert [R.mix64((k * gamma) % 2 ** 64) for k in (1, 2, 3)] == want
    arr = R.mix64(np.array([(k * gamma) % 2 ** 64 for k in (1, 2, 3)], dtype=np.uint64))
    assert [int(x) for x in arr] == want
    assert [R.table_size(F) for F in (0, 1, 511, 512, 513, 1024, 1025)] == [1024, 1024, 1024, 1024, 2048, 2048, 4096]
    for T, slot in ((1024, 17), (1024, 1023), (2048, 2047)):
        h, r = R.colliding_keys(300, slot, T, 64, 16384)
        assert len(set(zip(h.tolist(), r.tolist()))) == 300
        assert (R.home_slot(h, r, T) == slot).all()
        assert all(R.mix64((int(a) << 32) | int(b)) & (T - 1) == slot for a, b in zip(h[:20], r[:20]))


# ---- graft staging -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", graftnet_goldens.CASES)
def test_graft_stage_matches_oracle_sparse_matrices(name):
    """The (b, f, head, tail, relation) facts of index_ref.graft_stage equal the slots where graft_oracle.forward's
    entity2fact [B, max_fact, N] and fact2entity [B, N, max_fact] both have an entry."""
    from oracle import graft_oracle
    g = graftnet_goldens.GraftGolden(name)
    local_entity, graft, kfr = g.batch[0], g.batch[3], np.asarray(g.batch[5])
    B, N = local_entity.shape
    M = kfr.shape[1]
    R1 = g.sd["relation_embedding.weight"].shape[0]
    (e2f_b, e2f_f, e2f_e, _v0), (f2e_b, f2e_e, f2e_f, _v1) = graft
    e2f = graft_oracle._sparse([e2f_b, e2f_f, e2f_e], len(e2f_b), (B, M, N)).coalesce()
    f2e = graft_oracle._sparse([f2e_b, f2e_e, f2e_f], len(f2e_b), (B, N, M)).coalesce()
    assert (e2f.values() == 1).all() and (f2e.values() == 1).all()        # no slot listed twice
    head = {(b, f): e for b, f, e in e2f.indices().t().tolist()}
    tail = {(b, f): e for b, e, f in f2e.indices().t().tolist()}
    want = sorted((b, f, head[b, f], tail[b, f], int(kfr[b, f])) for b, f in head.keys() & tail.keys())
    st = R.graft_stage((e2f_b, e2f_f, e2f_e), (f2e_b, f2e_e, f2e_f), kfr, B, N, M, R1)
    b, f = np.divmod(st["slot_of"], M)
    got = list(zip(b.tolist(), f.tolist(), (st["heads"] - b * N).tolist(), (st["tails"] - b * N).tolist(),
                   st["rels"].tolist()))
    assert got == want                                                     # slot order is (b, f) order
    assert st["nfacts"] == len(want) and st["status"] == (0 if head.keys() == tail.keys() else R.UNPAIRED)


def test_graft_stage_status_bits_and_live_counts():
    B, N, M, R1 = 2, 5, 4, 3
    kfr = np.array([[0, 1, 2, 1], [2, 0, 1, 0]])
    e2f = ([0, 0, 1], [0, 3, 2], [1, 2, 4])
    f2e = ([1, 0, 0], [3, 4, 0], [2, 3, 0])
    st = R.graft_stage(e2f, f2e, kfr, B, N, M, R1)
    assert st["status"] == 0 and st["nfacts"] == 3
    assert st["slot_of"].tolist() == [0, 3, 6] and st["heads"].tolist() == [1, 2, 9]
    assert st["tails"].tolist() == [0, 4, 8] and st["rels"].tolist() == [0, 1, 1]
    bad = ([0, 0, 1, 0], [0, 3, 2, M], [1, 2, 4, 0])                       # slot (0, M) does not exist
    assert R.graft_stage(bad, f2e, kfr, B, N, M, R1)["status"] == R.BAD_ID
    k2 = kfr.copy()
    k2[0, 3] = R1
    s2 = R.graft_stage(e2f, f2e, k2, B, N, M, R1)
    assert s2["status"] == R.BAD_REL and s2["rels"].tolist() == [0, 0, 1]
    dup = ([0, 0, 1, 0], [0, 3, 2, 3], [1, 2, 4, 2])
    assert R.graft_stage(dup, f2e, kfr, B, N, M, R1)["status"] == R.DUP_SLOT
    lone = ([0, 0, 1, 1], [0, 3, 2, 0], [1, 2, 4, 3])
    s3 = R.graft_stage(lone, f2e, kfr, B, N, M, R1)
    assert s3["status"] == R.UNPAIRED and s3["nfacts"] == 3
    s4 = R.graft_stage(lone, f2e, kfr, B, N, M, R1, live=(3, 3))                # the lone head is past the live count
    assert s4["status"] == 0 and s4["slot_of"].tolist() == [0, 3, 6] and s4["nfacts"] == 3
    s5 = R.graft_stage(lone, f2e, kfr, B, N, M, R1, live=(9, -1))
    assert s5["status"] == R.UNPAIRED and s5["nfacts"] == 0
