"""CPU: GraftNet's host-side serving pieces.  ``loader.build_fact_mat_maxfacts`` against golden outputs of the
unmodified reference ``_build_fact_mat_maxfacts`` (tests/golden/loader/graft_fact_mat_*.npz, made by
tests/golden/make_graft_fact_mat_golden.py), alone and after ``_build_fact_mat`` in one ``get_batch``;
``install_graft``; ``parallel.shard_graft_batch`` and a gloo world-2 gather of GraftNet-shaped score blocks."""
import multiprocessing as mp
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist

from gnn_rag_b200 import loader, parallel, synthetic as S
from graft_loader_fixture import CASES, OUT_KEYS, SEQUENCE, ReplayGraftLoader, flatten_output

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loader")
FM_KEYS = ("heads", "rels", "tails", "batch_ids", "fact_ids", "weight_list", "weight_rel_list")


def _gold(name):
    return np.load(os.path.join(GOLD, "graft_fact_mat_%s.npz" % name))


def _assert_bitwise(got, gold, keys, prefix=""):
    for k in keys:
        g, w = np.asarray(got[k]), gold[prefix + k]
        assert g.dtype == w.dtype, (k, g.dtype, w.dtype)
        assert g.shape == w.shape, k
        assert np.array_equal(g, w), k           # floats included: bit for bit


@pytest.mark.parametrize("name", sorted(CASES))
def test_build_fact_mat_maxfacts_matches_reference_golden(name):
    kw, ids, dropout, seed = CASES[name]
    gold = _gold(name)
    ld = ReplayGraftLoader(gold, **kw)
    np.random.seed(seed)
    out = loader.build_fact_mat_maxfacts(ld, ids, dropout)
    assert isinstance(out[0], tuple) and len(out[0]) == 2 and all(len(m) == 4 for m in out[0])
    _assert_bitwise(flatten_output(out), gold, OUT_KEYS)
    # one permutation per question, in order: the next draw agrees with a plain replay of those draws
    np.random.seed(seed)
    for sid in ids:
        np.random.permutation(len(gold["q%d_e2f_v" % sid]))
    expect_next = np.random.rand()
    np.random.seed(seed)
    loader.build_fact_mat_maxfacts(ld, ids, dropout)
    assert np.random.rand() == expect_next
    # create_kb_adj_mats_facts ran once per distinct sample over both calls (cached on the instance)
    assert ld.calls == len(set(ids))


@pytest.mark.parametrize("first", ["drop_in", "reference_form"])
def test_get_batch_sequence_after_build_fact_mat(first):
    """``get_batch`` calls ``_build_fact_mat`` and then ``_build_fact_mat_maxfacts`` under one RNG state: with either
    version of the first (this package's drop-in or oracle/loader_oracle.py's reference-form restatement), both results
    equal the reference's bit for bit."""
    from oracle import loader_oracle
    kw, ids, dropout, seed = CASES[SEQUENCE]
    gold = _gold(SEQUENCE)
    ld = ReplayGraftLoader(gold, **kw)
    fm = loader.build_fact_mat if first == "drop_in" else loader_oracle.build_fact_mat
    np.random.seed(seed)
    got_fm = fm(ld, ids, dropout)
    got_mf = loader.build_fact_mat_maxfacts(ld, ids, dropout)
    for k, g in zip(FM_KEYS, got_fm):
        assert np.array_equal(np.asarray(g), gold["seq_fm_" + k]), k
    _assert_bitwise(flatten_output(got_mf), gold, OUT_KEYS, prefix="seq_")


def test_install_graft_patches_and_restores():
    kw, ids, dropout, seed = CASES["str"]
    gold = _gold("str")

    class Loader(ReplayGraftLoader):
        def _build_fact_mat_maxfacts(self, sample_ids, fact_dropout):
            return "original"

    orig = loader.install_graft(Loader)
    ld = Loader(gold, **kw)
    np.random.seed(seed)
    _assert_bitwise(flatten_output(ld._build_fact_mat_maxfacts(ids, dropout)), gold, OUT_KEYS)
    Loader._build_fact_mat_maxfacts = orig
    assert Loader(gold, **kw)._build_fact_mat_maxfacts(ids, dropout) == "original"
    # one instance only
    one, other = Loader(gold, **kw), Loader(gold, **kw)
    orig_bound = loader.install_graft(one)
    np.random.seed(seed)
    _assert_bitwise(flatten_output(one._build_fact_mat_maxfacts(ids, dropout)), gold, OUT_KEYS)
    assert other._build_fact_mat_maxfacts(ids, dropout) == "original"
    assert orig_bound(ids, dropout) == "original"


def _graft_batch(B, test=True):
    return S.make_graft_batch(3, B=B, N=30, E=90, num_entity=400, num_relation=11, num_word=40, fact_dropout=0.2,
                              test=test)


@pytest.mark.parametrize("B,world", [(5, 2), (7, 3), (2, 2)])
def test_shard_graft_batch_reassembles(B, world):
    b = _graft_batch(B)
    parts = [parallel.shard_graft_batch(b, r, world) for r in range(world)]
    assert [p[0].shape[0] for p in parts] == [hi - lo for lo, hi in (parallel.question_range(B, r, world)
                                                                     for r in range(world))]
    for i in (0, 1, 4, 5, 6, 8):        # local_entity, query_entities, q_input, kb_fact_rel, seed_dist, answer_dist
        assert np.array_equal(np.concatenate([p[i] for p in parts]), b[i])
    assert [list(x) for p in parts for x in p[9]] == [list(x) for x in b[9]]          # answer_lists
    for lst, bcol in ((0, 0), (1, 0)):
        want = [np.asarray(a) for a in b[3][lst]]
        got, off = [[] for _ in want], 0
        for p in parts:
            cols = p[3][lst]
            assert len(cols) == 4
            nq = p[0].shape[0]
            assert len(cols[bcol]) == 0 or (cols[bcol].min() >= 0 and cols[bcol].max() < nq)
            for k, a in enumerate(cols):
                got[k].append(a + off if k == bcol else a)
            off += nq
        for k in range(4):              # the original entries, in their original order
            assert np.array_equal(np.concatenate(got[k]), want[k]), (lst, k)
    # the kb part is sliced exactly like shard_batch slices the 7-tuple
    for r, p in enumerate(parts):
        kb7 = parallel.shard_batch((b[0], b[1], b[2], b[4], b[6], b[7], b[8]), r, world)
        for x, y in zip(p[2], kb7[2]):
            assert (x is None and y is None) or np.array_equal(np.asarray(x), np.asarray(y))
    nine = parallel.shard_graft_batch(_graft_batch(B, test=False), 0, world)
    assert len(nine) == 9


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _scores(batch):
    """A GraftNet-shaped [B, N] score block that depends on every row-sliced part of the batch."""
    le, qe, _kb, _g, qi, kfr, sd, _tb, ad = batch[:9]
    return torch.from_numpy((le % 97 + qe + sd + ad).astype(np.float32) + np.float32(kfr.sum(1, keepdims=True) % 13)
                            + np.float32(qi.sum(1, keepdims=True) % 7))


def _gather_worker(rank, world, port, B, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    b = _graft_batch(B)
    out = parallel.all_gather_scores(_scores(parallel.shard_graft_batch(b, rank, world)), B)
    q.put((rank, bool(torch.equal(out, _scores(b)))))
    dist.destroy_process_group()


@pytest.mark.parametrize("B", [6, 7])
def test_all_gather_graft_scores_gloo_world2(B):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_gather_worker, args=(r, 2, port, B, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, True), (1, True)]
