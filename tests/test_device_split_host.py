"""CPU: loader.DeviceSplit's entry points (csrc/split.cu) -- header and binding agreement, the refusals of the entry
points and of the ops shape rules, and the refusals DeviceSplit makes before it touches a device.

Also home of the stand-in loaders the GPU tests wrap: loader_fixture.FakeLoader plus the fields the reference's
``get_batch`` reads (gnn/dataset_load.py:599-629, gnn/dataset_load_graft.py:113-149), with ``get_batch`` assembling
its facts by loader.build_fact_mat(shuffle=False) and, for GraftNet, loader.build_fact_mat_maxfacts under the
identity permutation.  Every entry-point call below is refused before any CUDA call, so the pointers are
placeholders that are never dereferenced."""
import ctypes
from unittest import mock

import numpy as np
import pytest
import torch

from gnn_rag_b200 import _lib, loader, ops
from loader_fixture import CASES, FakeLoader

NE, NR, NW = 3000, 40, 100       # entity, relation (num_kb_relation) and word vocabulary of the stand-ins
PTR = 0x1000
INVALID, WORKSPACE = -1, -3
INT_MAX = 2 ** 31 - 1


class SplitLoader(FakeLoader):
    """FakeLoader + the fields ``SingleDataLoader.get_batch`` reads.  Every question has one seed (local 0), up to two
    answers and 2..Q tokens; pads are NE (entities) and NW (words)."""
    q_type = "seq"

    def __init__(self, seed, num_questions, max_local_entity, num_kb_relation=NR, Q=6, weights="arrays",
                 index_dtype=np.int64, **kw):
        super().__init__(seed, num_questions, max_local_entity, num_kb_relation, **kw)
        rs = np.random.RandomState(seed + 1000)
        n, N = num_questions, max_local_entity
        self.num_data = n
        self.batches = np.arange(n)
        self.weights, self.index_dtype = weights, index_dtype
        self.candidate_entities = np.full((n, N), NE, dtype=int)
        self.query_entities = np.zeros((n, N))
        self.seed_distribution = np.zeros((n, N))
        self.answer_dists = np.zeros((n, N))
        self.query_texts = np.full((n, Q), NW, dtype=int)
        self.answer_lists = np.empty(n, dtype=object)
        for q in range(n):
            ne = len(self.global2local_entity_maps[q])
            self.candidate_entities[q, :ne] = rs.randint(0, NE, ne)
            self.query_entities[q, 0] = self.seed_distribution[q, 0] = 1.0
            ans = rs.choice(ne, min(2, ne), replace=False)
            self.answer_dists[q, ans] = 1.0
            self.answer_lists[q] = self.candidate_entities[q, ans].tolist()
            k = int(rs.randint(2, Q + 1))
            self.query_texts[q, :k] = rs.randint(0, NW, k)

    def _build_fact_mat(self, sample_ids, fact_dropout):
        return loader.build_fact_mat(self, sample_ids, fact_dropout, weights=self.weights,
                                     index_dtype=self.index_dtype, shuffle=False)

    def reset_batches(self, is_sequential=True):
        self.batches = np.arange(self.num_data) if is_sequential else np.random.permutation(self.num_data)

    def get_quest(self, training=False):
        return ["question %d" % s for s in self.sample_ids]

    def _head(self, iteration, batch_size):
        start = batch_size * iteration
        sample_ids = self.batches[start:min(batch_size * (iteration + 1), self.num_data)]
        self.sample_ids = sample_ids
        return sample_ids

    def get_batch(self, iteration, batch_size, fact_dropout, q_type=None, test=False):
        ids = self._head(iteration, batch_size)
        kb = self._build_fact_mat(ids, fact_dropout)
        out = (self.candidate_entities[ids], self.query_entities[ids], kb, self.query_texts[ids],
               self.seed_distribution[ids], None, self.answer_dists[ids])
        return out + ((self.answer_lists[ids],) if test else ())


class GraftSplitLoader(SplitLoader):
    """SplitLoader + GraftNet's fields: ``create_kb_adj_mats_facts`` restated for integer tuples (one graft fact per
    stored fact; with ``use_inverse_relation`` facts 2i and 2i+1, gnn/dataset_load_graft.py:27-68), ``max_facts`` and
    the loader's ``kb_fact_rels`` table."""

    def __init__(self, seed, num_questions, max_local_entity, num_relations=(NR - 1) // 2, use_inverse_relation=False,
                 **kw):
        num_kb_relation = (2 if use_inverse_relation else 1) * num_relations + 1
        super().__init__(seed, num_questions, max_local_entity, num_kb_relation=num_kb_relation, **kw)
        self.num_relations, self.use_inverse_relation = num_relations, use_inverse_relation
        self.max_facts = 2 * max([len(m[0]) for m in self.kb_adj_mats] + [0]) + max_local_entity
        self.kb_fact_rels = np.full((num_questions, self.max_facts), self.num_kb_relation, dtype=int)
        for q in range(num_questions):
            self.kb_fact_rels[q] = self.create_kb_adj_mats_facts(q)[1]

    def create_kb_adj_mats_facts(self, q):
        h, r, t = (np.asarray(a, dtype=int) for a in self.kb_adj_mats[q])
        r = r % self.num_relations
        T = len(h)
        kfr = np.full(self.max_facts, self.num_kb_relation, dtype=int)
        if self.use_inverse_relation:
            f = np.arange(2 * T)
            e2f_e, f2e_e = np.stack([h, t], 1).reshape(-1), np.stack([t, h], 1).reshape(-1)
            kfr[0:2 * T:2], kfr[1:2 * T:2] = r, r + self.num_relations
        else:
            f, e2f_e, f2e_e = np.arange(T), h, t
            kfr[:T] = r
        ones = np.ones(len(f))
        return ((f, e2f_e, ones), (f2e_e, f.copy(), ones.copy())), kfr

    def get_batch(self, iteration, batch_size, fact_dropout, q_type=None, test=False):
        ids = self._head(iteration, batch_size)
        kb = self._build_fact_mat(ids, fact_dropout)
        with mock.patch.object(np.random, "permutation", np.arange):        # stored order
            graft, _ = loader.build_fact_mat_maxfacts(self, ids, fact_dropout)
        out = (self.candidate_entities[ids], self.query_entities[ids], kb, graft, self.query_texts[ids],
               self.kb_fact_rels[ids], self.seed_distribution[ids], None, self.answer_dists[ids])
        return out + ((self.answer_lists[ids],) if test else ())


def fake_cases():
    """loader_fixture.CASES without fact dropout: name -> (loader kwargs, sample ids)."""
    return {name: (kw, ids) for name, (kw, ids, _drop, _seed) in CASES.items()}


# ---- header and bindings ----------------------------------------------------------------------------------------------

I64, I32, VP = ctypes.c_int64, ctypes.c_int, ctypes.c_void_p

EXPECTED = {
    "gr_split_assemble": [VP] * 5 + [I64, VP, I32, I64, I64, I32, I32, I64] + [VP] * 7,
    "gr_split_assemble_graft": [VP] * 7 + [I64, VP, I32, I64, I64, I32, I64] + [VP] * 11,
    "gr_fact_weights_workspace_bytes": [I64, I64],
    "gr_fact_weights": [VP, VP, I32, I64, I64, VP, VP, VP, VP, ctypes.c_size_t, VP],
}


@pytest.mark.parametrize("name", sorted(EXPECTED))
def test_header_prototypes_bind(name):
    res, args = _lib.SIGNATURES[name]
    assert args == EXPECTED[name]
    assert res == (ctypes.c_size_t if name.endswith("_bytes") else ctypes.c_int)
    fn = getattr(_lib.load(), name)
    assert fn.argtypes == EXPECTED[name]


# ---- entry-point refusals (before any CUDA call) -----------------------------------------------------------------------

def _assemble(**over):
    a = dict(q_off=PTR, q_heads=PTR, q_rels=PTR, q_tails=PTR, q_ents=PTR, num_q=3, ids=PTR, B=2, N=5, self_rel=4,
             use_self_loop=1, idx_bytes=4, F=10, heads=PTR, rels=PTR, tails=PTR, batch_ids=PTR, fact_ids=PTR,
             status=PTR, stream=None)
    a.update(over)
    lib = _lib.load()
    return lib.gr_split_assemble(*a.values()), lib.gr_last_error().decode()


@pytest.mark.parametrize("over,msg", [
    (dict(q_off=None), "null pointer"),
    (dict(ids=None), "null pointer"),
    (dict(status=None), "null pointer"),
    (dict(B=0), "need num_q >= 0, B > 0, N > 0 and F >= 0"),
    (dict(N=0), "need num_q >= 0, B > 0, N > 0 and F >= 0"),
    (dict(F=-1), "need num_q >= 0, B > 0, N > 0 and F >= 0"),
    (dict(num_q=-1), "need num_q >= 0, B > 0, N > 0 and F >= 0"),
    (dict(idx_bytes=2), "idx_bytes must be 4 or 8"),
    (dict(B=2, N=2 ** 30), "the batch overflows int32 indices"),
    (dict(F=2 ** 31), "the batch overflows int32 indices"),
    (dict(self_rel=-1), "self_rel must be non-negative"),
    (dict(tails=None), "null output arrays"),
    (dict(q_ents=None), "null resident arrays"),
])
def test_split_assemble_refusals(over, msg):
    assert _assemble(**over) == (INVALID, "gr_split_assemble: invalid argument: " + msg)


def _graft(**over):
    a = dict(g_off=PTR, g_e2f_f=PTR, g_e2f_e=PTR, g_f2e_e=PTR, g_f2e_f=PTR, r_off=PTR, r_vals=PTR, num_q=3, ids=PTR,
             B=2, max_facts=7, rel_pad=9, idx_bytes=4, G=10, e2f_b=PTR, e2f_f=PTR, e2f_e=PTR, e2f_v=PTR, f2e_b=PTR,
             f2e_e=PTR, f2e_f=PTR, f2e_v=PTR, kb_fact_rel=PTR, status=PTR, stream=None)
    a.update(over)
    lib = _lib.load()
    return lib.gr_split_assemble_graft(*a.values()), lib.gr_last_error().decode()


@pytest.mark.parametrize("over,msg", [
    (dict(g_off=None), "null pointer"),
    (dict(r_off=None), "null pointer"),
    (dict(r_vals=None), "null resident arrays"),
    (dict(B=0), "need num_q >= 0, B > 0, max_facts >= 0 and G >= 0"),
    (dict(G=-1), "need num_q >= 0, B > 0, max_facts >= 0 and G >= 0"),
    (dict(idx_bytes=16), "idx_bytes must be 4 or 8"),
    (dict(G=2 ** 31), "the batch overflows int32 indices"),
    (dict(f2e_v=None), "null output arrays"),
    (dict(kb_fact_rel=None), "null kb_fact_rel"),
])
def test_split_assemble_graft_refusals(over, msg):
    assert _graft(**over) == (INVALID, "gr_split_assemble_graft: invalid argument: " + msg)


def _weights(**over):
    a = dict(heads=PTR, rels=PTR, idx_bytes=8, F=10, Nt=20, weight=PTR, weight_rel=PTR, status=PTR, workspace=PTR,
             workspace_bytes=1 << 20, stream=None)
    a.update(over)
    lib = _lib.load()
    return lib.gr_fact_weights(*a.values()), lib.gr_last_error().decode()


@pytest.mark.parametrize("over,rc,msg", [
    (dict(heads=None), INVALID, "invalid argument: null pointer"),
    (dict(status=None), INVALID, "invalid argument: null pointer"),
    (dict(weight=None, weight_rel=None), INVALID, "invalid argument: no output requested"),
    (dict(idx_bytes=3), INVALID, "invalid argument: idx_bytes must be 4 or 8"),
    (dict(Nt=0), INVALID, "invalid argument: need F >= 0 and 0 < Nt <= 2^32 - 1"),
    (dict(F=-1), INVALID, "invalid argument: need F >= 0 and 0 < Nt <= 2^32 - 1"),
    (dict(F=2 ** 31), INVALID, "invalid argument: F must fit int32 (hash slots are 32-bit)"),
    (dict(workspace=None), WORKSPACE, "workspace too small"),
    (dict(workspace_bytes=16), WORKSPACE, "workspace too small"),
])
def test_fact_weights_refusals(over, rc, msg):
    got_rc, got_msg = _weights(**over)
    assert got_rc == rc and got_msg.startswith("gr_fact_weights: " + msg)


def test_fact_weights_workspace_grows_with_facts_and_rows():
    ws = _lib.load().gr_fact_weights_workspace_bytes
    assert ws(-1, 10) == 0 and ws(10, 0) == 0
    assert ws(0, 10) > 0
    assert ws(10 ** 6, 10) > ws(10 ** 3, 10) and ws(10, 10 ** 6) > ws(10, 10)
    # the hash table alone holds >= 2F 8-byte keys and 4-byte counts
    assert ws(10 ** 6, 1) >= 2 * 10 ** 6 * 12


# ---- shape rules agree with the entry points ---------------------------------------------------------------------------

@pytest.mark.parametrize("B,N,F,dt", [(1, 1, 1, torch.int32), (2, 2 ** 30 - 1, 5, torch.int32),
                                      (2, 2 ** 30, 5, torch.int32), (2, 2 ** 30, 5, torch.int64),
                                      (1, 5, INT_MAX, torch.int32), (1, 5, INT_MAX + 1, torch.int32),
                                      (0, 5, 1, torch.int64), (3, 0, 1, torch.int64), (3, 5, -1, torch.int64)])
def test_split_assemble_ok_matches_the_entry_point(B, N, F, dt):
    ok = ops.split_assemble_ok(B, N, F, dt)
    _rc, msg = _assemble(B=B, N=N, F=F, idx_bytes=4 if dt == torch.int32 else 8, tails=None)
    # with a null output the entry point refuses anyway; the message tells whether the shape passed
    assert ok == msg.endswith("null output arrays"), msg
    assert not ops.split_assemble_ok(1, 1, 0, torch.int16)


@pytest.mark.parametrize("B,M,G,dt", [(1, 0, 5, torch.int32), (2, 7, INT_MAX, torch.int32),
                                      (2, 7, INT_MAX + 1, torch.int32), (2, 7, INT_MAX + 1, torch.int64),
                                      (0, 7, 1, torch.int64), (2, -1, 1, torch.int64)])
def test_split_assemble_graft_ok_matches_the_entry_point(B, M, G, dt):
    ok = ops.split_assemble_graft_ok(B, M, G, dt)
    _rc, msg = _graft(B=B, max_facts=M, G=G, idx_bytes=4 if dt == torch.int32 else 8, f2e_v=None)
    assert ok == msg.endswith("null output arrays"), msg


@pytest.mark.parametrize("F,Nt", [(0, 1), (10, 1), (INT_MAX, 5), (INT_MAX + 1, 5), (-1, 5), (5, 0), (5, 2 ** 32)])
def test_fact_weights_ok_matches_the_entry_point(F, Nt):
    _rc, msg = _weights(F=F, Nt=Nt, workspace=None)
    assert ops.fact_weights_ok(F, Nt) == msg.startswith("gr_fact_weights: workspace too small"), msg


# ---- DeviceSplit refusals before the upload ----------------------------------------------------------------------------

def _small():
    return SplitLoader(seed=1, num_questions=4, max_local_entity=8)


@pytest.mark.parametrize("kw,msg", [
    (dict(weights="lists"), "weights must be 'arrays' or 'none'"),
    (dict(index_dtype=torch.int16), "index_dtype must be torch.int32 or torch.int64"),
    (dict(device="cpu"), "the split lives on a CUDA device"),
])
def test_device_split_refuses_bad_arguments(kw, msg):
    kw = dict(dict(device="cuda"), **kw)
    with pytest.raises(ValueError, match=msg):
        loader.DeviceSplit(_small(), **kw)


def test_device_split_refuses_data_eff():
    L = _small()
    L.data_eff = True
    with pytest.raises(ValueError, match="data_eff"):
        loader.DeviceSplit(L, "cuda")


def test_stand_ins_match_the_host_drop_ins():
    """The stand-ins' get_batch is the host reference of the GPU tests: check its layout here."""
    L = SplitLoader(seed=5, num_questions=5, max_local_entity=9)
    b = L.get_batch(0, 3, 0.0, test=True)
    assert len(b) == 8 and b[5] is None and list(L.sample_ids) == [0, 1, 2]
    want = loader.build_fact_mat(L, [0, 1, 2], 0.0, weights="arrays", shuffle=False)
    for x, y in zip(b[2], want):
        np.testing.assert_array_equal(x, y)
    g = GraftSplitLoader(seed=6, num_questions=4, max_local_entity=7, use_inverse_relation=True)
    gb = g.get_batch(0, 4, 0.0)
    assert len(gb) == 9 and gb[5].shape == (4, g.max_facts)
    (hb, hf, he, hv), (tb, te, tf, tv) = gb[3]
    np.testing.assert_array_equal(hf, tf)              # stored order: both lists walk the slots in order
    assert len(hb) == 2 * sum(len(m[0]) for m in g.kb_adj_mats)
