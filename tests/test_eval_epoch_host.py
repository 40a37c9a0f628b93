"""CPU: the host side of a graphed evaluation epoch -- the answer packing (loader.pack_answers), the candidate capacity
bound, the binding of gr_eval_step_record and its refusals before any CUDA call.  The GPU half is
tests/test_eval_epoch_gpu.py."""
import ctypes

import numpy as np
import pytest

from gnn_rag_b200 import _lib, graphed, loader
from oracle import kgqa_oracle as O

from test_device_split_host import NE, SplitLoader

PTR = 0x1000          # a non-null device pointer: never dereferenced, every call below is refused first


def test_pack_answers_offsets_sorted_runs_and_repeats():
    lists = np.empty(5, dtype=object)
    lists[:] = [[7, 3, 7], [], [np.int64(-1), 2 ** 40], [5], [9, 1, 9, 9, 0]]
    off, ids = loader.pack_answers(lists)
    assert off.dtype == ids.dtype == np.int64
    assert off.tolist() == [0, 3, 3, 5, 6, 11]
    assert ids.tolist() == [3, 7, 7, -1, 2 ** 40, 5, 0, 1, 9, 9, 9]
    for q in range(5):                    # every run is its list sorted, repeats kept: len(answers) is its length
        assert ids[off[q]:off[q + 1]].tolist() == sorted(int(a) for a in lists[q])


def test_pack_answers_without_any_answer_keeps_one_element():
    off, ids = loader.pack_answers([[], []])
    assert off.tolist() == [0, 0, 0] and ids.size == 1
    off, ids = loader.pack_answers([])
    assert off.tolist() == [0] and ids.size == 1


@pytest.mark.parametrize("bad", [1.0, "m.0abc", None, 2 ** 63, -2 ** 63 - 1, np.float64(3)])
def test_pack_answers_refuses_what_is_not_an_int64_id(bad):
    with pytest.raises(ValueError, match="question 2 has an answer that is not an int64 entity id"):
        loader.pack_answers([[1], [2, 3], [4, bad]])


def test_candidate_capacity_bounds_every_ranking():
    """The records of a whole split never overflow: with eps >= 1 (no probability cut, and no mass cut for rows that
    sum below eps) the ranking retrieves at most the split's non-pad entities, all of them without seeds."""
    L = SplitLoader(seed=3, num_questions=9, max_local_entity=40)
    cap = loader.candidate_capacity(L.candidate_entities, NE)
    assert cap == sum(int((row != NE).sum()) for row in L.candidate_entities)
    rs = np.random.RandomState(0)
    no_seeds = np.zeros_like(L.query_entities)
    for qe in (L.query_entities, no_seeds):
        dist = (rs.rand(*L.candidate_entities.shape) / L.max_local_entity).astype(np.float32)
        got = sum(len(r) for r in O.rank_candidates(L.candidate_entities, qe, dist, NE, 2.0))
        assert got <= cap
        if qe is no_seeds:
            assert got == cap
    assert loader.candidate_capacity(L.candidate_entities, -5) == L.candidate_entities.size


def test_eval_plan_is_the_sequential_order():
    """start_eval plans over the loader's sequential order without dropout: every question's stored facts."""
    L = SplitLoader(seed=4, num_questions=11, max_local_entity=30)
    L.reset_batches(is_sequential=True)
    stored = np.array([len(m[0]) for m in L.kb_adj_mats])
    ents = np.array([len(g) for g in L.global2local_entity_maps])
    plan = graphed.epoch_plan(L.batches[:L.num_data], stored, ents, 4, 0.0)
    assert plan.B.tolist() == [4, 4, 3]
    assert plan.F.tolist() == [int((stored + ents)[s:s + 4].sum()) for s in (0, 4, 8)]


# ---- the entry point -------------------------------------------------------------------------------------------------

def _types():
    P, I64, I = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    return [P, I64, I64, I, I64, I64] + [P] * 7 + [I64] + [P] * 8 + [I64, P, P, P, P]


def test_header_declaration_and_binding():
    I = ctypes.c_int
    assert _lib.SIGNATURES["gr_eval_step_record"] == (I, _types())
    assert _lib.load().gr_eval_step_record.argtypes == _types()


def _record(**over):
    a = dict(cursor=PTR, steps=3, batch_size=4, B=4, num_data=10, N=16, ids=PTR, local_entity=PTR, pred_dist=PTR,
             cand_idx=PTR, cand_count=PTR, a_off=PTR, a_ids=PTR, num_a=10, seed=None, split_status=PTR,
             csr_status=PTR, metrics=PTR, cases=PTR, counts=PTR, cand_off=PTR, cand=PTR, capacity=100,
             cand_total=PTR, seeds=None, eval_status=PTR, stream=None)
    a.update(over)
    lib = _lib.load()
    return lib.gr_eval_step_record(*a.values()), lib.gr_last_error().decode()


@pytest.mark.parametrize("over,msg", [
    (dict(cursor=None), "null pointer"), (dict(ids=None), "null pointer"), (dict(local_entity=None), "null pointer"),
    (dict(pred_dist=None), "null pointer"), (dict(cand_idx=None), "null pointer"),
    (dict(cand_count=None), "null pointer"), (dict(a_off=None), "null pointer"), (dict(a_ids=None), "null pointer"),
    (dict(split_status=None), "null pointer"), (dict(csr_status=None), "null pointer"),
    (dict(metrics=None), "null output"), (dict(cases=None), "null output"), (dict(counts=None), "null output"),
    (dict(cand_off=None), "null output"), (dict(cand=None), "null output"), (dict(cand_total=None), "null output"),
    (dict(eval_status=None), "null output"),
    (dict(seed=PTR), "seed and its record go together"), (dict(seeds=PTR), "seed and its record go together"),
    (dict(B=0), "need 0 < B <= batch_size"), (dict(B=5), "need 0 < B <= batch_size"),
    (dict(steps=-1), "need 0 < B <= batch_size, steps >= 0"), (dict(num_data=-1), "need 0 < B"),
    (dict(num_a=-1), "need 0 < B"), (dict(N=0), "N must be in [1, INT_MAX]"),
    (dict(N=2 ** 31), "N must be in [1, INT_MAX]"), (dict(capacity=-1), "capacity must be >= 0")])
def test_record_refusals(over, msg):
    rc, err = _record(**over)
    assert rc == -1 and err.startswith("gr_eval_step_record: invalid argument: " + msg)
