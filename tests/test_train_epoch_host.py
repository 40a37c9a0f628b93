"""CPU: the host arithmetic of a graphed training epoch (graphed.epoch_plan) against the host loader's batches, and the
refusals of the epoch's entry points (gr_epoch_step_begin, gr_epoch_step_record, gr_fact_weights_live) before any
CUDA call.  The GPU half is tests/test_train_epoch_gpu.py."""
import ctypes

import numpy as np
import pytest

from gnn_rag_b200 import _lib, graphed, loader

from test_device_split_host import SplitLoader

PTR = 0x1000          # a non-null device pointer: never dereferenced, every call below is refused first


def _counts(L):
    """Stored facts and self-loops per question, read straight from the loader's per-question lists."""
    stored = np.array([len(m[0]) for m in L.kb_adj_mats], dtype=np.int64)
    ents = np.array([len(g) if L.use_self_loop else 0 for g in L.global2local_entity_maps], dtype=np.int64)
    return stored, ents


LOADERS = {   # name -> SplitLoader kwargs
    "spread": dict(seed=5, num_questions=23, max_local_entity=60, facts_lo=20, facts_hi=1200),
    "empty_questions": dict(seed=4, num_questions=9, max_local_entity=6, facts_hi=1),
    "no_self_loop": dict(seed=3, num_questions=11, max_local_entity=9, use_self_loop=False, facts_hi=300),
    "large": dict(seed=8, num_questions=7, max_local_entity=40, facts_lo=3000, facts_hi=20000),
}


@pytest.mark.parametrize("p", [0.0, 0.3, 1.0])
@pytest.mark.parametrize("batch_size", [1, 4, 5, 64])
@pytest.mark.parametrize("name", sorted(LOADERS))
def test_plan_equals_the_loaders_batches(name, batch_size, p):
    """Per step: B, the fact count F of the host loader's batch (build_fact_mat with fact dropout p), the kept facts
    (F less the self-loops), and the capacity bucket of F."""
    L = SplitLoader(**LOADERS[name])
    np.random.seed(3)
    L.reset_batches(is_sequential=False)
    stored, ents = _counts(L)
    plan = graphed.epoch_plan(L.batches, stored, ents, batch_size, p)
    steps = -(-L.num_data // batch_size)
    assert plan.steps == steps and len(plan.B) == len(plan.F) == len(plan.K) == len(plan.capacity) == steps
    for it in range(steps):
        ids = L.batches[batch_size * it:min(batch_size * (it + 1), L.num_data)]
        heads = loader.build_fact_mat(L, ids, p, weights="none")[0]
        loops = sum(len(L.global2local_entity_maps[q]) for q in ids) if L.use_self_loop else 0
        assert plan.starts[it] == batch_size * it
        assert plan.B[it] == len(ids)
        assert plan.F[it] == len(heads)
        assert plan.K[it] == len(heads) - loops
        assert plan.capacity[it] == graphed.fact_capacity(len(heads))
    if name == "empty_questions":
        assert (stored == 0).any()


def test_plan_of_the_spread_split_covers_several_buckets():
    L = SplitLoader(**LOADERS["spread"])
    plan = graphed.epoch_plan(L.batches, *_counts(L), 4)
    assert L.num_data % 4 != 0 and plan.B[-1] == L.num_data % 4
    assert len(set(plan.capacity.tolist())) >= 3


def test_plan_counts_an_out_of_range_id_as_an_empty_question():
    L = SplitLoader(**LOADERS["spread"])
    stored, ents = _counts(L)
    order = np.array([0, 1, 99, 2, -1, 3])
    plan = graphed.epoch_plan(order, stored, ents, 4)
    assert plan.F.tolist() == [int(stored[[0, 1, 2]].sum() + ents[[0, 1, 2]].sum()), int(stored[3] + ents[3])]
    assert plan.B.tolist() == [4, 2]
    assert graphed.epoch_plan([], stored, ents, 4).steps == 0


# ---- the entry points ------------------------------------------------------------------------------------------------

def test_header_declarations_and_bindings():
    P, I64, I, S = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_size_t
    sig = _lib.SIGNATURES
    assert sig["gr_epoch_step_begin"] == (I, [P, P, I64, I64, I, P, P, P, I64, I, I64, P, P, P, P, P, P, P])
    assert sig["gr_epoch_step_record"] == (I, [P, I64, I64, I, I64] + [P] * 13 + [P])
    assert sig["gr_fact_weights_live"] == (I, [P, P, I, I64, P, I64, P, P, P, P, S, P])


def _begin(**over):
    a = dict(cursor=PTR, order=PTR, num_data=10, batch_size=4, B=4, kept_table=None, q_off=PTR, q_ents=PTR, num_q=5,
             use_self_loop=1, capacity=1024, ids=PTR, rows=PTR, kept=PTR, nfacts=PTR, kept_total=PTR, status=PTR,
             stream=None)
    a.update(over)
    lib = _lib.load()
    return lib.gr_epoch_step_begin(*a.values()), lib.gr_last_error().decode()


def _record(**over):
    a = dict(cursor=PTR, steps=3, batch_size=4, B=4, num_data=10, loss=PTR, grad_norm=PTR, seed=None, h1=PTR, f1=PTR,
             split_status=PTR, csr_status=PTR, losses=PTR, grad_norms=PTR, seeds=None, h1_all=PTR, f1_all=PTR,
             epoch_status=PTR, stream=None)
    a.update(over)
    lib = _lib.load()
    return lib.gr_epoch_step_record(*a.values()), lib.gr_last_error().decode()


@pytest.mark.parametrize("over,msg", [
    (dict(cursor=None), "null pointer"), (dict(q_ents=None), "null pointer"), (dict(rows=None), "null output"),
    (dict(status=None), "null output"), (dict(B=0), "need 0 < B <= batch_size"),
    (dict(B=5), "need 0 < B <= batch_size"), (dict(num_q=-1), "need 0 < B <= batch_size"),
    (dict(capacity=-1), "capacity must be in [0, INT_MAX]"), (dict(capacity=2 ** 31), "capacity must be in")])
def test_step_begin_refusals(over, msg):
    rc, err = _begin(**over)
    assert rc == -1 and err.startswith("gr_epoch_step_begin: invalid argument: " + msg)


@pytest.mark.parametrize("over,msg", [
    (dict(loss=None), "null pointer"), (dict(csr_status=None), "null pointer"), (dict(f1_all=None), "null output"),
    (dict(grad_norms=None), "go together"), (dict(seed=PTR), "go together"), (dict(B=5), "need 0 < B"),
    (dict(steps=-1), "need 0 < B")])
def test_step_record_refusals(over, msg):
    rc, err = _record(**over)
    assert rc == -1 and err.startswith("gr_epoch_step_record: invalid argument: ") and msg in err


def test_fact_weights_live_refusals():
    lib = _lib.load()
    args = [PTR, PTR, 4, 1024, PTR, 4096, PTR, PTR, PTR, PTR, 0, None]
    need = lib.gr_fact_weights_workspace_bytes(1024, 4096)
    for i, v, msg in [(4, None, "invalid argument: null nfacts"), (0, None, "invalid argument: null pointer"),
                      (2, 2, "invalid argument: idx_bytes must be 4 or 8"),
                      (3, 2 ** 31, "invalid argument: F must fit int32 (hash slots are 32-bit)"),
                      (10, need - 1, "workspace too small (%d < %d)" % (need - 1, need))]:
        a = list(args)
        a[10] = need
        a[i] = v
        assert lib.gr_fact_weights_live(*a) in (-1, -3)
        assert lib.gr_last_error().decode() == "gr_fact_weights_live: " + msg
