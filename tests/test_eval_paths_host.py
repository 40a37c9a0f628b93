"""CPU: the host side of the shortest-path node sets of an evaluation epoch -- the refusals of ``path_targets`` and
their order, the seed counts and record sizes, the record layout :meth:`EvalRun.paths` decodes, the sweep's job form,
and the binding and refusals of gr_eval_step_paths before any CUDA call.  The GPU half is tests/test_eval_paths_gpu.py."""
import ctypes
import types

import numpy as np
import pytest

from gnn_rag_b200 import _lib, graphed, loader

from test_device_split_host import NE, SplitLoader

PTR = 0x1000          # a non-null device pointer: never dereferenced, every call below is refused first
INT_MAX = 2 ** 31 - 1


def _split(num_data=10, N=50, seeds=(1, 3, 0)):
    """A stand-in with what paths_refusal reads from a DeviceSplit."""
    return types.SimpleNamespace(num_data=num_data, N=N, max_seeds=lambda: max(seeds, default=0))


@pytest.mark.parametrize("bad", [0, -1, True, False, 2.0, "3", np.float32(4)])
def test_path_targets_must_be_a_positive_int(bad):
    why = graphed.paths_refusal(_split(), 4, bad)
    assert why == "path_targets must be a positive int, got %r" % (bad,)


@pytest.mark.parametrize("T", [1, 32, np.int64(7), np.int32(1000)])
def test_positive_ints_are_admitted(T):
    assert graphed.paths_refusal(_split(), 4, T) is None


def test_workspace_past_int32_indexing_is_refused_at_the_boundary():
    """B is the largest batch, min(batch_size, num_data): (1 + T) * 65 536 cells fit up to T = 32 766."""
    split = _split(num_data=1, N=2 ** 16, seeds=(1,))
    assert graphed.paths_refusal(split, 8, 32766) is None
    why = graphed.paths_refusal(split, 8, 32767)
    assert why == ("path_targets 32767: the BFS workspace of a batch, B * (max_seeds + T) * N = 1 * (1 + 32767) * "
                   "65536, overflows int32 indexing")
    split = _split(num_data=100, N=1000, seeds=(5,))
    assert (20 * (5 + 107_369) * 1000 <= INT_MAX) and (20 * (5 + 107_370) * 1000 > INT_MAX)
    assert graphed.paths_refusal(split, 20, 107_369) is None
    assert graphed.paths_refusal(split, 20, 107_370).startswith("path_targets 107370: the BFS workspace")


def test_existing_refusals_come_first():
    """start_eval checks the split and the batch size before path_targets, with their messages."""
    step = graphed.GraphedStep.__new__(graphed.GraphedStep)
    L = SplitLoader(seed=1, num_questions=4, max_local_entity=20)
    for bad in (0, True, 2.5):
        with pytest.raises(ValueError, match="^start_eval: the split must be a loader.DeviceSplit, got SplitLoader$"):
            step.start_eval(L, 4, path_targets=bad)


def test_seed_counts_and_max_seeds():
    qe = np.zeros((5, 6))
    qe[0, [0, 3]] = 1.0
    qe[1, 5] = -2.0                        # nonzero counts, whatever its value
    qe[2, 1] = 1e-50                       # zero once in fp32, the table the split uploads
    qe[3, :] = 0.5
    counts = loader.seed_counts(qe)
    assert counts.dtype == np.int64 and counts.tolist() == [2, 1, 0, 6, 0]
    L = SplitLoader(seed=2, num_questions=6, max_local_entity=15)
    L.query_entities[2, [4, 7]] = 1.0
    L.query_entities[5] = 0.0
    split = loader.DeviceSplit.__new__(loader.DeviceSplit)
    split.loader, split._seed_counts = L, None
    assert split.seed_counts().tolist() == [1, 1, 3, 1, 1, 0]
    assert split.max_seeds() == 3
    assert split.seed_counts() is split.seed_counts()           # counted once and kept
    split.loader, split._seed_counts = SplitLoader(seed=2, num_questions=0, max_local_entity=15), None
    assert split.max_seeds() == 0


def test_record_sizes_and_layout():
    """Node offsets, the total, node counts, the [S, T] pair blocks and the node records: contiguous, aligned, sized by
    the split's non-pad entities (the candidate records' capacity)."""
    L = SplitLoader(seed=3, num_questions=9, max_local_entity=40)
    cap = loader.candidate_capacity(L.candidate_entities, NE)
    assert cap == sum(int((row != NE).sum()) for row in L.candidate_entities)
    n, S, T = 9, 3, 5
    nbytes = graphed._EvalPaths.nbytes(n, S, T, cap)
    assert nbytes == 8 * n + 8 + 4 * n + 4 * n * S * T + 4 * cap
    v = graphed._EvalPaths.views(np.zeros(nbytes, dtype=np.uint8), n, S, T, cap)
    assert [(k, a.dtype.name, a.shape) for k, a in v.items()] == [
        ("node_off", "int64", (n,)), ("node_total", "int64", (1,)), ("node_count", "int32", (n,)),
        ("pair_dist", "int32", (n, S, T)), ("nodes", "int32", (cap,))]
    base = blob_start = v["node_off"].__array_interface__["data"][0]
    for a in v.values():                    # back to back, each at a multiple of its element size
        start = a.__array_interface__["data"][0]
        assert start == blob_start and (start - base) % a.itemsize == 0
        blob_start = start + a.nbytes
    assert blob_start - base == nbytes


def test_decode_restated_on_hand_made_records():
    """Three questions: two nodes and a 2 x 1 block, no seeds (an empty set and a 0 x 3 block), one node on a path of
    a source equal to its target; the blocks are cut to each question's counts."""
    n, S, T, cap = 3, 2, 3, 6
    blob = np.zeros(graphed._EvalPaths.nbytes(n, S, T, cap), dtype=np.uint8)
    v = graphed._EvalPaths.views(blob, n, S, T, cap)
    v["node_off"][:] = [0, 2, 2]
    v["node_count"][:] = [2, 0, 1]
    v["node_total"][0] = 3
    v["nodes"][:] = [4, 9, 7, -1, -1, -1]
    v["pair_dist"][:] = -1
    v["pair_dist"][0, :2, 0] = [1, -1]
    v["pair_dist"][2, 0, :2] = [0, 3]
    sets, blocks = graphed._EvalPaths.decode(graphed._EvalPaths.views(blob, n, S, T, cap), [2, 0, 1], [1, 3, 2])
    assert sets == [[4, 9], [], [7]]
    assert [b.shape for b in blocks] == [(2, 1), (0, 3), (1, 2)]
    assert blocks[0].tolist() == [[1], [-1]] and blocks[2].tolist() == [[0, 3]]
    assert all(b.dtype == np.int32 for b in blocks)


def test_run_without_paths_refuses_paths():
    run = graphed.EvalRun(None, None, None, 0, None)
    with pytest.raises(ValueError, match="EvalRun.paths: the evaluation was started without path_targets"):
        run.paths()


@pytest.mark.parametrize("job,ok", [((1, 2, 3), False), ((1, 2), True), ([1, 2], True), ((1, 2, 3, 4), False)])
def test_sweep_job_form(job, ok):
    """A three-element evaluation job is (DeviceSplit, batch_size, path_targets); any other form is refused by its
    shape, before the start_eval checks."""
    from test_sweep_host import _cpu_model, _member
    step = graphed.GraphedStep(_cpu_model(), NE)
    why = graphed._job_refusal(_member(step), job, False)
    if ok:
        assert why.startswith("start_eval: the split must be a loader.DeviceSplit")
    else:
        assert why.startswith("Sweep.start_evals: a job is (split, batch_size[, path_targets]) or None")


# ---- the entry point -------------------------------------------------------------------------------------------------

def _types():
    P, I64, I, SZ = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_size_t
    return [P, I64, I64, I, I64, I64, P, P, P, I, I] + [P] * 8 + [I64, P, P, P, SZ, P]


def test_header_declaration_and_binding():
    I = ctypes.c_int
    assert _lib.SIGNATURES["gr_eval_step_paths"] == (I, _types())
    assert _lib.load().gr_eval_step_paths.argtypes == _types()
    assert _lib.SIGNATURES["gr_eval_paths_workspace_bytes"] == (
        ctypes.c_size_t, [ctypes.c_int, ctypes.c_int64, ctypes.c_int, ctypes.c_int])


def test_workspace_bytes():
    lib = _lib.load()
    B, N, S, T = 3, 50, 2, 4
    want = 4 * (B * (S + T) * N + B * S + B + B * T + B + B + 1) + B * N + 16
    assert lib.gr_eval_paths_workspace_bytes(B, N, S, T) == want
    assert lib.gr_eval_paths_workspace_bytes(B, N, 0, T) == 4 * (B * T * N + 3 * B + B * T + 1) + B * N + 16
    for bad in ((0, N, S, T), (B, 0, S, T), (B, N, -1, T), (B, N, S, 0)):
        assert lib.gr_eval_paths_workspace_bytes(*bad) == 0


def _paths(**over):
    a = dict(cursor=PTR, steps=3, batch_size=4, B=4, num_data=10, N=16, query_entities=PTR, cand_idx=PTR,
             cand_count=PTR, S=2, T=3, rowptr_t=PTR, src_t=PTR, rowptr_h=PTR, src_h=PTR, node_off=PTR, node_count=PTR,
             pair_dist=PTR, nodes=PTR, capacity=100, node_total=PTR, eval_status=PTR, workspace=None,
             workspace_bytes=0, stream=None)
    a.update(over)
    lib = _lib.load()
    return lib.gr_eval_step_paths(*a.values()), lib.gr_last_error().decode()


@pytest.mark.parametrize("over,msg", [
    (dict(cursor=None), "null pointer"), (dict(query_entities=None), "null pointer"), (dict(cand_idx=None), "null"),
    (dict(cand_count=None), "null pointer"), (dict(rowptr_t=None), "null pointer"), (dict(src_t=None), "null pointer"),
    (dict(rowptr_h=None), "null pointer"), (dict(src_h=None), "null pointer"),
    (dict(node_off=None), "null output"), (dict(node_count=None), "null output"), (dict(pair_dist=None), "null output"),
    (dict(nodes=None), "null output"), (dict(node_total=None), "null output"), (dict(eval_status=None), "null output"),
    (dict(B=0), "need 0 < B <= batch_size"), (dict(B=5), "need 0 < B <= batch_size"),
    (dict(steps=-1), "need 0 < B <= batch_size, steps >= 0"), (dict(num_data=-1), "need 0 < B"),
    (dict(N=0), "N must be in [1, INT_MAX]"), (dict(N=2 ** 31), "N must be in [1, INT_MAX]"),
    (dict(S=-1), "need S >= 0 and T > 0"), (dict(T=0), "need S >= 0 and T > 0"),
    (dict(B=1, batch_size=1, N=2 ** 20, S=1, T=2047), "B * (S + T) * N overflows int32 indexing"),
    (dict(capacity=-1), "capacity must be >= 0")])
def test_entry_refusals(over, msg):
    rc, err = _paths(**over)
    assert rc == -1 and err.startswith("gr_eval_step_paths: invalid argument: " + msg)


def test_entry_refuses_a_small_workspace():
    lib = _lib.load()
    need = lib.gr_eval_paths_workspace_bytes(4, 16, 2, 3)
    rc, err = _paths(workspace=PTR, workspace_bytes=need - 1)
    assert rc == -3 and err == "gr_eval_step_paths: workspace too small (%d < %d)" % (need - 1, need)
    rc, err = _paths(workspace=None, workspace_bytes=need)
    assert rc == -3
