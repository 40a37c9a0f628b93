"""CPU: the host logic of graphed.Sweep -- the step-major replay order with members dropping out, the per-member
``np.random`` stand-in around ``reset_batches``, the refusal of members that share a model or a device-less or mixed
placement, and the job checks, which refuse with the messages of ``start_epoch`` / ``start_eval``.  The GPU half is
tests/test_sweep_gpu.py."""
import types

import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import graphed, synthetic as S

from test_device_split_host import SplitLoader

NE, NR, NW = 3000, 40, 100


def _cpu_model(name="ReaRev"):
    torch.manual_seed(0)
    return {"ReaRev": G.ReaRev, "NSM": G.NSM}[name](dict(S.model_args(name, entity_dim=16, use_cuda=False)), NE, NR, NW)


# ---- the replay order ------------------------------------------------------------------------------------------------

def test_replay_schedule_is_step_major_and_members_drop_out():
    assert graphed.replay_schedule([3, 1, 2]) == [(0, 0), (1, 0), (2, 0), (0, 1), (2, 1), (0, 2)]
    assert graphed.replay_schedule([1, 4]) == [(0, 0), (1, 0), (1, 1), (1, 2), (1, 3)]


def test_replay_schedule_of_one_job_is_its_steps_in_order():
    assert graphed.replay_schedule([5]) == [(0, s) for s in range(5)]


@pytest.mark.parametrize("steps,want", [([], []), ([0], []), ([0, 0], []), ([0, 2], [(1, 0), (1, 1)])])
def test_replay_schedule_of_jobs_without_steps(steps, want):
    assert graphed.replay_schedule(steps) == want


@pytest.mark.parametrize("steps", [[7, 3, 7, 1], [2, 9], [4, 4, 4]])
def test_replay_schedule_replays_every_step_once_in_each_jobs_order(steps):
    sched = graphed.replay_schedule(steps)
    assert len(sched) == sum(steps)
    for k, n in enumerate(steps):
        assert [s for j, s in sched if j == k] == list(range(n))
    assert [s for _j, s in sched] == sorted(s for _j, s in sched)


# ---- np.random per member --------------------------------------------------------------------------------------------

def test_numpy_random_stands_in_for_the_global_stream_inside_the_block_only():
    np.random.seed(1)
    outside = np.random.get_state()
    rs = np.random.RandomState(7)
    want = np.random.RandomState(7).permutation(40)
    with graphed._numpy_random(rs):
        got = np.random.permutation(40)
    np.testing.assert_array_equal(got, want)
    assert _same_state(np.random.get_state(), outside)         # the global stream did not move
    twin = np.random.RandomState(7)
    twin.permutation(40)
    assert _same_state(rs.get_state(), twin.get_state())       # the member's stream moved by the draw


def test_numpy_random_orders_a_loader_as_the_global_stream_at_the_same_state():
    L = SplitLoader(seed=5, num_questions=23, max_local_entity=20, facts_hi=50)
    rs = np.random.RandomState(11)
    np.random.seed(3)
    with graphed._numpy_random(rs):
        L.reset_batches(is_sequential=False)
    member_order = np.array(L.batches)
    np.random.seed(11)
    L.reset_batches(is_sequential=False)
    np.testing.assert_array_equal(member_order, L.batches)


def test_numpy_random_restores_the_global_stream_when_the_block_raises():
    np.random.seed(2)
    outside = np.random.get_state()
    rs = np.random.RandomState(3)
    with pytest.raises(KeyError):
        with graphed._numpy_random(rs):
            np.random.rand(3)
            raise KeyError("x")
    assert _same_state(np.random.get_state(), outside)


def test_numpy_random_of_none_is_the_global_stream():
    np.random.seed(4)
    with graphed._numpy_random(None):
        a = np.random.rand(3)
    np.random.seed(4)
    np.testing.assert_array_equal(a, np.random.rand(3))


def _same_state(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


# ---- members -----------------------------------------------------------------------------------------------------

def test_members_must_be_graphed_steps():
    with pytest.raises(ValueError, match="Sweep: member 1 is a Linear; members are GraphedTrainStep"):
        graphed._check_members([graphed.GraphedStep(_cpu_model(), NE), torch.nn.Linear(2, 2)])
    with pytest.raises(ValueError, match="Sweep: no members"):
        graphed._check_members([])


def test_the_same_model_in_two_members_is_refused():
    m = _cpu_model()
    steps = [graphed.GraphedStep(_cpu_model("NSM"), NE), graphed.GraphedStep(m, NE), graphed.GraphedStep(m, NE)]
    with pytest.raises(ValueError, match="Sweep: members 1 and 2 hold the same model"):
        graphed._check_members(steps)


def test_members_on_the_cpu_are_refused():
    with pytest.raises(ValueError, match="Sweep: the members' models are on cpu; a sweep runs on one CUDA device"):
        graphed._check_members([graphed.GraphedStep(_cpu_model(), NE), graphed.GraphedStep(_cpu_model("NSM"), NE)])


def test_members_on_different_devices_are_refused():
    a, b = graphed.GraphedStep(_cpu_model(), NE), graphed.GraphedStep(_cpu_model("NSM"), NE)
    a.device, b.device = torch.device("cuda", 0), torch.device("cuda", 1)
    with pytest.raises(ValueError, match=r"Sweep: members on different devices \(cuda:0, cuda:1\)"):
        graphed._check_members([a, b])
    b.device = torch.device("cuda", 0)
    graphed._check_members([a, b])                              # one device: accepted


# ---- jobs --------------------------------------------------------------------------------------------------------

def _member(step):
    return types.SimpleNamespace(step=step, eval_step=lambda: step)


def _message(fn):
    with pytest.raises(ValueError) as e:
        fn()
    return str(e.value)


def test_evaluation_jobs_are_refused_with_start_evals_messages():
    step = graphed.GraphedStep(_cpu_model(), NE)
    for job in [(object(), 4), ([1, 2], 0)]:
        want = _message(lambda: step.start_eval(*job))
        assert want.startswith("start_eval: the split must be a loader.DeviceSplit")
        assert graphed._job_refusal(_member(step), job, False) == want


def test_training_jobs_are_refused_with_start_epochs_messages():
    step = graphed.GraphedTrainStep.__new__(graphed.GraphedTrainStep)     # no CUDA model on this machine
    step.optimizer = None
    job = (object(), 4, 0.0)
    want = _message(lambda: step.start_epoch(*job))
    assert want == "train_epoch: an epoch steps the optimizer in its graphs: build the step with optimizer="
    assert graphed._job_refusal(_member(step), job, True) == want


def test_a_training_job_for_an_evaluation_member_is_refused():
    step = graphed.GraphedStep(_cpu_model(), NE)
    why = graphed._job_refusal(_member(step), (object(), 4, 0.0), True)
    assert why.startswith("Sweep.start_epochs: a GraphedStep member evaluates only")


@pytest.mark.parametrize("training,job", [(True, (1, 2)), (False, (1, 2, 3)), (True, "split"), (False, 4)])
def test_jobs_that_are_not_argument_tuples_are_refused(training, job):
    step = graphed.GraphedStep(_cpu_model(), NE)
    why = graphed._job_refusal(_member(step), job, training)
    assert why.startswith("Sweep.%s: a job is (split, batch_size" % ("start_epochs" if training else "start_evals"))


def test_a_member_without_a_job_sits_out():
    step = graphed.GraphedStep(_cpu_model(), NE)
    assert graphed._job_refusal(_member(step), None, True) is None
    assert graphed._job_refusal(_member(step), None, False) is None


# ---- what members must not share ----------------------------------------------------------------------------------

# containers kept at module or class level that are not scratch a graph writes: constants, and the weight cache, whose
# entries belong to one weight tensor (so to one model) and which a graph inside graph_private_weights never reads
NOT_SHARED_SCRATCH = {"gnn_rag_b200.ops._CACHE", "gnn_rag_b200.ops._INDEX_BYTES", "gnn_rag_b200.ops.GraftGraph._MESSAGES",
                      "gnn_rag_b200.modules._LM_SPECS", "gnn_rag_b200.graphed._GraftLayout.LIST_NAMES",
                      "gnn_rag_b200.paths.ReasoningPaths._field_defaults"}


def _module_level_containers():
    import importlib
    import inspect
    found = {}
    for name in ("ops", "modules", "models", "autograd_path", "batching", "optim", "loader", "evaluate", "graphed",
                 "parallel", "paths"):
        mod = importlib.import_module("gnn_rag_b200." + name)
        for n, v in vars(mod).items():
            if isinstance(v, (dict, list, set)) and not n.startswith("__"):
                found["%s.%s" % (mod.__name__, n)] = (mod, n)
            if inspect.isclass(v) and v.__module__ == mod.__name__:
                for cn, cv in vars(v).items():
                    if isinstance(cv, (dict, list, set)) and not cn.startswith("__"):
                        found["%s.%s.%s" % (mod.__name__, n, cn)] = (v, cn)
    return found


def test_every_shared_container_is_a_members_own_scratch_or_not_scratch():
    """A dict the forwards keep per shape rather than per model is written by every graph of that shape; members that
    replay side by side each need their own (graphed._member_scope).  A new one must join graphed._shared_scratch."""
    found = _module_level_containers()
    scratch = {(owner, name) for owner, name in graphed._shared_scratch()}
    for key, where in found.items():
        assert where in scratch or key in NOT_SHARED_SCRATCH, key
    assert scratch <= set(found.values())
    assert NOT_SHARED_SCRATCH <= set(found)


# ---- a refusal while planning --------------------------------------------------------------------------------------

def test_a_refusal_while_planning_puts_every_members_order_back():
    loaders = [SplitLoader(seed=5, num_questions=9, max_local_entity=8, facts_hi=20) for _ in range(2)]
    rngs = [np.random.RandomState(1), np.random.RandomState(2)]
    before = [r.get_state() for r in rngs]
    batches = [L.batches for L in loaders]

    def job(k, refuse):
        j = graphed._EpochJob(types.SimpleNamespace(loader=loaders[k]), types.SimpleNamespace(rng=rngs[k]))

        def start():
            with graphed._numpy_random(j.rng()):
                loaders[k].reset_batches(is_sequential=False)
            if refuse:
                raise ValueError("train_epoch: a batch overflows int32 indices; use index_dtype=torch.int64")
        j.start = start
        return j
    np.random.seed(7)
    outside = np.random.get_state()
    with pytest.raises(ValueError, match="overflows int32"):
        graphed._start_all([job(0, False), job(1, True)])
    for r, st in zip(rngs, before):
        assert _same_state(r.get_state(), st)
    for L, b in zip(loaders, batches):
        assert L.batches is b
    assert _same_state(np.random.get_state(), outside)
