"""Several runs side by side on one GPU (graphed.Sweep) against the same runs alone.

Under torch's deterministic flag, with model dropout and fact dropout on over shuffled splits, every member of a sweep
computes over two epochs the bits it computes alone -- ``start_epoch`` with torch's default CUDA generator at the
member's generator state and ``np.random`` at its ``RandomState`` -- in the losses, gradient norms, h1 / F1, recorded
seeds and status, the parameters, ``p.grad`` and the Adam state, and leaves its generator and ``RandomState`` where
the solo run leaves the global ones: for a ReaRev + NSM + GraftNet mix with different batch sizes and step counts,
two of them over one split, listed in either order, and for a one-member sweep.  Evaluation members return the
records, cases and ``.info`` bytes of ``start_eval`` alone, after their training epoch in the same sweep and as
evaluation-only members.  A warm sweep does not synchronise with the host, and the refusals come before any capture
with the messages of the single-run methods."""
import copy

import numpy as np
import pytest
import torch

from gnn_rag_b200 import graphed, loader

from test_clip_adam_gpu import _assert_same_training
import test_graft_train_epoch_gpu as graft_epoch
import test_train_epoch_gpu as kb_epoch
from test_device_split_host import NE
from test_eval_epoch_gpu import _evaluator

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
DROP, FACT_DROP = 0.2, 0.1


@pytest.fixture(autouse=True)
def _deterministic():
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    torch.use_deterministic_algorithms(True, warn_only=True)
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        yield
    torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])


class Run:
    """One training run: a model and its twin (a deep copy), each with its own Adam and graphed step."""

    def __init__(self, name, L, split, B):
        self.name, self.L, self.split, self.B = name, L, split, B
        if name == "GraftNet":
            self.m = graft_epoch._model(L, dropout=DROP)
        else:
            self.m = kb_epoch._model(name, L, dropout=DROP)
        self.twin = copy.deepcopy(self.m)
        make = graft_epoch._step if name == "GraftNet" else kb_epoch._step
        self.step, self.opt = make(self.m)
        self.twin_step, self.twin_opt = make(self.twin)

    def job(self):
        return (self.split, self.B, FACT_DROP)


def _splits():
    L_kb = kb_epoch._loader()
    L_g = graft_epoch._loader()
    return L_kb, loader.DeviceSplit(L_kb, dev, shuffle=True), L_g, loader.DeviceSplit(L_g, dev, shuffle=True)


def _streams(n, base):
    gens = [torch.Generator(device=dev).manual_seed(base + k) for k in range(n)]
    rngs = [np.random.RandomState(base + 50 + k) for k in range(n)]
    return gens, rngs


def _states(sweep):
    return [(g.get_state(), r.get_state()) for g, r in zip(sweep.generators, sweep.rngs)]


def _alone(state, fn):
    """``fn()`` with torch's default CUDA generator and ``np.random`` at a member's ``state``; -> (what it returned,
    the generator state and the ``np.random`` state it left)."""
    torch.cuda.set_rng_state(state[0])
    np.random.set_state(state[1])
    out = fn()
    return out, torch.cuda.get_rng_state(), np.random.get_state()


def _same_np_state(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


def _same_epoch(a, b):
    for x, y in [(a.losses, b.losses), (a.grad_norms, b.grad_norms), (a.h1, b.h1), (a.f1, b.f1), (a.seeds, b.seeds),
                 (a.status, b.status)]:
        assert (x is None) == (y is None)
        if x is not None:
            assert torch.equal(x, y)
    kb_epoch._same_result(a.result(), b.result())
    a.check()
    b.check()


def _member_equals_alone(run, before, after, sweep_run):
    """A member's epoch ``sweep_run`` against ``run``'s twin alone from the member's state ``before``; ``after``: the
    member's state once the sweep's epoch has started."""
    solo, gen_after, np_after = _alone(before, lambda: run.twin_step.start_epoch(*run.job()))
    _same_epoch(sweep_run, solo)
    assert sweep_run.seeds is not None and torch.unique(sweep_run.seeds).numel() == sweep_run.seeds.numel()
    _assert_same_training(run.twin, run.m, run.twin_opt, run.opt)
    assert torch.equal(after[0], gen_after)                   # only the member's replays advanced its generator
    assert _same_np_state(after[1], np_after)


@pytest.mark.parametrize("order", ["listed", "reversed"])
def test_members_are_bit_equal_to_their_solo_runs(order):
    """ReaRev (B 4, 6 steps) and NSM (B 3, 8 steps) over one kb split, GraftNet (B 5, 5 steps) over a graft split."""
    L_kb, kb, L_g, gs = _splits()
    runs = [Run("ReaRev", L_kb, kb, 4), Run("NSM", L_kb, kb, 3), Run("GraftNet", L_g, gs, 5)]
    gens, rngs = _streams(3, 100)
    if order == "reversed":
        runs, gens, rngs = runs[::-1], gens[::-1], rngs[::-1]      # each run keeps its generator and RandomState
    sweep = graphed.Sweep([r.step for r in runs], generators=gens, rngs=rngs)
    for _epoch in range(2):
        before = _states(sweep)
        got = sweep.start_epochs([r.job() for r in runs])
        after = _states(sweep)
        last_kb = max(k for k, r in enumerate(runs) if r.split is kb)
        ids_after_sweep = list(L_kb.sample_ids)
        for k, (r, run) in enumerate(zip(runs, got)):
            _member_equals_alone(r, before[k], after[k], run)
            if k == last_kb:                 # the shared split's sample_ids: the last member's over it
                assert list(L_kb.sample_ids) == ids_after_sweep


def test_one_member_sweep_is_the_solo_epoch():
    L_kb, kb, _L_g, _gs = _splits()
    run = Run("ReaRev", L_kb, kb, 4)
    gens, rngs = _streams(1, 300)
    sweep = graphed.Sweep([run.step], generators=gens, rngs=rngs)
    for _epoch in range(2):
        before = _states(sweep)
        got, = sweep.start_epochs([run.job()])
        _member_equals_alone(run, before[0], _states(sweep)[0], got)


def test_default_streams_are_drawn_once_and_differ_per_member():
    L_kb, kb, _L_g, _gs = _splits()
    runs = [Run("ReaRev", L_kb, kb, 4), Run("NSM", L_kb, kb, 4)]
    torch.manual_seed(5)
    np.random.seed(6)
    sweep = graphed.Sweep([r.step for r in runs])
    a, b = sweep.generators
    assert a.initial_seed() != b.initial_seed()
    assert sweep.rngs[0].randint(2 ** 31) != sweep.rngs[1].randint(2 ** 31)


def _same_eval(a, b, tables):
    ra, rb = a.result(), b.result()
    for x, y in zip(ra[:6], rb[:6]):
        np.testing.assert_array_equal(x, y)
    assert len(ra[6]) == len(rb[6])
    for x, y in zip(ra[6], rb[6]):
        for f in ("idx", "ent", "prob"):
            np.testing.assert_array_equal(getattr(x, f), getattr(y, f))
    assert (a.seeds is None) == (b.seeds is None) and (a.seeds is None or torch.equal(a.seeds, b.seeds))
    a.check()
    b.check()
    assert a.info(tables).tobytes() == b.info(tables).tobytes()


def test_evaluation_members_equal_start_eval_alone(tmp_path):
    """Member 0 trains ReaRev and then evaluates it in the same sweep; member 1 only evaluates an NSM model; member 2
    trains GraftNet and sits the evaluation out."""
    L_kb, kb, L_g, gs = _splits()
    train, g_run = Run("ReaRev", L_kb, kb, 4), Run("GraftNet", L_g, gs, 5)
    m_eval = kb_epoch._model("NSM", L_kb).eval()
    m_eval_twin = copy.deepcopy(m_eval)
    gens, rngs = _streams(3, 400)
    sweep = graphed.Sweep([train.step, graphed.GraphedStep(m_eval, NE), g_run.step], generators=gens, rngs=rngs)
    tables = _evaluator("ReaRev", train.m, L_kb, tmp_path, "sweep", train.m.eps).info_tables(kb)
    before = _states(sweep)
    epochs = sweep.start_epochs([train.job(), None, g_run.job()])
    assert epochs[1] is None
    mid = _states(sweep)
    evals = sweep.start_evals([(kb, 4), (kb, 5), None])
    end = _states(sweep)
    assert evals[2] is None
    _member_equals_alone(train, before[0], mid[0], epochs[0])
    _member_equals_alone(g_run, before[2], mid[2], epochs[2])
    for k, (m, B) in enumerate([(train.twin, 4), (m_eval_twin, 5)]):
        solo, gen_after, _np_after = _alone(mid[k], lambda: graphed.GraphedStep(m, NE).start_eval(kb, B))
        _same_eval(evals[k], solo, tables)
        assert torch.equal(end[k][0], gen_after)


def test_warm_sweep_does_not_synchronise():
    L_kb, kb, L_g, gs = _splits()
    runs = [Run("ReaRev", L_kb, kb, 4), Run("GraftNet", L_g, gs, 5)]
    m_eval = kb_epoch._model("NSM", L_kb).eval()
    gens, rngs = _streams(3, 500)
    sweep = graphed.Sweep([runs[0].step, runs[1].step, graphed.GraphedStep(m_eval, NE)], generators=gens, rngs=rngs)
    orders = [r.get_state() for r in sweep.rngs]
    jobs = [runs[0].job(), runs[1].job(), None]
    evals = [(kb, 4), None, (kb, 4)]
    sweep.start_epochs(jobs)
    sweep.start_evals(evals)
    graphs = [len(m.step._cache) for m in sweep.members] + [len(sweep.eval_step(0)._cache)]
    for r, st in zip(sweep.rngs, orders):
        r.set_state(st)                  # the same orders: every graph the sweep needs is captured
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = sweep.start_epochs(jobs)
        got_evals = sweep.start_evals(evals)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert [len(m.step._cache) for m in sweep.members] + [len(sweep.eval_step(0)._cache)] == graphs
    for run in got[:2] + [got_evals[0], got_evals[2]]:
        run.check()
    assert all(np.isfinite(run.result()[0]) for run in got[:2])


def _message(fn):
    with pytest.raises(ValueError) as e:
        fn()
    return str(e.value)


def test_the_same_model_in_two_members_is_refused():
    L_kb, kb, _L_g, _gs = _splits()
    run = Run("ReaRev", L_kb, kb, 4)
    with pytest.raises(ValueError, match="Sweep: members 0 and 1 hold the same model"):
        graphed.Sweep([run.step, graphed.GraphedStep(run.m, NE)])


@pytest.mark.parametrize("bad", ["batch_size", "fact_dropout", "graft_split", "no_optimizer"])
def test_a_refused_training_job_raises_its_message_before_any_capture(bad):
    L_kb, kb, _L_g, gs = _splits()
    ok, other = Run("ReaRev", L_kb, kb, 4), Run("NSM", L_kb, kb, 4)
    step = other.step
    job = {"batch_size": (kb, 0, 0.0), "fact_dropout": (kb, 4, 1.5), "graft_split": (gs, 4, 0.0),
           "no_optimizer": (kb, 4, 0.0)}[bad]
    if bad == "no_optimizer":
        step = graphed.GraphedTrainStep(other.m)
    gens, rngs = _streams(2, 600)
    sweep = graphed.Sweep([ok.step, step], generators=gens, rngs=rngs)
    states = _states(sweep)
    batches = np.array(L_kb.batches)
    want = _message(lambda: step.start_epoch(*job))
    assert _message(lambda: sweep.start_epochs([ok.job(), job])) == want
    assert len(ok.step._cache) == 0 and len(step._cache) == 0
    assert all(_same_np_state(a[1], b[1]) for a, b in zip(states, _states(sweep)))
    np.testing.assert_array_equal(L_kb.batches, batches)      # no member's order was drawn


def test_refused_evaluation_jobs_and_training_jobs_for_evaluation_members():
    L_kb, kb, _L_g, gs = _splits()
    ok = Run("ReaRev", L_kb, kb, 4)
    ev = graphed.GraphedStep(kb_epoch._model("NSM", L_kb), NE)
    sweep = graphed.Sweep([ok.step, ev], *_streams(2, 700))
    want = _message(lambda: ev.start_eval(gs, 4))
    assert want.startswith("start_eval: a ReaRev / NSM model evaluates a kb split")
    assert _message(lambda: sweep.start_evals([(kb, 4), (gs, 4)])) == want
    assert _message(lambda: sweep.start_evals([(kb, -1), None])) == _message(lambda: ev.start_eval(kb, -1))
    assert _message(lambda: sweep.start_epochs([ok.job(), ok.job()])).startswith(
        "Sweep.start_epochs: a GraphedStep member evaluates only")
    assert _message(lambda: sweep.start_epochs([ok.job()])).startswith("Sweep.start_epochs: 1 jobs for 2 members")
    assert len(ok.step._cache) == 0 and len(ev._cache) == 0 and len(sweep.eval_step(0)._cache) == 0


def _perturbed(m, seed):
    """``m`` with every parameter moved by a little noise of ``seed``: another run of the same family and shape."""
    g = torch.Generator(device=dev).manual_seed(seed)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.05 * torch.randn(p.shape, device=dev, generator=g))
    return m


@pytest.mark.parametrize("name", ["ReaRev", "GraftNet"])
def test_evaluation_members_of_one_family_and_shape_equal_start_eval_alone(name, tmp_path):
    """Three evaluation-only runs of one family over one split: the forwards keep their operand planes, relation
    features and tile counter per shape, and each member's graphs write copies of their own."""
    L_kb, kb, L_g, gs = _splits()
    L, split = (L_g, gs) if name == "GraftNet" else (L_kb, kb)
    make = (lambda: graft_epoch._model(L)) if name == "GraftNet" else (lambda: kb_epoch._model(name, L))
    models = [_perturbed(make().eval(), 800 + k) for k in range(3)]
    twins = [copy.deepcopy(m) for m in models]
    gens, rngs = _streams(3, 800)
    sweep = graphed.Sweep([graphed.GraphedStep(m, NE) for m in models], generators=gens, rngs=rngs)
    tables = _evaluator(name, models[0], L, tmp_path, "same_shape", models[0].eps).info_tables(split)
    for _round in range(2):
        before = _states(sweep)
        got = sweep.start_evals([(split, 4)] * 3)
        end = _states(sweep)
        for k, (twin, run) in enumerate(zip(twins, got)):
            solo, gen_after, _np_after = _alone(before[k], lambda: graphed.GraphedStep(twin, NE).start_eval(split, 4))
            _same_eval(run, solo, tables)
            assert torch.equal(end[k][0], gen_after)
    probs = {tuple(np.concatenate([x.prob for x in r.result()[6]]).tolist()) for r in got}
    assert len(probs) == 3                                      # three different models
