"""Inference on the current weights after in-place training updates.

The inference forwards read their GEMM weights and relation tables pre-formatted (bf16 hi/lo splits) from a cache
that trusts ``tensor._version`` (ops._cached), and ``GraphedStep`` keys its serving graphs on the parameters'
versions.  Each case here warms every reader on a model, lets one writer update the parameters in place, and reads
again, twice: read, write, read, write, read.  After every round each reader's output is held to

- a cold twin, bit for bit: a fresh instance of the same args with ``load_state_dict(model.state_dict())``, whose
  tensors are new and whose cache is cold, through the same reader.  In round 0 the model is cold too, so that round
  checks that the twin reproduces itself on every path before later rounds rely on it;
- the oracle on the current parameters (``kgqa_oracle.forward`` on the state dict, ``graft_oracle.forward`` on a CPU
  copy), to ``test_parity_gpu``'s bound with ranking equivalence.

The readers: eager ``model(batch)``, ``GraphedStep(model)(batch)`` and ``submit`` / ``collect``, an ``Evaluator``
over the host loader, and an ``Evaluator(step=)`` over a ``DeviceSplit`` (evaluation-epoch graphs).  The writers: eager
``torch.optim.Adam`` and ``load_state_dict`` (controls), eager backward + ``optim.ClipAdam``, the graphed training
step with its fused optimizer, ``train_epoch`` and ``Sweep.start_epochs``.  Two guards keep a case from passing
without exercising anything: the model's parameters own cache entries after the first read, and the oracle's
``pred_dist`` moves by more than ten times the bound with every update.

Also the contract the fix rests on: ``ClipAdam.prepare`` / ``advance`` bump the version of every parameter they
update and of nothing else, and the cache then re-formats."""
import gc

import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import evaluate, graphed, loader, ops, optim, synthetic as S
from oracle import graft_oracle, kgqa_oracle as O

import test_graft_train_epoch_gpu as graft_epoch
import test_train_epoch_gpu as kb_epoch
from test_clip_adam_gpu import _trainable
from test_device_split_host import NE, NW, SplitLoader
from test_eval_epoch_gpu import _evaluator, _run
from test_parity_gpu import RTOL, assert_ranking_equivalent, rel_err

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
EPS = 0.95
LR = 2e-2              # large enough that every update moves pred_dist by more than 10 * RTOL
LR_D200 = 1e-3         # at D = 200 a larger step sharpens the logits until fp32 rounding alone exceeds RTOL
STEPS = 2              # optimizer steps per write of the step writers


@pytest.fixture(autouse=True)
def _deterministic():
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    torch.use_deterministic_algorithms(True, warn_only=True)
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        yield
    torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])


def _args(name, D):
    args = S.model_args(name, entity_dim=D, use_cuda=True, word_dim=64, linear_dropout=0.0, lm_dropout=0.0)
    if name == "ReaRev":
        args.update(num_ins=2, num_iter=2, num_gnn=2)
    elif name == "NSM":
        args.update(num_step=2)
    else:
        args.update(num_layer=2)
    return args


def _model(name, L, D, use_cuda=True):
    torch.manual_seed(0)
    cls = {"ReaRev": G.ReaRev, "NSM": G.NSM, "GraftNet": G.GraftNet}[name]
    m = cls(dict(_args(name, D), use_cuda=use_cuda), NE, L.num_kb_relation, NW)
    return m.cuda() if use_cuda else m


def _d200_loader():
    """Nine questions of up to 2 000 entities: B * N = 18 000 rows, enough for the one-kernel dense layer."""
    L = SplitLoader(seed=9, num_questions=9, max_local_entity=2000, facts_lo=1500, facts_hi=4000)
    assert 9 * 2000 >= ops.FUSED_MIN_ROWS
    return L


class Subject:
    """A model, its data and the readers it keeps across the rounds, so that their caches and graphs stay warm."""

    def __init__(self, name, L, B, D, tmp_path, lr=LR):
        self.name, self.L, self.B, self.D, self.tmp_path = name, L, B, D, tmp_path
        self.m = _model(name, L, D)
        self.split = loader.DeviceSplit(L, dev)
        self.train_split = loader.DeviceSplit(L, dev, shuffle=True)
        self.batch = L.get_batch(0, B, 0.0, test=True)
        self.train_batch = L.get_batch(1 if L.num_data > B else 0, B, 0.0)
        self.readers = Readers(self, self.m, "model")
        self.opt = torch.optim.Adam(_trainable(self.m), lr=lr)
        cls = graphed.GraphedGraftTrainStep if name == "GraftNet" else graphed.GraphedTrainStep
        self.train_step = cls(self.m, optimizer=self.opt, max_norm=1.0)

    def twin(self):
        t = _model(self.name, self.L, self.D)
        t.load_state_dict(self.m.state_dict())
        return t

    def oracle(self):
        """pred_dist of the oracle on the model's current parameters (CPU fp32) and its candidate lists."""
        if self.name == "GraftNet":
            cpu = _model(self.name, self.L, self.D, use_cuda=False)
            cpu.load_state_dict({k: v.cpu() for k, v in self.m.state_dict().items()})
            want = torch.from_numpy(graft_oracle.forward(cpu.eval(), self.batch)["pred_dist"])
        else:
            sd = {k: v.detach().cpu().clone() for k, v in self.m.state_dict().items()}
            want = O.forward(sd, _args(self.name, self.D), NE, NW, self.batch)[2]
        return want, O.rank_candidates(self.batch[0], self.batch[1], want.numpy(), NE, EPS)


class Readers:
    """Every inference path over one model: eager, GraphedStep (call and submit / collect), the per-batch Evaluator
    over the host loader and the evaluation epoch."""

    def __init__(self, subj, m, tag):
        self.subj, self.m, self.tag = subj, m, tag
        self.step = graphed.GraphedStep(m, NE, eps=EPS)
        self.host = _evaluator(subj.name, m, subj.L, subj.tmp_path, tag + "_host", EPS)
        self.epoch = _evaluator(subj.name, m, subj.L, subj.tmp_path, tag + "_epoch", EPS, step=self.step)

    def read(self):
        s, m = self.subj, self.m
        m.eval()
        x = s.batch[:-1]
        with torch.no_grad():
            eager = m(x)[2].clone()
        eager_ret = evaluate.retrieve(eager, m.last_batch, NE, EPS)[0]
        out = self.step(x)
        served = out.pred_dist.clone()
        served_ret = self.step.retrieve(out)[0]
        ret, _nbytes, loss, pred = self.step.collect(self.step.submit(x))
        collected = ([(r.idx.tolist(), r.ent.tolist(), r.prob.tobytes()) for r in ret], loss, pred.tolist())
        host = _run(self.host, s.L, s.B, s.tmp_path, self.tag + "_host")
        epoch = _run(self.epoch, s.split, s.B, s.tmp_path, self.tag + "_epoch")
        return dict(eager=eager, eager_ret=eager_ret, served=served, served_ret=served_ret, collected=collected,
                    host=host, epoch=epoch)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _against_twin(got, want, where):
    bad = []
    for k in ("eager", "served"):
        if not torch.equal(_bits(got[k]), _bits(want[k])):
            bad.append("%s: %s pred_dist differs from the cold twin's" % (where, k))
    if got["collected"] != want["collected"]:
        bad.append("%s: submit / collect differs from the cold twin's" % where)
    for k, what in (("host", "Evaluator over the host loader"), ("epoch", "Evaluator(step=) over a DeviceSplit")):
        for i, part in enumerate(("F1 / hit / EM", "case_ct", ".info bytes")):
            if got[k][i] != want[k][i]:
                bad.append("%s: %s: %s differ from the cold twin's" % (where, what, part))
    return bad


def _against_oracle(got, want, ref, where):
    bad = []
    for k in ("eager", "served"):
        err = rel_err(got[k].cpu(), want, 1e-30)
        if not err < RTOL:
            bad.append("%s: %s pred_dist rel_err %.3g vs the oracle" % (where, k, err))
            continue
        try:
            assert_ranking_equivalent(got[k + "_ret"], ref, want.numpy(), name="weight_updates_" + k)
        except AssertionError as e:
            bad.append("%s: %s ranking vs the oracle: %r" % (where, k, e))
    return bad


def _owns_cache_entries(m):
    ids = {id(p) for p in m.parameters()}
    return any(id(e[2]()) in ids for e in ops._CACHE.values())


def _rounds(subjects, write, rounds=3):
    """Read, then ``write(round)`` and read again, ``rounds - 1`` times; every read against the cold twin and the
    oracle.  Collects every mismatch before failing, so one run shows which readers go wrong."""
    bad, before = [], {}
    for r in range(rounds):
        if r:
            write(r)
        for s in subjects:
            where = "round %d, %s D=%d" % (r, s.name, s.D)
            got = s.readers.read()
            if r == 0:
                assert _owns_cache_entries(s.m), "%s: no cached weight belongs to the model" % where
            twin = s.twin()
            bad += _against_twin(got, Readers(s, twin, "twin%d" % r).read(), where)
            want, ref = s.oracle()
            bad += _against_oracle(got, want, ref, where)
            if r:
                moved = rel_err(want, before[id(s)], 1e-30)
                assert moved > 10 * RTOL, "%s: the update moved the oracle's pred_dist by only %.3g" % (where, moved)
            before[id(s)] = want
            del twin
            gc.collect()
    assert not bad, "\n".join(bad)


def _eager_backward(s):
    s.m.train()
    for p in s.m.parameters():
        p.grad = None
    s.m(s.train_batch, training=True)[0].backward()


def _write(kind, s):
    params = _trainable(s.m)
    if kind == "load":
        g = torch.Generator(device=dev).manual_seed(17)
        s.m.load_state_dict({k: v + 0.05 * torch.randn(v.shape, device=dev, generator=g) if v.is_floating_point()
                             else v for k, v in s.m.state_dict().items()})
    elif kind == "epoch":
        s.train_step.train_epoch(s.train_split, s.B, 0.0)
    else:
        for _ in range(STEPS):
            if kind == "graphed":
                s.m.train()
                s.train_step.step(s.train_batch)
                continue
            _eager_backward(s)
            if kind == "adam":
                s.opt.step()
            else:
                optim.ClipAdam(s.opt, params, [p.grad for p in params], max_norm=1.0).step()
    torch.cuda.synchronize()


WRITERS = ["adam", "load", "clip_adam", "graphed", "epoch"]


@pytest.mark.parametrize("writer", WRITERS)
@pytest.mark.parametrize("name", ["ReaRev", "NSM", "GraftNet"])
def test_readers_follow_in_place_updates_d50(name, writer, tmp_path):
    L = graft_epoch._loader() if name == "GraftNet" else kb_epoch._loader()
    s = Subject(name, L, kb_epoch.B, 50, tmp_path)
    _rounds([s], lambda r: _write(writer, s))
    if writer == "graphed":
        assert len(s.train_step._cache) == 1                 # versions are not part of the training graphs' key


@pytest.mark.parametrize("writer", ["clip_adam", "graphed"])
def test_readers_follow_in_place_updates_d200(writer, tmp_path):
    """The one-kernel dense layer with its K-order W and the sparse-prior fix-up with e2e.weight[:, :D]."""
    s = Subject("ReaRev", _d200_loader(), 9, 200, tmp_path, lr=LR_D200)
    _rounds([s], lambda r: _write(writer, s))


def test_readers_follow_a_sweep(tmp_path):
    """Sweep.start_epochs over a ReaRev and a GraftNet member; each model against its own twin afterwards."""
    L_kb, L_g = kb_epoch._loader(), graft_epoch._loader()
    subjects = [Subject("ReaRev", L_kb, kb_epoch.B, 50, tmp_path), Subject("GraftNet", L_g, kb_epoch.B, 50, tmp_path)]
    gens = [torch.Generator(device=dev).manual_seed(31 + k) for k in range(2)]
    sweep = graphed.Sweep([s.train_step for s in subjects], generators=gens,
                          rngs=[np.random.RandomState(41 + k) for k in range(2)])

    def write(r):
        runs = sweep.start_epochs([(s.train_split, s.B, 0.0) for s in subjects])
        for run in runs:
            run.result()
            run.check()
        torch.cuda.synchronize()
    _rounds(subjects, write)


# ---- the contract the cache relies on ------------------------------------------------------------------------------

def test_clip_adam_bumps_the_versions_it_updates():
    """prepare() and advance(n) bump ``_version`` of every parameter the optimizer updates, and of nothing else: not
    a clip-only parameter (with a gradient, outside the optimizer) nor one the optimizer holds without a gradient.
    The cached weight split of an updated parameter is then not current, and the relation planes are re-formatted."""
    torch.manual_seed(3)
    upd = [torch.nn.Parameter(torch.randn(96, 72, device=dev)) for _ in range(2)]
    clip_only = torch.nn.Parameter(torch.randn(40, device=dev))
    frozen = torch.nn.Parameter(torch.randn(7, 5, device=dev))
    params = upd + [clip_only, frozen]
    opt = torch.optim.Adam(upd + [frozen], lr=LR)
    grads = [torch.randn_like(p) for p in params[:3]] + [None]
    fused = optim.ClipAdam(opt, params, grads, max_norm=1.0)
    W, P = upd
    ops.clear_weight_cache()

    def ws_current():
        return ops._weight_ws(W, 96, 72, 0, 0, 4096)[1]

    def planes_fresh():
        hi, lo = ops.param_planes(P)
        want = [torch.zeros_like(hi) for _ in range(2)]
        ops.split_bf16(P.detach(), *want)
        return torch.equal(hi, want[0]) and torch.equal(lo, want[1])

    ws_current()
    assert ws_current() and planes_fresh()
    for advance in (lambda: fused.step(), lambda: fused.advance(3)):
        versions = [p._version for p in params]
        advance()
        torch.cuda.synchronize()
        now = [p._version for p in params]
        assert now[0] > versions[0] and now[1] > versions[1]
        assert now[2:] == versions[2:]
        assert not ws_current() and ws_current()
        assert planes_fresh()
    versions = [p._version for p in params]
    fused.advance(0)
    assert [p._version for p in params] == versions
    ops.clear_weight_cache()
