"""graphed.GraphedGraftTrainStep: GraftNet's ``model(batch, training=True)`` + ``loss.backward()`` + the train-time
metrics captured as one CUDA graph per batch shape.

Under torch.use_deterministic_algorithms the graphed step is bit-equal to the eager step: loss, pred_dist, pred, h1,
f1 and every parameter gradient, with the graft facts at and below their capacity, with none at all, under bf16
autocast and over a three-step Adam loop.  Without the flag the gradients agree within the atomics' rounding."""
import copy
import gc
import weakref

import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import autograd_path, batching, graphed, loader, ops, synthetic as S

from test_graftnet_host import load_model
from test_graphed_train_gpu import _assert_bit_equal, _det, _eager, _fp32_cudnn, _graphed, _no_dropout  # noqa: F401
from test_device_split_gpu import _loader, _model, _train_mode

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")

NE, NR, NW = 3000, 40, 100


def _synthetic(D=50, B=4, N=200, E=700, seed=3, dropout=0.0, lm_dropout=None, **over):
    args = S.model_args("GraftNet", entity_dim=D, num_layer=3, use_cuda=True, linear_dropout=dropout,
                        lm_dropout=dropout if lm_dropout is None else lm_dropout, **over)
    torch.manual_seed(seed)
    m = G.GraftNet(dict(args), NE, NR, NW).cuda().train()
    b = S.make_graft_batch(seed, B=B, N=N, E=E, num_entity=NE, num_relation=NR, num_word=NW, n_real="ragged",
                           use_inverse_relation=over.get("use_inverse_relation", False))
    return m, b


def _golden(name):
    m, g = load_model(name, "cuda")
    m = _no_dropout(m.cuda())
    if not isinstance(m.instruction.node_encoder, torch.nn.LSTM):
        m.instruction.node_encoder.eval()
    batch = list(g.batch[:9])
    if "answer_dist" in g.train:                              # the training goldens' answers; graft_hub_clamp: its own
        batch[8] = g.train["answer_dist"]
    return m, tuple(batch)


def _with_graft(batch, keep):
    """``batch`` with only the graft facts of the head-list entries ``keep`` (and their tail-list partners)."""
    (hb, hf, he, hv), (tb, te, tf, tv) = batch[3]
    keep = np.asarray(keep, dtype=np.int64)
    slots = set(zip(hb[keep].tolist(), hf[keep].tolist()))
    tk = np.array([(b, f) in slots for b, f in zip(tb.tolist(), tf.tolist())], dtype=bool)
    out = list(batch)
    out[3] = ((hb[keep], hf[keep], he[keep], np.asarray(hv)[keep]), (tb[tk], te[tk], tf[tk], np.asarray(tv)[tk]))
    return tuple(out)


def _at_capacity():
    """Exactly 1024 graft facts: the live count equals the capacity of their bucket."""
    m, b = _synthetic(D=50, B=4, N=200, E=900, seed=5)
    assert len(b[3][0][0]) > 1024
    b = _with_graft(b, np.arange(1024))
    assert len(b[3][0][0]) == len(b[3][1][0]) == graphed.fact_capacity(1024) == 1024
    return m, b


def _no_graft_facts():
    m, b = _synthetic(D=50, seed=6)
    return m, _with_graft(b, [])


def _one_question_without_facts():
    m, b = _synthetic(D=50, seed=7)
    hb = b[3][0][0]
    b = _with_graft(b, np.nonzero(hb != 1)[0])
    assert (b[3][0][0] != 1).all() and (b[3][1][0] != 1).all() and len(b[3][0][0]) > 0
    return m, b


def _case(name):
    if name == "d50_lstm":
        return _synthetic(D=50)
    if name == "d200":
        return _synthetic(D=200, B=3, N=300, E=1200)
    if name == "inverse_norm_rel":
        return _synthetic(D=64, use_inverse_relation=True, norm_rel=True)
    if name == "at_capacity":
        return _at_capacity()
    if name == "no_graft_facts":
        return _no_graft_facts()
    if name == "question_without_facts":
        return _one_question_without_facts()
    return _golden(name)


CASES = ["d50_lstm", "d200", "inverse_norm_rel", "at_capacity", "no_graft_facts", "question_without_facts",
         "graft_small", "graft_inverse", "graft_sbert_reltext", "graft_hub_clamp"]


@pytest.mark.parametrize("name", CASES)
def test_bit_equal_to_eager_under_the_deterministic_flag(name, monkeypatch):
    """graft_sbert_reltext: outside a capture the HuggingFace encoder drops an all-ones attention mask (a host check)
    and SDPA runs another kernel; under capture it always passes the mask.  The eager reference runs the encoder's
    capture branch, so that what is compared is the GraftNet step itself."""
    m, batch = _case(name)
    assert m.encode_type                                     # the TypeLayer kernels run in every case
    F = len(batch[3][0][0])
    assert F <= graphed.fact_capacity(F)
    _det(True)
    if name == "graft_sbert_reltext":
        from transformers import masking_utils
        monkeypatch.setattr(masking_utils, "is_tracing", lambda *a, **k: True)
    want = _eager(m, batch)
    monkeypatch.undo()
    step = graphed.GraphedGraftTrainStep(m)
    _assert_bit_equal(want, _graphed(step, batch))
    _assert_bit_equal(want, _graphed(step, batch))           # the replay of the captured key
    assert len(step._cache) == 1


@pytest.mark.parametrize("name", ["d50_lstm", "d200", "graft_hub_clamp", "graft_sbert_reltext"])
def test_close_to_eager_without_the_deterministic_flag(name):
    """fp32 atomics in the backward kernels: loss and pred_dist within 1e-5 relative, every gradient within 1e-4 of
    its own scale plus 1e-6 of the largest gradient (observed: printed)."""
    m, batch = _case(name)
    _det(False)
    want = _eager(m, batch)
    got = _graphed(graphed.GraphedGraftTrainStep(m), batch)
    assert abs(float(got[0]) - float(want[0])) <= 1e-5 * abs(float(want[0]))
    assert (got[2] - want[2]).abs().max().item() <= 1e-5 * want[2].abs().max().item() + 1e-9
    gmax = max(g.abs().max().item() for g in want[4].values())
    assert set(got[4]) == set(want[4])
    worst = 0.0
    for k, w in want[4].items():
        err = (got[4][k] - w).abs().max().item()
        scale = w.abs().max().item()
        if scale > 1e-3 * gmax:
            worst = max(worst, err / scale)
        assert err <= 1e-4 * scale + 1e-6 * gmax + 1e-9, (k, err, scale)
    print("%s: largest gradient error relative to the tensor's scale %.2e" % (name, worst))


@pytest.mark.parametrize("name", ["d50_lstm", "d200"])
def test_bf16_autocast_bit_equal_to_eager(name):
    m, batch = _case(name)
    _det(True)
    want = _eager(m, batch, torch.bfloat16)
    step = graphed.GraphedGraftTrainStep(m)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        got = _graphed(step, batch)
    _assert_bit_equal(want, got)
    assert len(step._cache) == 1
    _graphed(step, batch)                                    # outside autocast: another key, another graph
    assert len(step._cache) == 2


def test_three_step_adam_loop_bit_equal():
    """Replays read the weights the caller's clip + Adam step wrote in place."""
    m, batch = _case("d50_lstm")
    m2 = copy.deepcopy(m)
    _det(True)
    step = graphed.GraphedGraftTrainStep(m2)

    def loop(model, run):
        opt = torch.optim.Adam([p for p in model.parameters() if p.requires_grad], lr=5e-3)
        losses = []
        for _ in range(3):
            opt.zero_grad(set_to_none=True)
            losses.append(run(batch))
            torch.nn.utils.clip_grad_norm_([p for p in model.parameters() if p.requires_grad], 1.0)
            opt.step()
        return losses, {k: v.clone() for k, v in model.state_dict().items()}

    def eager(b):
        loss = m(b, training=True)[0]
        loss.backward()
        return loss.detach().clone()
    want = loop(m, eager)
    got = loop(m2, lambda b: step.step(b)[0].clone())
    assert len(step._cache) == 1
    assert [float(x) for x in want[0]] == [float(x) for x in got[0]]
    assert float(want[0][2]) != float(want[0][0])
    for k in want[1]:
        assert torch.equal(want[1][k], got[1][k]), k


def test_buckets_replay_and_lru_eviction():
    """Batches that differ in their graft fact count only: two in one capacity bucket replay one graph, two more
    buckets evict it."""
    m, base = _synthetic(D=50, E=2600)
    n = len(base[3][0][0])
    same = [base, _with_graft(base, np.arange(n - 40))]
    assert graphed.fact_capacity(n) == graphed.fact_capacity(n - 40)
    _det(True)
    step = graphed.GraphedGraftTrainStep(m, max_graphs=2)
    for b in same:
        _assert_bit_equal(_eager(m, b), _graphed(step, b))
    assert len(step._cache) == 1
    first = weakref.ref(next(iter(step._cache.values())))
    for k in (n // 2, n // 4):
        assert graphed.fact_capacity(k) != graphed.fact_capacity(n)
        b = _with_graft(base, np.arange(k))
        _assert_bit_equal(_eager(m, b), _graphed(step, b))
    assert len(step._cache) == 2
    gc.collect()
    assert first() is None                                  # the least recently used graph was released


def _step_without_sync(step, batch):
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = step.step(batch)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    return out


def test_replay_does_not_synchronise_with_the_host():
    m, batch = _synthetic(D=50, dropout=0.2)
    pinned = batching.pin_graft_batch(batch)
    step = graphed.GraphedGraftTrainStep(m)
    step.step(pinned)
    out = _step_without_sync(step, pinned)
    out.check()
    assert torch.isfinite(out[0]).item()


def test_device_split_batches_do_not_synchronise():
    L = _loader("GraftNet")
    m = _train_mode(_model("GraftNet", L, eval_mode=False))
    split = loader.DeviceSplit(L, dev, shuffle=True)
    step = graphed.GraphedGraftTrainStep(m)
    for it in (0, 1):                                         # the captures of both batches' buckets
        step.step(split.get_batch(it, 6, 0.1))
    graphs = len(step._cache)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        outs = [step.step(split.get_batch(it, 6, 0.1)) for it in (1, 0)]
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    outs[-1].check()
    assert len(step._cache) == graphs
    split.check()


def test_dropout_masks_are_fresh_on_every_replay(monkeypatch):
    """The fact-message masks (gr_graft_dropout_mask of the seeds the graph draws) and the linear dropout masks differ
    between replays, and keep about 1 - p."""
    p = 0.3
    m, batch = _synthetic(D=50, dropout=p, lm_dropout=0.0)     # the first two dropouts then see the same input
    seeds, drops = [], []
    orig = autograd_path._GraftAggregateFn.apply

    def spy(self_tab, head_tab, s, gg, seed, p_):
        seeds.append((seed, p_, gg.B * gg.max_fact))
        return orig(self_tab, head_tab, s, gg, seed, p_)
    monkeypatch.setattr(autograd_path._GraftAggregateFn, "apply", spy)
    m.reasoning.linear_drop_train.register_forward_hook(lambda mod, inp, out: drops.append((inp[0], out)))
    step = graphed.GraphedGraftTrainStep(m)
    step.step(batch)                                          # warm-ups and the capture: the last 3 / k are captured
    k = len(drops) // 3
    seeds, drops = seeds[-3:], drops[-k:][:2]                 # layer 0: drop(query), drop(h)
    assert all(sd is not None and p_ == pytest.approx(p) for sd, p_, _ in seeds)
    D = m.entity_dim

    def masks():
        fact = [ops.graft_dropout_mask(sd, p, S_, D) for sd, _p, S_ in seeds]
        lin = [(o != 0)[i != 0] for i, o in drops]
        return fact, lin
    a = masks()
    step.step(batch)
    b = masks()
    for x, y in zip(a[0] + a[1], b[0] + b[1]):
        assert not torch.equal(x, y)
        frac = float(y.double().mean())
        assert abs(frac - (1 - p)) <= 5 * np.sqrt(p * (1 - p) / y.numel()), frac
    assert not torch.equal(a[0][0], a[0][1])                  # one seed per layer


def _malformed(how):
    m, b = _synthetic(D=50, seed=8)
    (hb, hf, he, hv), (tb, te, tf, tv) = (tuple(np.array(a) for a in lst) for lst in b[3])
    i = int(np.nonzero(hb == hb[0])[0][1])
    if how == "slot listed twice":
        hf[i] = hf[0]
    else:
        he[0] = b[0].shape[1] + 5
    bad = list(b)
    bad[3] = ((hb, hf, he, hv), (tb, te, tf, tv))
    return m, batching.pin_graft_batch(b), batching.pin_graft_batch(tuple(bad))


@pytest.mark.parametrize("how,msg", [("slot listed twice", "a fact slot listed twice"),
                                     ("id outside the batch", "a batch, fact-slot or node id outside the batch")])
def test_malformed_graft_lists_are_reported_by_check(how, msg):
    m, good, bad = _malformed(how)
    step = graphed.GraphedGraftTrainStep(m)
    step.step(good).check()
    assert step.key(bad) == step.key(good)
    out = _step_without_sync(step, bad)
    with pytest.raises(RuntimeError, match="graft fact lists rejected: .*" + msg):
        out.check()
    step.step(good).check()


def test_refusals():
    with pytest.raises(ValueError, match="covers ReaRev and NSM; GraftNet"):
        graphed.GraphedTrainStep(_synthetic(D=32)[0])
    cpu = G.GraftNet(dict(S.model_args("GraftNet", entity_dim=32, use_cuda=False)), NE, NR, NW)
    with pytest.raises(ValueError, match="needs a model on a CUDA device"):
        graphed.GraphedGraftTrainStep(cpu)
    m, batch = _synthetic(D=513, B=2, N=50, E=100)
    step = graphed.GraphedGraftTrainStep(m)
    with pytest.raises(ValueError, match="_fact_kernels is false: entity_dim 513"):
        step.step(batch)
    m, batch = _synthetic(D=32, B=2, N=50, E=100)
    step = graphed.GraphedGraftTrainStep(m)
    old = autograd_path.USE_KERNELS
    autograd_path.USE_KERNELS = False
    try:
        with pytest.raises(ValueError, match="USE_KERNELS is off"):
            step.step(batch)
    finally:
        autograd_path.USE_KERNELS = old
    kb = S.make_batch(1, B=2, N=50, E=100, num_entity=NE, num_relation=NR, num_word=NW)[:7]
    with pytest.raises(ValueError, match="9/10-tuple"):
        step.step(kb)
    assert not step._cache
