"""graphed.GraphedTrainStep: ``model(batch, training=True)`` + ``loss.backward()`` + the train-time metrics captured as
one CUDA graph per batch shape (ReaRev, NSM), and gr_train_metrics (csrc/rank.cu) against autograd_path.eval_metric.

Under torch.use_deterministic_algorithms the graphed step is bit-equal to the eager step: loss, pred_dist, pred, h1,
f1 and every parameter gradient, also under bf16 autocast and over a three-step Adam loop in which the caller clips
and steps the optimizer between replays.  Without the flag the gradients agree within the atomics' rounding."""
import copy
import gc
import weakref
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import autograd_path, batching, graphed, ops, synthetic as S
from golden_io import Golden

import test_graphed_train_host as HT
import test_training_path as TP

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")

NE, NR, NW = 3000, 40, 100


@pytest.fixture(autouse=True)
def _fp32_cudnn():
    """cuDNN's LSTM in fp32 (no TF32), as in the training tests; torch's deterministic flag restored afterwards."""
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        yield
    torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])


def _det(on):
    torch.use_deterministic_algorithms(on, warn_only=True)


def _no_dropout(m):
    m.train()                                     # cuDNN's LSTM backward needs training mode ...
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.eval()                            # ... the dropouts stay the identity
    return m


def _golden(name):
    m, batch, _t = TP._load(name, device="cuda")
    m = _no_dropout(m.cuda())
    if getattr(m, "rel_texts", None) is not None:
        g = Golden(name)
        m.encode_rel_texts(g.rel_texts, g.rel_texts_inv)
    return m, batch


def _synthetic(model_name="ReaRev", D=50, B=4, N=200, E=700, seed=3, dropout=0.0, **over):
    args = S.model_args(model_name, entity_dim=D, use_cuda=True, linear_dropout=dropout, lm_dropout=dropout, **over)
    torch.manual_seed(seed)
    cls = G.ReaRev if model_name == "ReaRev" else G.NSM
    m = cls(dict(args), NE, NR, NW).cuda().train()
    w = bool(over.get("normalized_gnn") or over.get("norm_rel"))
    return m, S.make_batch(seed, B=B, N=N, E=E, num_entity=NE, num_relation=NR, num_word=NW, with_weights=w)[:7]


def _case(name):
    if name == "rearev_d50_lstm":
        return _synthetic(D=50, num_ins=3, num_iter=2, num_gnn=3)
    if name == "rearev_d200":
        return _synthetic(D=200, num_ins=2, num_iter=2, num_gnn=2, B=3, N=300, E=1200)
    return _golden(name)


CASES = ["rearev_d50_lstm", "rearev_d200", "rearev_posemb", "rearev_norm", "nsm_small", "nsm_reason_kb"]


def _eager(m, batch, autocast=None):
    """Loss, pred, pred_dist, tp_list and gradients of the eager step (the forward under ``autocast``, the backward
    outside it); the model's first step runs once more before (cuBLAS may choose another GEMM algorithm on a
    process's first calls)."""
    if not getattr(m, "_eager_warm", False):
        _eager_once(m, batch, autocast)
        m._eager_warm = True
    return _eager_once(m, batch, autocast)


def _eager_once(m, batch, autocast):
    for p in m.parameters():
        p.grad = None
    with torch.autocast("cuda", dtype=autocast, enabled=autocast is not None):
        loss, pred, pred_dist, tp = m(batch, training=True)
    loss.backward()
    grads = {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}
    return loss.detach().clone(), pred.clone(), pred_dist.detach().clone(), tp, grads


def _graphed(step, batch):
    loss, pred, pred_dist, h1, f1 = out = step.step(batch)
    out.check()
    grads = {k: p.grad.clone() for k, p in step.model.named_parameters() if p.grad is not None}
    return loss.clone(), pred.clone(), pred_dist.clone(), step.tp_list(h1, f1), grads


def _assert_bit_equal(a, b):
    for x, y, what in zip(a[:3], b[:3], ("loss", "pred", "pred_dist")):
        assert torch.equal(x, y), what
    assert a[3] == b[3]                          # [h1 list, f1 list]
    assert set(a[4]) == set(b[4])
    for k in a[4]:
        assert torch.equal(a[4][k], b[4][k]), k


@pytest.mark.parametrize("name", CASES)
def test_bit_equal_to_eager_under_the_deterministic_flag(name):
    m, batch = _case(name)
    _det(True)
    want = _eager(m, batch)
    step = graphed.GraphedTrainStep(m)
    _assert_bit_equal(want, _graphed(step, batch))
    _assert_bit_equal(want, _graphed(step, batch))           # the replay of the captured key


@pytest.mark.parametrize("name", CASES)
def test_close_to_eager_without_the_deterministic_flag(name):
    """fp32 atomics in the backward kernels: loss and pred_dist within 1e-5 relative, every gradient within 1e-4 of
    its own scale plus 1e-6 of the largest gradient (observed: printed)."""
    m, batch = _case(name)
    _det(False)
    want = _eager(m, batch)
    got = _graphed(graphed.GraphedTrainStep(m), batch)
    assert abs(float(got[0]) - float(want[0])) <= 1e-5 * abs(float(want[0]))
    assert (got[2] - want[2]).abs().max().item() <= 1e-5 * want[2].abs().max().item() + 1e-9
    gmax = max(g.abs().max().item() for g in want[4].values())
    assert set(got[4]) == set(want[4])
    worst = 0.0
    for k, w in want[4].items():
        err = (got[4][k] - w).abs().max().item()
        scale = w.abs().max().item()
        if scale > 1e-3 * gmax:                  # tensors whose gradient is ~0 hold rounding noise only
            worst = max(worst, err / scale)
        assert err <= 1e-4 * scale + 1e-6 * gmax + 1e-9, (k, err, scale)
    print("%s: largest gradient error relative to the tensor's scale %.2e" % (name, worst))


@pytest.mark.parametrize("name", ["rearev_d50_lstm", "rearev_d200", "nsm_reason_kb"])
def test_bf16_autocast_bit_equal_to_eager(name):
    m, batch = _case(name)
    _det(True)
    want = _eager(m, batch, torch.bfloat16)
    step = graphed.GraphedTrainStep(m)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        got = _graphed(step, batch)
    _assert_bit_equal(want, got)
    assert len(step._cache) == 1
    _graphed(step, batch)                                    # outside autocast: another key, another graph
    assert len(step._cache) == 2


def _adam_loop(m, run, batches):
    opt = torch.optim.Adam([p for p in m.parameters() if p.requires_grad], lr=5e-3)
    losses = []
    for b in batches:
        opt.zero_grad(set_to_none=True)
        losses.append(run(b))
        torch.nn.utils.clip_grad_norm_([p for p in m.parameters() if p.requires_grad], 1.0)
        opt.step()
    return losses, {k: v.clone() for k, v in m.state_dict().items()}


@pytest.mark.parametrize("name", ["rearev_d50_lstm", "nsm_reason_kb"])
def test_three_step_adam_loop_bit_equal(name):
    """Replays read the weights the caller's clip + Adam step wrote in place."""
    m, batch = _case(name)
    m2 = copy.deepcopy(m)
    _det(True)

    def eager(b):
        loss = m(b, training=True)[0]
        loss.backward()
        return loss.detach().clone()
    step = graphed.GraphedTrainStep(m2)
    want = _adam_loop(m, eager, [batch] * 3)
    got = _adam_loop(m2, lambda b: step.step(b)[0].clone(), [batch] * 3)
    assert len(step._cache) == 1
    assert [float(x) for x in want[0]] == [float(x) for x in got[0]]
    assert float(want[0][2]) != float(want[0][0])           # the weights moved
    for k in want[1]:
        assert torch.equal(want[1][k], got[1][k]), k


def test_buckets_replay_and_lru_eviction():
    m, _ = _synthetic(D=50, num_ins=2, num_iter=2, num_gnn=2)
    mk = lambda seed, E: S.make_batch(seed, B=4, N=200, E=E, num_entity=NE, num_relation=NR,   # noqa: E731
                                      num_word=NW, with_weights=False)[:7]
    same = [mk(11, 700), mk(12, 720), mk(13, 690)]
    Fs = [len(b[2][0]) for b in same]
    assert len(set(Fs)) == 3 and len({graphed.fact_capacity(F) for F in Fs}) == 1
    _det(True)
    step = graphed.GraphedTrainStep(m, max_graphs=2)
    for b in same:
        want = _eager(m, b)
        _assert_bit_equal(want, _graphed(step, b))
    assert len(step._cache) == 1
    first = weakref.ref(next(iter(step._cache.values())))
    big = mk(14, 1400)
    assert graphed.fact_capacity(len(big[2][0])) != graphed.fact_capacity(Fs[0])
    _assert_bit_equal(_eager(m, big), _graphed(step, big))
    assert len(step._cache) == 2
    bigger = mk(15, 2600)
    _assert_bit_equal(_eager(m, bigger), _graphed(step, bigger))
    assert len(step._cache) == 2
    gc.collect()
    assert first() is None                                  # the least recently used graph was released


def test_replay_does_not_synchronise_with_the_host():
    m, batch = _synthetic(D=50, num_ins=3, num_iter=2, num_gnn=3)
    pinned = batching.pin_batch(batch)
    step = graphed.GraphedTrainStep(m)
    step.step(pinned)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = step.step(pinned)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    out.check()
    assert torch.isfinite(out[0]).item()


def test_dropout_masks_are_fresh_on_every_replay():
    m, batch = _synthetic(D=50, num_ins=2, num_iter=2, num_gnn=2, dropout=0.3)
    step = graphed.GraphedTrainStep(m)
    a = float(step.step(batch)[0])
    b = float(step.step(batch)[0])
    assert a != b
    m0, batch0 = _synthetic(D=50, num_ins=2, num_iter=2, num_gnn=2, dropout=0.0)
    _det(True)
    step0 = graphed.GraphedTrainStep(m0)
    assert float(step0.step(batch0)[0]) == float(step0.step(batch0)[0])


# ---- gr_train_metrics against eval_metric -----------------------------------------------------------------------------

def _metrics_both(pred_dist, answer_dist, seed_dist, local_entity, pad=NE, eps=0.95):
    t = lambda a, dt=torch.float32: torch.as_tensor(np.asarray(a)).to(dev, dt)   # noqa: E731
    pd, ad, sd, le = t(pred_dist), t(answer_dist), t(seed_dist), t(local_entity, torch.int64)
    want = autograd_path.eval_metric(SimpleNamespace(num_entity=pad, eps=eps), pd, ad, sd, le)
    ci, cc, _ = ops.rank_candidates(pd, le, (sd > 0).float(), pad, eps)
    got = ops.train_metrics(pd, ad, sd, le, ci, cc, pad)
    return want, got


def _assert_metrics(*a, **k):
    (h1w, f1w), (h1g, f1g) = _metrics_both(*a, **k)
    assert torch.equal(h1w, h1g), (h1w, h1g)
    assert torch.equal(f1w, f1g), (f1w, f1g)
    return h1g.tolist(), f1g.tolist()


@pytest.mark.parametrize("name", TP.CASES)
def test_train_metrics_on_the_goldens(name):
    g = Golden(name)
    t = np.load(TP.os.path.join(TP.GOLDEN_DIR, "train", name + ".npz"))
    b = g.batch
    h1, f1 = _assert_metrics(t["pred_dist"], t["answer_dist"], b[4], b[0], pad=g.num_entity, eps=g.args["eps"])
    assert h1 == t["h1"].tolist()


def test_train_metrics_on_cfg2_sized_batches():
    c = S.CONFIGS["cfg2"]
    rs = np.random.RandomState(0)
    for seed in (1, 2):
        b = S.make_batch(seed, B=c["B"], N=c["N"], E=c["E"], with_weights=False, multi_seed=True)
        pad = S.WEBQSP_NUM_ENTITY
        logits = rs.randn(c["B"], c["N"]).astype(np.float32) * (3.0 if seed == 1 else 0.3)
        ans = np.asarray(b[6], dtype=np.float32)
        logits[:, :] += 4.0 * (ans > 0)               # most questions hit
        pd = np.exp(logits - logits.max(1, keepdims=True))
        pd /= pd.sum(1, keepdims=True)
        _assert_metrics(pd, ans, b[4], b[0], pad=pad)


def test_train_metrics_edge_cases():
    """No answers, no candidates, every candidate correct, hit@1 = 0, a tie at the maximum, a repeated entity id
    (test_graphed_train_host.edge_batch), each also as a batch of one question."""
    pd, ad, sd, le, pad = HT.edge_batch()
    h1, f1 = _assert_metrics(pd, ad, sd, le, pad=pad)
    assert h1 == HT.EDGE_H1
    assert f1[1] == 0.0 and f1[2] == 1.0 and f1[3] == 0.0
    assert f1[6] == 1.0                                    # no answers and no candidates
    for b in range(len(h1)):                               # B = 1
        _assert_metrics(pd[b:b + 1], ad[b:b + 1], sd[b:b + 1], le[b:b + 1], pad=pad)


def test_train_metrics_more_answers_than_shared_memory_holds():
    B, N, pad = 2, 5000, 10 ** 6
    rs = np.random.RandomState(5)
    le = rs.randint(0, 3000, size=(B, N)).astype(np.int64)      # many repeated ids
    ad = (rs.rand(B, N) < 0.6).astype(np.float32)
    sd = np.zeros((B, N), np.float32)
    pd = rs.rand(B, N).astype(np.float32) + 3.0 * ad
    pd[:, :10] += 50.0 * ad[:, :10]
    pd /= pd.sum(1, keepdims=True)
    _assert_metrics(pd, ad, sd, le, pad=pad)


def test_refusals():
    args = S.model_args("GraftNet", entity_dim=32, use_cuda=True)
    with pytest.raises(ValueError, match="GraftNet"):
        graphed.GraphedTrainStep(G.GraftNet(dict(args), NE, NR, NW))
    cpu = G.ReaRev(dict(S.model_args("ReaRev", entity_dim=32, use_cuda=False)), NE, NR, NW)
    with pytest.raises(ValueError, match="CUDA"):
        graphed.GraphedTrainStep(cpu)
    m, batch = _synthetic(D=264, num_ins=2, num_iter=1, num_gnn=1, B=2, N=50, E=100)
    step = graphed.GraphedTrainStep(m)
    with pytest.raises(ValueError, match="_kernel_graph is None: entity_dim 264"):
        step.step(batch)
    assert not step._cache
