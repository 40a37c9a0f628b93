"""A whole training epoch replayed as CUDA graphs (GraphedTrainStep.train_epoch / start_epoch) on the GPU.

Under torch's deterministic flag the epoch is bit-equal to the loop it replaces -- ``split.get_batch`` +
``GraphedTrainStep.step`` + ``loss.item()`` + ``tp_list`` per batch -- for ReaRev and NSM over two epochs, in the
returned mean and lists, the parameters, ``p.grad`` and the Adam state, with the fact order drawn in the graph
(``shuffle``) or stored, with fact weights, and with fact dropout replayed from the recorded seeds.  Model dropout
reproduces under one ``torch.manual_seed`` whether the graphs are captured during the call or cached.  A warm epoch
does not synchronise with the host, and malformed orders reach ``EpochRun.check``.  The two new kernels are held to
exact restatements: the live-prefix fact weights and the step bookkeeping."""
import copy
import math

import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import graphed, loader, ops, synthetic as S

from test_clip_adam_gpu import _assert_same_training, _trainable
from test_device_split_host import NE, NW, SplitLoader
from test_graphed_graft_train_gpu import _synthetic as _graft_synthetic

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
B = 4


@pytest.fixture(autouse=True)
def _deterministic():
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    torch.use_deterministic_algorithms(True, warn_only=True)
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        yield
    torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])


def _loader(**kw):
    """23 questions of 20..1200 facts: batches of 4 spread over several fact-capacity buckets, the last one short."""
    L = SplitLoader(seed=5, num_questions=23, max_local_entity=60, facts_lo=20, facts_hi=1200, **kw)
    plan = graphed.epoch_plan(L.batches, [len(m[0]) for m in L.kb_adj_mats],
                              [len(g) for g in L.global2local_entity_maps], B)
    assert L.num_data % B != 0 and len(set(plan.capacity.tolist())) >= 3
    return L


def _model(name, L, dropout=0.0, **over):
    torch.manual_seed(0)
    args = S.model_args(name, entity_dim=50, use_cuda=True, word_dim=64, linear_dropout=dropout, lm_dropout=dropout,
                        **over)
    if name == "ReaRev":
        args.update(num_ins=2, num_iter=2, num_gnn=2)
    else:
        args.update(num_step=2)
    return {"ReaRev": G.ReaRev, "NSM": G.NSM}[name](dict(args), NE, L.num_kb_relation, NW).cuda()


def _step(m, max_norm=1.0):
    opt = torch.optim.Adam(_trainable(m), lr=5e-3)
    return graphed.GraphedTrainStep(m, optimizer=opt, max_norm=max_norm), opt


def _loop_epoch(gts, split, p, seeds=None):
    """The loop ``train_epoch`` runs today around the graphed step."""
    gts.model.train()
    split.reset_batches(is_sequential=False)
    losses, h1_all, f1_all = [], [], []
    for it in range(math.ceil(split.num_data / B)):
        kw = {} if seeds is None else dict(seed=seeds[it:it + 1])
        out = gts.step(split.get_batch(it, B, p, **kw))
        losses.append(out[0].item())
        h1, f1 = gts.tp_list(out[3], out[4])
        h1_all.extend(h1)
        f1_all.extend(f1)
    return np.mean(losses), [0, 0], h1_all, f1_all


def _same_result(a, b):
    assert type(a[0]) is type(b[0]) and a[0] == b[0]
    assert a[1] == b[1] == [0, 0]
    assert a[2] == b[2] and a[3] == b[3]
    assert all(type(x) is float for x in a[2] + a[3])


@pytest.mark.parametrize("name,shuffle,over", [
    ("ReaRev", False, {}), ("ReaRev", True, {}), ("ReaRev", True, dict(normalized_gnn=True)),
    ("NSM", False, {}), ("NSM", True, {})])
def test_epoch_bit_equal_to_the_loop(name, shuffle, over):
    L = _loader()
    m_loop = _model(name, L, **over)
    m_ep = copy.deepcopy(m_loop)
    split = loader.DeviceSplit(L, dev, shuffle=shuffle)
    step_loop, opt_loop = _step(m_loop)
    step_ep, opt_ep = _step(m_ep)
    for epoch in range(2):
        np.random.seed(10 + epoch)
        torch.manual_seed(20 + epoch)
        want = _loop_epoch(step_loop, split, 0.0)
        ids_loop = list(L.sample_ids)
        np.random.seed(10 + epoch)
        torch.manual_seed(20 + epoch)
        got = step_ep.train_epoch(split, B, 0.0)
        assert list(L.sample_ids) == ids_loop
        _same_result(got, want)
        _assert_same_training(m_loop, m_ep, opt_loop, opt_ep)
    assert opt_ep.state[_trainable(m_ep)[0]]["step"].item() == 2 * math.ceil(L.num_data / B)


def test_fact_dropout_replays_from_the_recorded_seeds():
    L = _loader()
    m_loop = _model("ReaRev", L)
    m_ep = copy.deepcopy(m_loop)
    split = loader.DeviceSplit(L, dev, shuffle=True)
    step_loop, opt_loop = _step(m_loop)
    step_ep, opt_ep = _step(m_ep)
    for epoch in range(2):
        np.random.seed(30 + epoch)
        run = step_ep.start_epoch(split, B, 0.3)
        got = run.result()
        run.check()
        assert run.seeds.shape == (math.ceil(L.num_data / B),) and run.grad_norms.shape == run.seeds.shape
        np.random.seed(30 + epoch)
        want = _loop_epoch(step_loop, split, 0.3, seeds=run.seeds)
        _same_result(got, want)
        _assert_same_training(m_loop, m_ep, opt_loop, opt_ep)


def _snapshot(m, opt):
    return ([p.detach().clone() for p in m.parameters()],
            {id(p): {k: v.clone() for k, v in opt.state[p].items()} for p in _trainable(m) if p in opt.state})


def _restore(m, opt, snap):
    params, state = snap
    with torch.no_grad():
        for p, v in zip(m.parameters(), params):
            p.copy_(v)
    for p in _trainable(m):
        for k, v in state.get(id(p), {}).items():
            opt.state[p][k].copy_(v)


def test_model_dropout_reproduces_captured_or_cached():
    L = _loader()
    m = _model("ReaRev", L, dropout=0.2)
    split = loader.DeviceSplit(L, dev, shuffle=True)
    step, opt = _step(m)
    np.random.seed(1)
    step.train_epoch(split, B, 0.1)              # the optimizer state exists from here on, as in the second run
    snap = _snapshot(m, opt)
    step._cache.clear()
    runs = []
    for captured in (True, False):
        _restore(m, opt, snap)
        graphs = len(step._cache)
        np.random.seed(2)
        torch.manual_seed(3)
        res = step.train_epoch(split, B, 0.1)
        assert (len(step._cache) > graphs) == captured
        runs.append((res, [p.detach().clone() for p in m.parameters()],
                     [p.grad.clone() for p in _trainable(m) if p.grad is not None]))
    (ra, pa, ga), (rb, pb, gb) = runs
    _same_result(ra, rb)
    assert all(torch.equal(x, y) for x, y in zip(pa, pb)) and all(torch.equal(x, y) for x, y in zip(ga, gb))
    assert any(not torch.equal(x, y) for x, y in zip(pa, snap[0]))


def test_warm_epoch_does_not_synchronise():
    L = _loader()
    m = _model("NSM", L)
    split = loader.DeviceSplit(L, dev, shuffle=True)
    step, _opt = _step(m)
    np.random.seed(4)
    step.train_epoch(split, B, 0.2)
    graphs = len(step._cache)
    torch.cuda.synchronize()
    np.random.seed(4)                            # the same order: every graph the epoch needs is cached
    torch.cuda.set_sync_debug_mode("error")
    try:
        run = step.start_epoch(split, B, 0.2)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(step._cache) == graphs
    mean, _x, h1, f1 = run.result()
    run.check()
    assert math.isfinite(mean) and len(h1) == len(f1) == L.num_data


def test_out_of_range_question_id_reaches_check():
    L = _loader()
    m = _model("ReaRev", L)
    split = loader.DeviceSplit(L, dev, shuffle=True)
    step, _opt = _step(m)

    def bad_order(is_sequential=True):
        L.batches = np.random.permutation(L.num_data)
        L.batches[5] = L.num_data + 7
    L.reset_batches = bad_order
    run = step.start_epoch(split, B, 0.0)
    run.result()
    with pytest.raises(RuntimeError, match=r"DeviceSplit: batch assembly status 1 \(1: question id out of range"):
        run.check()
    with pytest.raises(RuntimeError, match="batch assembly status 1"):
        step.train_epoch(split, B, 0.0)


def test_refusals():
    L = _loader()
    m = _model("ReaRev", L, normalized_gnn=True)
    split = loader.DeviceSplit(L, dev, shuffle=True)
    step, opt = _step(m)
    before = L.batches.copy()
    cases = [
        (graphed.GraphedTrainStep(m), split, B, 0.0, "optimizer="),
        (step, L, B, 0.0, "takes a loader.DeviceSplit"),
        (step, split, 0, 0.0, "batch_size must be a positive int"),
        (step, split, -2, 0.0, "batch_size must be a positive int"),
        (step, split, B, 1.5, r"fact_dropout must be in \[0, 1\]"),
        (step, split, B, -0.1, r"fact_dropout must be in \[0, 1\]"),
        (step, loader.DeviceSplit(L, dev), B, 0.1, "fact_dropout must be 0"),
        (step, loader.DeviceSplit(L, dev, weights="none", shuffle=True), B, 0.0, "weights='none'"),
    ]
    other = loader.DeviceSplit(L, dev, shuffle=True)
    other.device = torch.device("cuda", torch.cuda.device_count())
    cases.append((step, other, B, 0.0, "the split lives on"))
    gm = _graft_synthetic(D=50)[0]
    gstep = graphed.GraphedGraftTrainStep(gm, optimizer=torch.optim.Adam(_trainable(gm)), max_norm=1.0)
    cases.append((gstep, split, B, 0.0, "covers ReaRev and NSM"))
    for gts, sp, bs, p, msg in cases:
        with pytest.raises(ValueError, match=msg):
            gts.train_epoch(sp, bs, p)
        with pytest.raises(ValueError, match=msg):
            gts.start_epoch(sp, bs, p)
    assert np.array_equal(L.batches, before) and len(step._cache) == 0


# ---- the kernels against exact restatements ---------------------------------------------------------------------------

def _weights_ref(h, r):
    """fp32 of the host's float64 1/outdeg(head) and 1/count(head, rel) over the live facts (h, r)."""
    if h.size == 0:
        return np.zeros(0, np.float32), np.zeros(0, np.float32)
    w = 1.0 / np.bincount(h)[h]
    _, inv, cnt = np.unique(h * (int(r.max()) + 1) + r, return_inverse=True, return_counts=True)
    return w.astype(np.float32), (1.0 / cnt[inv.reshape(-1)]).astype(np.float32)


@pytest.mark.parametrize("idt", [torch.int32, torch.int64])
@pytest.mark.parametrize("case", ["zero", "full", "stale_in_range", "stale_out_of_range", "hub", "negative", "past"])
def test_live_prefix_weights_against_a_restatement(case, idt):
    rs = np.random.RandomState(sum(map(ord, case)))
    cap, Nt = 3072, 500
    h = rs.randint(0, Nt, cap)
    r = rs.randint(0, 9, cap)
    live = {"zero": 0, "full": cap, "stale_in_range": 1500, "stale_out_of_range": 1000, "hub": 2999,
            "negative": -5, "past": cap + 100}[case]
    F = min(max(live, 0), cap)
    if case == "stale_out_of_range":                     # padding a count would flag: ids past Nt, negative relations
        h[F:] = Nt + rs.randint(0, 1000, cap - F)
        r[F::2] = -1
    if case == "hub":
        h[:2500] = 7
        r[:2500] = rs.randint(0, 2, 2500)
    heads, rels = (torch.from_numpy(a).to(dev, idt) for a in (h, r))
    w = torch.full((cap,), 123.0, device=dev)
    wr = torch.full((cap,), 456.0, device=dev)
    nf = torch.tensor([live], dtype=torch.int32, device=dev)
    st = ops.fact_weights_live(heads, rels, nf, Nt, w, wr)
    rw, rwr = _weights_ref(h[:F], r[:F])
    wh, wrh = w.cpu().numpy(), wr.cpu().numpy()
    np.testing.assert_array_equal(wh[:F].view(np.uint32), rw.view(np.uint32))
    np.testing.assert_array_equal(wrh[:F].view(np.uint32), rwr.view(np.uint32))
    assert (wh[F:] == 123.0).all() and (wrh[F:] == 456.0).all()
    assert int(st.item()) == 0
    if F:
        dw, dwr, _ = ops.fact_weights(heads[:F], rels[:F], Nt)
        assert torch.equal(dw, w[:F]) and torch.equal(dwr, wr[:F])
    one = torch.full((cap,), -1.0, device=dev)
    ops.fact_weights_live(heads, rels, nf, Nt, None, one)
    assert torch.equal(one[:F], wr[:F]) and bool((one[F:] == -1.0).all())


def _begin_ref(c, order, bs, Bc, kept_table, q_off, q_ents, self_loop, cap):
    num_q = len(q_ents)
    ids, rows, kept = [], [], []
    bad = 0
    for j in range(Bc):
        p = c * bs + j
        i = int(order[p]) if 0 <= c and p < len(order) else -1
        ok = 0 <= i < num_q
        n = int(q_off[i + 1] - q_off[i]) if ok else 0
        k = min(max(int(kept_table[i]), 0), n) if (kept_table is not None and ok) else n
        ids.append(i)
        rows.append(i if ok else 0)
        kept.append(k)
        bad |= not ok
    tot = sum(kept) + sum(int(q_ents[i]) for i in ids if 0 <= i < num_q and self_loop)
    return ids, rows, kept, min(tot, cap), sum(kept), int(bad) | (2 if tot > cap else 0)


@pytest.mark.parametrize("self_loop", [True, False])
@pytest.mark.parametrize("with_kept", [True, False])
def test_step_begin_against_a_restatement(with_kept, self_loop):
    rs = np.random.RandomState(7)
    num_q, bs = 40, 6
    counts = rs.randint(0, 300, num_q)
    counts[3] = 0
    q_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    q_ents = rs.randint(0, 50, num_q).astype(np.int32)
    order = rs.permutation(num_q)[:33].astype(np.int64)       # 33 = 5 full steps and a short one of 3
    order[8], order[20] = num_q + 3, -2                       # out of range: empty questions, status bit 1
    kept_table = rs.randint(-5, 320, num_q).astype(np.int64) if with_kept else None
    d = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
    for c, Bc, cap in [(0, 6, 4096), (1, 6, 4096), (3, 6, 4096), (5, 3, 4096), (2, 6, 50), (7, 6, 4096),
                       (-1, 2, 4096)]:
        outs = [torch.full((Bc,), -9, dtype=torch.int64, device=dev) for _ in range(3)]
        nf = torch.full((1,), -9, dtype=torch.int32, device=dev)
        kt = torch.full((1,), -9, dtype=torch.int64, device=dev)
        st = torch.full((1,), 8, dtype=torch.int32, device=dev)
        ops.epoch_step_begin(torch.tensor([c], device=dev), d(order), bs, d(kept_table), d(q_off), d(q_ents),
                             self_loop, cap, *outs, nf, kt, st)
        ids, rows, kept, nfacts, ktot, status = _begin_ref(c, order, bs, Bc, kept_table, q_off, q_ents, self_loop, cap)
        assert outs[0].tolist() == ids and outs[1].tolist() == rows and outs[2].tolist() == kept, c
        assert (int(nf.item()), int(kt.item()), int(st.item())) == (nfacts, ktot, status), c
        if c == 2 and self_loop:
            assert status & 2


def test_step_record_against_a_restatement():
    rs = np.random.RandomState(3)
    num_data, bs = 23, 4
    steps = -(-num_data // bs)
    cursor = torch.zeros(1, dtype=torch.int64, device=dev)
    losses, norms = torch.full((steps,), -1.0, device=dev), torch.full((steps,), -1.0, device=dev)
    seeds = torch.full((steps,), -1, dtype=torch.int64, device=dev)
    h1_all, f1_all = torch.full((num_data,), -1.0, device=dev), torch.full((num_data,), -1.0, device=dev)
    epoch_status = torch.zeros(2, dtype=torch.int32, device=dev)
    want = dict(loss=[], norm=[], seed=[], h1=[], f1=[])
    words = [0, 0]
    for s in range(steps):
        Bc = min(bs, num_data - s * bs)
        loss, norm = rs.rand(2).astype(np.float32)
        seed = int(rs.randint(0, 2 ** 62, dtype=np.int64))
        h1, f1 = rs.rand(Bc).astype(np.float32), rs.rand(Bc).astype(np.float32)
        sw, cw = [0, 0, 1, 0, 2, 0][s], [0, 4, 0, 0, 0, 1][s]
        t = lambda a, dt=torch.float32: torch.tensor(a, dtype=dt, device=dev)   # noqa: E731
        ops.epoch_step_record(cursor, bs, num_data, t(loss), t([norm]), t([seed], torch.int64), t(h1), t(f1),
                              t([sw], torch.int32), t([cw], torch.int32), losses, norms, seeds, h1_all, f1_all,
                              epoch_status)
        want["loss"].append(loss)
        want["norm"].append(norm)
        want["seed"].append(seed)
        want["h1"] += h1.tolist()
        want["f1"] += f1.tolist()
        words = [words[0] | sw, words[1] | cw]
        assert int(cursor.item()) == s + 1
    assert losses.cpu().numpy().tolist() == np.float32(want["loss"]).tolist()
    assert norms.cpu().numpy().tolist() == np.float32(want["norm"]).tolist()
    assert seeds.tolist() == want["seed"]
    assert h1_all.tolist() == want["h1"] and f1_all.tolist() == want["f1"]
    assert epoch_status.tolist() == words == [3, 5]
    # past the last step: nothing recorded, bit 2, the cursor still advances
    before = [t.clone() for t in (losses, h1_all, f1_all)]
    z = torch.zeros(1, device=dev)
    ops.epoch_step_record(cursor, bs, num_data, z, None, None, torch.zeros(bs, device=dev), torch.zeros(bs, device=dev),
                          torch.zeros(1, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev),
                          losses, None, None, h1_all, f1_all, epoch_status)
    assert all(torch.equal(a, b) for a, b in zip(before, (losses, h1_all, f1_all)))
    assert epoch_status.tolist() == [3 | 2, 5] and int(cursor.item()) == steps + 1
