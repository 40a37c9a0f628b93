"""A whole GraftNet training epoch replayed as CUDA graphs (GraphedGraftTrainStep.train_epoch / start_epoch) on the GPU.

Under torch's deterministic flag the epoch is bit-equal to the loop it replaces -- ``split.get_batch`` +
``GraphedGraftTrainStep.step`` + ``loss.item()`` + ``tp_list`` per batch -- over two epochs, in the returned mean and
lists, the parameters, ``p.grad`` and the Adam state: with the fact orders drawn in the graph (``shuffle``) or stored,
with inverse relations and ``norm_rel``, under bf16 autocast, with fact dropout replayed from the recorded seeds and
with a batch that has no graft entries.  Model dropout reproduces under one ``torch.manual_seed`` whether the graphs are
captured during the call or cached.  A warm epoch does not synchronise with the host, and malformed orders reach
``EpochRun.check``.  gr_epoch_graft_begin is held to an exact restatement, and the graft assembly into capacity
buffers (``out=``) to ``get_batch``'s lists."""
import contextlib
import copy
import math

import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import graphed, loader, ops, synthetic as S

from test_clip_adam_gpu import _assert_same_training, _trainable
from test_device_split_host import NE, NW, GraftSplitLoader
from test_train_epoch_gpu import _begin_ref, _loop_epoch, _restore, _same_result, _snapshot

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


def _graft_counts(L):
    return np.array([len(L.create_kb_adj_mats_facts(q)[0][0][2]) for q in range(L.num_data)], dtype=np.int64)


def _plan(L, p=0.0):
    stored = [len(m[0]) for m in L.kb_adj_mats]
    ents = [len(g) for g in L.global2local_entity_maps]
    return graphed.epoch_plan(L.batches, stored, ents, B, p, _graft_counts(L))


def _loader(**kw):
    """23 questions of 20..1200 facts: batches of 4 spread over several (fact, graft) capacity pairs, the last one
    short."""
    L = GraftSplitLoader(seed=5, num_questions=23, max_local_entity=60, facts_lo=20, facts_hi=1200, **kw)
    plan = _plan(L)
    assert L.num_data % B != 0 and len(set(zip(plan.capacity.tolist(), plan.graft_capacity.tolist()))) >= 3
    return L


def _model(L, dropout=0.0, **over):
    torch.manual_seed(0)
    args = S.model_args("GraftNet", entity_dim=50, use_cuda=True, word_dim=64, linear_dropout=dropout,
                        lm_dropout=dropout, **over)
    args.update(num_layer=2)
    return G.GraftNet(dict(args), NE, L.num_kb_relation, NW).cuda()


def _step(m, max_norm=1.0):
    opt = torch.optim.Adam(_trainable(m), lr=5e-3)
    return graphed.GraphedGraftTrainStep(m, optimizer=opt, max_norm=max_norm), opt


def _two_epochs_bit_equal(L, split, over=None, autocast=None):
    m_loop = _model(L, **(over or {}))
    m_ep = copy.deepcopy(m_loop)
    step_loop, opt_loop = _step(m_loop)
    step_ep, opt_ep = _step(m_ep)
    ac = (lambda: torch.autocast("cuda", dtype=autocast)) if autocast is not None else contextlib.nullcontext
    for epoch in range(2):
        np.random.seed(10 + epoch)
        torch.manual_seed(20 + epoch)
        with ac():
            want = _loop_epoch(step_loop, split, 0.0)
        ids_loop = list(L.sample_ids)
        np.random.seed(10 + epoch)
        torch.manual_seed(20 + epoch)
        with ac():
            got = step_ep.train_epoch(split, B, 0.0)
        assert list(L.sample_ids) == ids_loop
        _same_result(got, want)
        _assert_same_training(m_loop, m_ep, opt_loop, opt_ep)
    assert opt_ep.state[_trainable(m_ep)[0]]["step"].item() == 2 * math.ceil(L.num_data / B)
    return step_ep


@pytest.mark.parametrize("case", ["stored", "shuffle", "inverse_norm_rel", "bf16"])
def test_epoch_bit_equal_to_the_loop(case):
    inverse = case == "inverse_norm_rel"
    L = _loader(use_inverse_relation=inverse)
    split = loader.DeviceSplit(L, dev, shuffle=case != "stored")
    step = _two_epochs_bit_equal(L, split, over=dict(use_inverse_relation=True, norm_rel=True) if inverse else None,
                                 autocast=torch.bfloat16 if case == "bf16" else None)
    plan = _plan(L)                                           # of the last epoch's order
    shapes = set(zip(plan.B.tolist(), plan.capacity.tolist(), plan.graft_capacity.tolist()))
    assert {(k[0], k[2], k[5]) for k in step._cache if k[-2] == "epoch"} >= shapes     # one graph per shape


def test_fact_dropout_replays_from_the_recorded_seeds():
    L = _loader()
    m_loop = _model(L)
    m_ep = copy.deepcopy(m_loop)
    split = loader.DeviceSplit(L, dev, shuffle=True)
    step_loop, opt_loop = _step(m_loop)
    step_ep, opt_ep = _step(m_ep)
    for epoch in range(2):
        np.random.seed(30 + epoch)
        run = step_ep.start_epoch(split, B, 0.3)
        got = run.result()
        run.check()
        assert run.seeds.shape == (math.ceil(L.num_data / B),) and run.status.shape == (3,)
        np.random.seed(30 + epoch)
        want = _loop_epoch(step_loop, split, 0.3, seeds=run.seeds)
        _same_result(got, want)
        _assert_same_training(m_loop, m_ep, opt_loop, opt_ep)


def test_batch_without_graft_entries_trains_and_matches_the_loop():
    """The first batch's questions have no stored facts, so no graft entries (G = 0, graft_live = 0)."""
    L = _loader()
    empty = [0, 1, 2, 3]
    for q in empty:
        L.kb_adj_mats[q] = tuple(np.zeros(0, dtype=int) for _ in range(3))
        L.kb_fact_rels[q] = L.create_kb_adj_mats_facts(q)[1]

    def order_with_empty_batch_first(is_sequential=True):
        rest = np.random.permutation(np.arange(4, L.num_data))
        L.batches = np.concatenate([np.random.permutation(empty), rest])
    L.reset_batches = order_with_empty_batch_first
    L.reset_batches()
    assert _plan(L).G[0] == 0
    split = loader.DeviceSplit(L, dev, shuffle=True)
    _two_epochs_bit_equal(L, split)


def test_model_dropout_reproduces_captured_or_cached():
    L = _loader()
    m = _model(L, dropout=0.2)
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
    m = _model(L)
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
    m = _model(L)
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
    from test_device_split_host import SplitLoader
    L = _loader()
    m = _model(L, norm_rel=True)
    split = loader.DeviceSplit(L, dev, shuffle=True)
    step, _opt = _step(m)
    before = L.batches.copy()
    kb = loader.DeviceSplit(SplitLoader(seed=5, num_questions=9, max_local_entity=20), dev, shuffle=True)
    cases = [
        (graphed.GraphedGraftTrainStep(m), split, B, 0.0, "optimizer="),
        (step, L, B, 0.0, "takes a loader.DeviceSplit"),
        (step, kb, B, 0.0, "takes a GraftNet split.*covers ReaRev and NSM"),
        (step, split, 0, 0.0, "batch_size must be a positive int"),
        (step, split, B, 1.5, r"fact_dropout must be in \[0, 1\]"),
        (step, loader.DeviceSplit(L, dev), B, 0.1, "fact_dropout must be 0"),
        (step, loader.DeviceSplit(L, dev, weights="none", shuffle=True), B, 0.0, "weights='none'"),
    ]
    rm = G.ReaRev(dict(S.model_args("ReaRev", entity_dim=50, use_cuda=True, word_dim=64)), NE, L.num_kb_relation,
                  NW).cuda()
    rstep = graphed.GraphedTrainStep(rm, optimizer=torch.optim.Adam(_trainable(rm)), max_norm=1.0)
    cases.append((rstep, split, B, 0.0, "train_epoch takes a ReaRev / NSM split; this DeviceSplit holds GraftNet's"))
    for gts, sp, bs, p, msg in cases:
        with pytest.raises(ValueError, match=msg):
            gts.train_epoch(sp, bs, p)
        with pytest.raises(ValueError, match=msg):
            gts.start_epoch(sp, bs, p)
    assert np.array_equal(L.batches, before) and len(step._cache) == 0 and len(rstep._cache) == 0


# ---- the kernel and the capacity assembly against exact restatements ------------------------------------------------

def _graft_begin_ref(ids, kept_table, g_off, cap):
    num_q = len(g_off) - 1
    kept = []
    for i in ids:
        ok = 0 <= i < num_q
        n = int(g_off[i + 1] - g_off[i]) if ok else 0
        kept.append(min(max(int(kept_table[i]), 0), n) if (kept_table is not None and ok) else n)
    total = sum(kept)
    return kept, min(total, cap), 2 if total > cap else 0


@pytest.mark.parametrize("with_kept", [True, False])
def test_graft_begin_against_a_restatement(with_kept):
    rs = np.random.RandomState(11)
    num_q, bs = 40, 6
    counts = rs.randint(1, 300, num_q)
    counts[[3, 17]] = 0                                       # empty questions
    g_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    q_off = np.concatenate([[0], np.cumsum(rs.randint(0, 200, num_q))]).astype(np.int64)
    q_ents = rs.randint(0, 50, num_q).astype(np.int32)
    order = rs.permutation(num_q)[:33].astype(np.int64)       # 33 = 5 full steps and a short one of 3
    order[1], order[7] = 3, 17
    order[8], order[20] = num_q + 3, -2                       # out of range: empty questions
    kept_table = rs.randint(-5, 320, num_q).astype(np.int64) if with_kept else None
    if with_kept:
        kept_table[order[0]] = -7                             # below 0 and above the stored count
        kept_table[order[2]] = counts[order[2]] + 50
    d = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev)   # noqa: E731
    tested_cap = 0
    for c, Bc in [(0, 6), (1, 6), (3, 6), (5, 3), (7, 6), (-1, 2)]:
        ids = torch.full((Bc,), -9, dtype=torch.int64, device=dev)
        rows, kept = (torch.empty(Bc, dtype=torch.int64, device=dev) for _ in range(2))
        scratch = (torch.empty(1, dtype=torch.int32, device=dev), torch.empty(1, dtype=torch.int64, device=dev),
                   torch.empty(1, dtype=torch.int32, device=dev))
        ops.epoch_step_begin(torch.tensor([c], device=dev), d(order), bs, None, d(q_off), d(q_ents), True, 4096, ids,
                             rows, kept, *scratch)
        want_ids = _begin_ref(c, order, bs, Bc, None, q_off, q_ents, True, 4096)[0]
        assert ids.tolist() == want_ids, c
        kept_ref, _live, _st = _graft_begin_ref(want_ids, kept_table, g_off, 4096)
        total = sum(kept_ref)
        for cap in sorted({4096, total, max(total - 1, 0)}):
            kept_g = torch.full((Bc,), -9, dtype=torch.int64, device=dev)
            live = torch.full((2,), -9, dtype=torch.int32, device=dev)
            st = torch.full((1,), 8, dtype=torch.int32, device=dev)
            ops.epoch_graft_begin(ids, d(kept_table), d(g_off), cap, kept_g, live, st)
            k, lv, status = _graft_begin_ref(want_ids, kept_table, g_off, cap)
            assert kept_g.tolist() == k and live.tolist() == [lv, lv] and int(st.item()) == status, (c, cap)
            tested_cap += cap == total or cap == total - 1
    assert tested_cap >= 8                                    # G equal to the capacity and one past it


@pytest.mark.parametrize("shuffle", [False, True])
@pytest.mark.parametrize("idt", [torch.int32, torch.int64])
def test_graft_assembly_into_capacity_buffers(idt, shuffle):
    """``DeviceSplit.assemble_graft(..., out=)`` into int64 capacity buffers: the live prefix is ``get_batch``'s lists
    (cast to int64), the slots past it keep their sentinel, ``kb_fact_rel`` is ``get_batch``'s."""
    L = GraftSplitLoader(seed=7, num_questions=11, max_local_entity=40, facts_lo=10, facts_hi=400)
    split = loader.DeviceSplit(L, dev, index_dtype=idt, shuffle=shuffle)
    p = 0.3 if shuffle else 0.0
    for it in range(3):
        seed = torch.tensor([1234 + it], dtype=torch.int64, device=dev)
        b = split.get_batch(it, B, p, seed=seed) if shuffle else split.get_batch(it, B, p)
        ids = np.asarray(L.sample_ids, dtype=np.int64)
        n = split._graft_count[ids]
        kept_g = loader.kept_counts(n, p)
        Gn = int(kept_g.sum())
        cap = graphed.fact_capacity(Gn)
        idx = [torch.full((cap,), -77, dtype=torch.int64, device=dev) for _ in range(6)]
        vals = [torch.full((cap,), -5.0, device=dev) for _ in range(2)]
        kfr = torch.full((len(ids), split.max_facts), -3, dtype=torch.int64, device=dev)
        out = ((*idx[:3], vals[0]), (*idx[3:], vals[1]), kfr)
        ids_dev, kept_dev = torch.from_numpy(ids).to(dev), torch.from_numpy(kept_g).to(dev)
        graft, kfr_out, order, status = split.assemble_graft(ids_dev, kept_dev, seed, cap, int(n.sum()), out=out)
        assert kfr_out is kfr and all(a is c for a, c in zip(graft[0] + graft[1], out[0] + out[1]))
        assert (order is not None) == shuffle and int(status.item()) == 0
        (hb, hf, he, hv), (tb, te, tf, tv) = b[3]
        for got, want in zip(idx, (hb, hf, he, tb, te, tf)):
            assert want.dtype == idt and want.numel() == Gn
            assert torch.equal(got[:Gn], want.long()) and bool((got[Gn:] == -77).all())
        for got, want in zip(vals, (hv, tv)):
            assert torch.equal(got[:Gn], want) and bool((got[Gn:] == -5.0).all())
        assert torch.equal(kfr, b[5])
        # a capacity one short of the batch: flagged with bit 2 (stored order: cut there)
        if Gn:
            short = [torch.full((Gn - 1,), -77, dtype=torch.int64, device=dev) for _ in range(6)]
            sv = [torch.full((Gn - 1,), -5.0, device=dev) for _ in range(2)]
            o2 = ((*short[:3], sv[0]), (*short[3:], sv[1]), torch.empty_like(kfr))
            *_x, st2 = split.assemble_graft(ids_dev, kept_dev, seed, Gn - 1, int(n.sum()), out=o2)
            assert int(st2.item()) & 2
            if not shuffle:
                assert all(torch.equal(a, c[:Gn - 1]) for a, c in zip(short, idx))
