"""loader.DeviceSplit(shuffle=True) on the GPU: fact dropout drawn on the device (gr_split_fact_order) and batches
gathered through the drawn orders.

The permutations are checked three ways: against a numpy restatement of their definition (Philox keys, ascending
(key, index)), against the host drop-ins fed the same permutations through np.random.permutation (arrays element for
element, fp32 weights bit-equal, every model and GraphedTrainStep bit-equal under deterministic algorithms), and for
uniformity with chi-square and binomial bounds at a fixed torch seed (deterministic, so not flaky)."""
from unittest import mock

import numpy as np
import pytest
import torch
from scipy import stats

from gnn_rag_b200 import graphed, loader, ops
from loader_fixture import CASES
from test_device_split_gpu import NE, _bits, _compare_tuples, _loader, _model, _train_mode
from test_device_split_host import GraftSplitLoader, SplitLoader

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
IDX = {torch.int32: np.int32, torch.int64: np.int64}
DROPS = [0.0, 0.1, 0.5, 0.9, 1.0]
M32 = np.uint64(0xFFFFFFFF)


@pytest.fixture(autouse=True)
def _deterministic():
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    # the models' default GEMM route (GraftNet runs on no other), whatever an earlier test left in the switch
    prev_tc, ops.TC_LINEAR = ops.TC_LINEAR, True
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        yield
    ops.TC_LINEAR = prev_tc
    torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])


# ---- restatement of the permutation ------------------------------------------------------------------------------------

def _philox_x0(seed, c0, c1, c2, c3):
    """philox4x32_10_x0 (csrc/common.cuh) over uint64 arrays holding 32-bit words."""
    k0, k1 = np.uint64(seed) & M32, np.uint64(seed) >> np.uint64(32)
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & M32 for c in (c0, c1, c2, c3))
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M32)
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & M32, (k1 + np.uint64(0xBB67AE85)) & M32
    return c0


def restated_order(seed, n, b, perm, k):
    """The first k stored indices of the permutation of a question of n facts at batch position b."""
    i = np.arange(n, dtype=np.uint64)
    z = np.zeros_like(i)
    hi = _philox_x0(seed, i, z, z + np.uint64(b), z + np.uint64(perm))
    lo = _philox_x0(seed, i, z, z + np.uint64(b), z + np.uint64(perm | 2))
    key = (hi << np.uint64(32)) | lo
    return np.lexsort((i, key))[:k]


def _seed_of_next_batch(torch_seed):
    """The seed get_batch draws first after torch.manual_seed(torch_seed)."""
    torch.manual_seed(torch_seed)
    return int(torch.randint(0, 2 ** 62, (1,), device=dev).item())


def _runs(order, offsets):
    o = order.cpu().numpy()
    return [o[offsets[b]:offsets[b + 1]] for b in range(len(offsets) - 1)]


def _perms(order, offsets, counts):
    """What np.random.permutation returns per question to reproduce the device's draw: the kept indices in order,
    then the dropped ones."""
    return [np.concatenate([r, np.setdiff1d(np.arange(n), r)]).astype(np.int64)
            for r, n in zip(_runs(order, offsets), counts)]


def _host_tuple(L, split, ids, p, index_dtype):
    """The host loader's tuple for the questions ``ids`` under the permutations of the split's last batch."""
    o = split.last_order
    with mock.patch.object(np.random, "permutation",
                           side_effect=_perms(o["kb"], o["kb_offsets"], split._stored[ids])):
        kb = loader.build_fact_mat(L, list(ids), p, weights="arrays", index_dtype=IDX[index_dtype], shuffle=True)
    head = (L.candidate_entities[ids], L.query_entities[ids], kb)
    tail = (L.seed_distribution[ids], None, L.answer_dists[ids])
    if not split.graft:
        return head + (L.query_texts[ids],) + tail
    with mock.patch.object(np.random, "permutation",
                           side_effect=_perms(o["graft"], o["graft_offsets"], split._graft_count[ids])):
        graft, kfr = loader.build_fact_mat_maxfacts(L, list(ids), p)
    return head + (graft, L.query_texts[ids], kfr) + tail


def _check_structure(split, ids, p, torch_seed):
    """Per question: exactly kept_counts(n, p) distinct stored indices, equal to the restated permutation's prefix."""
    o, seed = split.last_order, _seed_of_next_batch(torch_seed)
    lists = [("kb", 0, split._stored)] + ([("graft", 1, split._graft_count)] if split.graft else [])
    for name, perm, counts in lists:
        for b, (run, n) in enumerate(zip(_runs(o[name], o[name + "_offsets"]), counts[ids])):
            k = int(loader.kept_counts([n], p)[0])
            assert len(run) == k and len(np.unique(run)) == k, (name, b)
            assert k == 0 or (run.min() >= 0 and run.max() < n), (name, b)
            np.testing.assert_array_equal(run, restated_order(seed, n, b, perm, k), err_msg="%s[%d]" % (name, b))


def _check_self_loops_last(db, split, ids, p):
    heads, rels = db[2][0].cpu().numpy(), db[2][1].cpu().numpy()
    pos = 0
    for b, q in enumerate(ids):
        k, m = int(loader.kept_counts([split._stored[q]], p)[0]), int(split._ents[q])
        assert (rels[pos + k:pos + k + m] == split.self_rel).all()
        np.testing.assert_array_equal(heads[pos + k:pos + k + m], b * split.N + np.arange(m))
        pos += k + m
    assert pos == len(heads)


# ---- exact against the host drop-ins -----------------------------------------------------------------------------------

def _hub_loader(index_dtype):
    """test_device_split_gpu's hub: a 7 000-fact question whose head 3 holds ~70 % of its facts."""
    L = SplitLoader(seed=4, num_questions=3, max_local_entity=500, facts_lo=100, facts_hi=300,
                    index_dtype=IDX[index_dtype])
    rs = np.random.RandomState(0)
    n = 7000
    h = np.where(rs.rand(n) < 0.7, 3, rs.randint(0, 400, n))
    L.kb_adj_mats[1] = (h, rs.randint(0, 3, n), rs.randint(0, 400, n))
    L.global2local_entity_maps[1] = {k: k for k in range(400)}
    return L, [0, 1, 2]


def _cases():
    out = {name: (kw, ids) for name, (kw, ids, _drop, _seed) in CASES.items()}
    out["repeated_out_of_order"] = (dict(seed=9, num_questions=6, max_local_entity=30, facts_hi=200), [3, 3, 0, 5, 3])
    out["hub"] = None
    return out


@pytest.mark.parametrize("p", DROPS)
@pytest.mark.parametrize("index_dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("case", sorted(_cases()))
def test_arrays_equal_the_host_drop_in(case, index_dtype, p):
    spec = _cases()[case]
    if spec is None:
        L, ids = _hub_loader(index_dtype)
    else:
        kw, ids = spec
        L = SplitLoader(**kw, index_dtype=IDX[index_dtype])
    L.batches = np.asarray(ids)
    split = loader.DeviceSplit(L, dev, index_dtype=index_dtype, shuffle=True)
    state = np.random.get_state()
    torch.manual_seed(5)
    db = split.get_batch(0, len(ids), p, test=True)
    assert list(L.sample_ids) == list(ids)
    _check_structure(split, np.asarray(ids), p, 5)
    _check_self_loops_last(db, split, ids, p)
    hb = _host_tuple(L, split, np.asarray(ids), p, index_dtype) + (L.answer_lists[np.asarray(ids)],)
    _compare_tuples(hb, db, index_dtype)
    split.check()
    after = np.random.get_state()
    assert state[0] == after[0] and np.array_equal(state[1], after[1]) and state[2:] == after[2:]


@pytest.mark.parametrize("p", DROPS)
@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("index_dtype", [torch.int32, torch.int64])
def test_graft_arrays_equal_the_host_drop_in(index_dtype, inverse, p):
    L = GraftSplitLoader(seed=12, num_questions=7, max_local_entity=25, use_inverse_relation=inverse,
                         index_dtype=IDX[index_dtype])
    L.kb_adj_mats[2] = tuple(np.zeros(0, dtype=int) for _ in range(3))          # an empty question
    L.kb_fact_rels[2] = L.create_kb_adj_mats_facts(2)[1]
    ids = np.array([2, 6, 0, 0, 5, 1])
    L.batches = ids
    split = loader.DeviceSplit(L, dev, index_dtype=index_dtype, shuffle=True)
    torch.manual_seed(6)
    db = split.get_batch(0, len(ids), p)
    _check_structure(split, ids, p, 6)
    _compare_tuples(_host_tuple(L, split, ids, p, index_dtype), db, index_dtype, graft=True)
    split.check()


# ---- past shared memory ------------------------------------------------------------------------------------------------

def _one_question_loader(n, B, graft=False, N=64):
    cls = GraftSplitLoader if graft else SplitLoader
    L = cls(seed=3, num_questions=1, max_local_entity=N, facts_lo=1, facts_hi=1)
    rs = np.random.RandomState(1)
    L.kb_adj_mats[0] = (rs.randint(0, N, n), rs.randint(0, 5, n), rs.randint(0, N, n))
    L.global2local_entity_maps[0] = {k: k for k in range(N)}
    if graft:
        L.max_facts = n
        L.kb_fact_rels = np.full((1, n), L.num_kb_relation, dtype=int)
        L.kb_fact_rels[0] = L.create_kb_adj_mats_facts(0)[1]
    L.batches = np.zeros(B, dtype=np.int64)
    L.num_data = B
    return L


@pytest.mark.parametrize("n,p", [(8192, 0.0), (8193, 0.1), (9000, 0.5), (50000, 0.5), (50000, 0.1), (50000, 0.98),
                                 (120000, 0.3)])
def test_large_questions_equal_the_restated_order(n, p):
    """Questions past the shared-memory sort (bucketed through the workspace), next to a small one."""
    L = _one_question_loader(n, 3)
    split = loader.DeviceSplit(L, dev, weights="none", shuffle=True)
    torch.manual_seed(11)
    split.get_batch(0, 3, p)
    _check_structure(split, np.zeros(3, dtype=np.int64), p, 11)
    split.check()


def test_kept_fraction_per_decile_of_a_50k_question():
    n, p, draws = 50000, 0.5, 8
    L = _one_question_loader(n, draws)
    split = loader.DeviceSplit(L, dev, weights="none", shuffle=True)
    torch.manual_seed(12)
    split.get_batch(0, draws, p)
    split.check()
    # per decile: hypergeometric, 5 000 of 50 000 drawn with 25 000 kept: sd = sqrt(5000 * 0.25 * 0.9) ~ 33.5
    sd = np.sqrt(n / 10 * p * (1 - p) * 0.9)
    for run in _runs(split.last_order["kb"], split.last_order["kb_offsets"]):
        assert len(run) == n // 2
        per = np.bincount(run // (n // 10), minlength=10)
        assert np.abs(per - n // 20).max() < 6 * sd, per


# ---- uniformity ----------------------------------------------------------------------------------------------------------

def _draws(n, B, calls, torch_seed, p=0.0):
    L = _one_question_loader(n, B)
    split = loader.DeviceSplit(L, dev, weights="none", shuffle=True)
    torch.manual_seed(torch_seed)
    out = []
    for _ in range(calls):
        split.get_batch(0, B, p)
        out += _runs(split.last_order["kb"], split.last_order["kb_offsets"])
    split.check()
    return out


def test_all_24_orders_of_four_facts_are_equally_likely():
    runs = _draws(4, 1000, 4, 21)
    codes = [int(r[0]) * 64 + int(r[1]) * 16 + int(r[2]) * 4 + int(r[3]) for r in runs]
    uniq, counts = np.unique(codes, return_counts=True)
    assert len(uniq) == 24
    assert stats.chisquare(counts).pvalue > 1e-3


def test_fact_position_counts_of_64_facts_are_uniform():
    runs = np.stack(_draws(64, 1000, 4, 22))                          # [4000, 64]: fact at each position
    counts = np.zeros((64, 64))
    np.add.at(counts, (runs, np.broadcast_to(np.arange(64), runs.shape)), 1)
    expect = len(runs) / 64
    chi2 = ((counts - expect) ** 2 / expect).sum()
    assert stats.chi2.sf(chi2, 63 * 63) > 1e-3


def test_kb_and_graft_keep_masks_are_uncorrelated():
    n, B = 2000, 64
    L = _one_question_loader(n, B, graft=True)
    split = loader.DeviceSplit(L, dev, weights="none", shuffle=True)
    torch.manual_seed(23)
    split.get_batch(0, B, 0.5)
    o = split.last_order
    masks = {}
    for name in ("kb", "graft"):
        m = np.zeros((B, n), dtype=np.float64)
        for b, run in enumerate(_runs(o[name], o[name + "_offsets"])):
            m[b, run] = 1.0
        masks[name] = m.ravel()
    r = np.corrcoef(masks["kb"], masks["graft"])[0, 1]
    assert abs(r) < 5 / np.sqrt(n * B), r
    assert not np.array_equal(masks["kb"], masks["graft"])


# ---- reproducibility -----------------------------------------------------------------------------------------------------

def test_same_torch_seed_same_batch_and_numpy_untouched():
    L = GraftSplitLoader(seed=7, num_questions=6, max_local_entity=20)
    split = loader.DeviceSplit(L, dev, shuffle=True)
    np.random.seed(3)
    state = np.random.get_state()

    def flat(batch):
        (kb, graft) = batch[2], batch[3]
        return [t.cpu().numpy().copy() for t in list(kb) + list(graft[0]) + list(graft[1])]

    torch.manual_seed(31)
    a = flat(split.get_batch(0, 6, 0.3))
    a2 = flat(split.get_batch(0, 6, 0.3))
    torch.manual_seed(31)
    b = flat(split.get_batch(0, 6, 0.3))
    for x, y in zip(a, b):
        assert x.dtype == y.dtype and np.array_equal(x.view(np.uint8), y.view(np.uint8))
    assert any(not np.array_equal(x, y) for x, y in zip(a, a2))
    after = np.random.get_state()
    assert np.array_equal(state[1], after[1]) and state[2:] == after[2:]
    split.check()


# ---- consumers -------------------------------------------------------------------------------------------------------

def _train_once(m, batch):
    m.zero_grad(set_to_none=True)
    loss, _pred, pred_dist, tp = m(batch, training=True)
    loss.backward()
    return (_bits(loss).tolist(), _bits(pred_dist), tp,
            {n: _bits(p.grad) for n, p in m.named_parameters() if p.grad is not None})


@pytest.mark.parametrize("name", ["ReaRev", "NSM", "GraftNet"])
def test_eager_training_is_bit_equal(name):
    torch.use_deterministic_algorithms(True, warn_only=True)
    over = dict(normalized_gnn=True) if name == "ReaRev" else dict(norm_rel=True) if name == "GraftNet" else {}
    L = _loader(name)
    m = _train_mode(_model(name, L, eval_mode=False, **over))
    split = loader.DeviceSplit(L, dev, shuffle=True)
    for it in range(2):
        d = _train_once(m, split.get_batch(it, 6, 0.2))
        ids = np.asarray(L.sample_ids)
        h = _train_once(m, _host_tuple(L, split, ids, 0.2, torch.int32))
        assert h[0] == d[0]
        np.testing.assert_array_equal(h[1], d[1])
        assert h[2] == d[2]
        assert h[3].keys() == d[3].keys()
        for k in h[3]:
            np.testing.assert_array_equal(h[3][k], d[3][k], err_msg=k)
    split.check()


@pytest.mark.parametrize("name", ["ReaRev", "NSM"])
def test_graphed_train_step_is_bit_equal(name):
    torch.use_deterministic_algorithms(True, warn_only=True)
    L = _loader(name, index_dtype=np.int32)
    m = _train_mode(_model(name, L, eval_mode=False))
    split = loader.DeviceSplit(L, dev, shuffle=True)
    step = graphed.GraphedTrainStep(m)
    for it, p in ((0, 0.1), (1, 0.5), (0, 0.1)):          # varying F: the fact-capacity buckets absorb it
        db = split.get_batch(it, 6, p)
        hb = _host_tuple(L, split, np.asarray(L.sample_ids), p, torch.int32)
        outs = []
        for b in (hb, db):
            o = step.step(b)
            outs.append(([_bits(t) for t in o], {n: _bits(q.grad) for n, q in m.named_parameters()
                                                  if q.grad is not None}))
            o.check()
        for x, y in zip(outs[0][0], outs[1][0]):
            np.testing.assert_array_equal(x, y)
        for k in outs[0][1]:
            np.testing.assert_array_equal(outs[0][1][k], outs[1][1][k], err_msg=k)
    split.check()


@pytest.mark.parametrize("name", ["ReaRev", "NSM", "GraftNet"])
def test_no_dropout_matches_stored_order_up_to_summation_order(name):
    """shuffle=True with p = 0 keeps every fact, in another order: the same multiset, so the forward agrees within
    fp32 rounding of reordered sums."""
    L = _loader(name)
    m = _model(name, L)
    plain, shuffled = loader.DeviceSplit(L, dev), loader.DeviceSplit(L, dev, shuffle=True)
    for it in range(2):
        a, b = plain.get_batch(it, 6, 0.0), shuffled.get_batch(it, 6, 0.0)
        ka = np.stack([t.cpu().numpy() for t in a[2][:3]], 1)
        kb = np.stack([t.cpu().numpy() for t in b[2][:3]], 1)
        assert sorted(map(tuple, ka)) == sorted(map(tuple, kb)) and not np.array_equal(ka, kb)
        la, _pa, da, _ = m(a)
        lb, _pb, dbb, _ = m(b)
        np.testing.assert_allclose(dbb.cpu().numpy(), da.cpu().numpy(), rtol=1e-3, atol=1e-7)
        assert abs(float(la) - float(lb)) <= 2e-5 * abs(float(la)) + 1e-7


@pytest.mark.parametrize("name", ["ReaRev", "GraftNet"])
def test_get_batch_and_submit_do_not_synchronise(name):
    L = _loader(name)
    m = _model(name, L)
    split = loader.DeviceSplit(L, dev, shuffle=True)
    step = graphed.GraphedStep(m, NE)
    for it in range(2):                                   # warm-up: capture, pipeline buffers
        step.collect(step.submit(split.get_batch(it, 6, 0.1)))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        t0 = step.submit(split.get_batch(0, 6, 0.1))
        t1 = step.submit(split.get_batch(1, 6, 0.1))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    step.collect(t0)
    step.collect(t1)
    split.check()


# ---- status word -------------------------------------------------------------------------------------------------------

def test_ordered_assembly_status_word():
    L = SplitLoader(seed=3, num_questions=4, max_local_entity=12, facts_lo=5, facts_hi=30)
    split = loader.DeviceSplit(L, dev, shuffle=True)
    r, st = split._res, split._stored
    seed = torch.tensor([1234], dtype=torch.int64, device=dev)

    def run(bad, kept, F=None, K=None):
        ids = torch.tensor(bad, dtype=torch.int64, device=dev)
        kept_t = torch.tensor(kept, dtype=torch.int64, device=dev)
        good = [i for i in bad if 0 <= i < 4]
        K_ = int(sum(min(k, st[i]) for i, k in zip(bad, kept) if 0 <= i < 4)) if K is None else K
        order, ost = ops.split_fact_order(r["q_off"], ids, kept_t, seed, 0, int(st[good].sum()), K_)
        F_ = K_ + int(split._ents[good].sum()) if F is None else F
        out = ops.split_assemble(r["q_off"], r["q_heads"], r["q_rels"], r["q_tails"], r["q_ents"], ids, 12, F_,
                                 NR_SELF, True, torch.int32, kept=kept_t, order=order)
        return int(ost.item()), int(out[5].item())

    NR_SELF = split.self_rel
    assert run([0, 1], [3, 4]) == (0, 0)
    assert run([1, 4, 2], [3, 3, 3]) == (1, 1)                       # an id out of range: an empty question
    assert run([-1, 0], [2, 2]) == (1, 1)
    ost, ast = run([0, 1, 2], [3, 3, 3], K=5)                        # the order past its capacity: questions 1
    assert ost == 2 and ast & 2                                       # and 2 are not written
    assert run([0, 1, 2], [3, 3, 3], F=5) == (0, 2)                  # the facts past theirs
    # an order entry that is not a stored index of its question
    ids = torch.tensor([0, 1], dtype=torch.int64, device=dev)
    kept = torch.tensor([2, 2], dtype=torch.int64, device=dev)
    order = torch.tensor([0, 1, 0, int(st[1])], dtype=torch.int32, device=dev)
    out = ops.split_assemble(r["q_off"], r["q_heads"], r["q_rels"], r["q_tails"], r["q_ents"], ids, 12,
                             4 + int(split._ents[[0, 1]].sum()), NR_SELF, True, torch.int32, kept=kept, order=order)
    assert int(out[5].item()) == 1
    G_ = GraftSplitLoader(seed=5, num_questions=3, max_local_entity=9, facts_lo=5)
    gs = loader.DeviceSplit(G_, dev, shuffle=True)
    r = gs._res
    ids = torch.tensor([0, 3], dtype=torch.int64, device=dev)
    kept = torch.tensor([2, 2], dtype=torch.int64, device=dev)
    gorder, ost = ops.split_fact_order(r["g_off"], ids, kept, seed, 1, int(gs._graft_count[0]), 2)
    _g, kfr, gst = ops.split_assemble_graft(r["g_off"], r["g_e2f_f"], r["g_e2f_e"], r["g_f2e_e"], r["g_f2e_f"],
                                            r["r_off"], r["r_vals"], ids, gs.max_facts, gs.rel_pad, 2, torch.int32,
                                            kept=kept, order=gorder)
    assert int(ost.item()) == 1 and int(gst.item()) == 1 and bool((kfr[1] == gs.rel_pad).all())
    _g, _kfr, gst = ops.split_assemble_graft(r["g_off"], r["g_e2f_f"], r["g_e2f_e"], r["g_f2e_e"], r["g_f2e_f"],
                                             r["r_off"], r["r_vals"], ids[:1], gs.max_facts, gs.rel_pad, 1,
                                             torch.int32, kept=kept[:1], order=gorder)
    assert int(gst.item()) == 2


# ---- one kernel per list: stored order is the ordered path through the identity order ----------------------------------

@pytest.mark.parametrize("cut,bad", [(0, False), (3, False), (0, True)])
@pytest.mark.parametrize("index_dtype", [torch.int32, torch.int64])
def test_stored_order_equals_the_identity_order(index_dtype, cut, bad):
    """The stored-order assembly and the ordered one at kept = the stored counts through the identity order write the
    same bits and the same status word, kb facts and graft lists: at the exact capacity, at a capacity ``cut`` short
    (bit 2) and with an out-of-range id (bit 1).  Outputs start as a sentinel, so unwritten entries compare too."""
    L = GraftSplitLoader(seed=8, num_questions=5, max_local_entity=16, facts_lo=3, facts_hi=40,
                         index_dtype=IDX[index_dtype])
    split = loader.DeviceSplit(L, dev, index_dtype=index_dtype)
    r = split._res
    ids_h = np.array([3, 0, 5, 2] if bad else [3, 0, 4, 2])
    ids, good = torch.tensor(ids_h, device=dev), ids_h[ids_h < 5]

    def identity(stored):
        n = np.array([stored[i] if i < 5 else 0 for i in ids_h], dtype=np.int64)
        order = np.concatenate([np.arange(k) for k in n]).astype(np.int32)
        return dict(kept=torch.tensor(n, device=dev), order=torch.tensor(order, device=dev))

    def bits(ts):
        return [t.cpu().numpy().view(np.uint8) for t in ts]

    want = (1 if bad else 0) | (2 if cut else 0)
    F = int(split._count[good].sum()) - cut
    kb = []
    for extra in ({}, identity(split._stored)):
        out = [torch.full((F,), -7, dtype=index_dtype, device=dev) for _ in range(5)]
        *arrays, st = ops.split_assemble(r["q_off"], r["q_heads"], r["q_rels"], r["q_tails"], r["q_ents"], ids,
                                         split.N, F, split.self_rel, split.use_self_loop, index_dtype, out=out,
                                         **extra)
        kb.append((bits(arrays), int(st.item())))
    G = int(split._graft_count[good].sum()) - cut
    lists = (r["g_off"], r["g_e2f_f"], r["g_e2f_e"], r["g_f2e_e"], r["g_f2e_f"], r["r_off"], r["r_vals"])
    graft = []
    for extra in ({}, identity(split._graft_count)):
        out = tuple(tuple(torch.full((G,), -7, dtype=dt, device=dev) for dt in (index_dtype,) * 3 + (torch.float32,))
                    for _ in range(2)) + (torch.full((len(ids_h), split.max_facts), -7, device=dev),)
        (e2f, f2e), kfr, st = ops.split_assemble_graft(*lists, ids, split.max_facts, split.rel_pad, G, out=out,
                                                       **extra)
        graft.append((bits((*e2f, *f2e, kfr)), int(st.item())))
    for name, (stored, ordered) in (("kb", kb), ("graft", graft)):
        assert stored[1] == ordered[1] == want, name
        for i, (a, b) in enumerate(zip(stored[0], ordered[0])):
            np.testing.assert_array_equal(a, b, err_msg="%s[%d]" % (name, i))


def test_kept_and_order_come_together():
    L = GraftSplitLoader(seed=5, num_questions=3, max_local_entity=9, facts_lo=5)
    split = loader.DeviceSplit(L, dev, shuffle=True)
    r = split._res
    ids = torch.tensor([0, 1], dtype=torch.int64, device=dev)
    kept = torch.tensor([2, 2], dtype=torch.int64, device=dev)
    order = torch.tensor([0, 1, 0, 1], dtype=torch.int32, device=dev)
    lists = (r["g_off"], r["g_e2f_f"], r["g_e2f_e"], r["g_f2e_e"], r["g_f2e_f"], r["r_off"], r["r_vals"])
    for half, only in ((dict(kept=kept), "kept"), (dict(order=order), "order")):
        with pytest.raises(RuntimeError, match="split_assemble: kept and order come together, got only " + only):
            ops.split_assemble(r["q_off"], r["q_heads"], r["q_rels"], r["q_tails"], r["q_ents"], ids, split.N, 8,
                               split.self_rel, True, torch.int32, **half)
        with pytest.raises(RuntimeError, match="split_assemble_graft: kept and order come together, got only " + only):
            ops.split_assemble_graft(*lists, ids, split.max_facts, split.rel_pad, 4, torch.int32, **half)
