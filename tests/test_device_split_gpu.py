"""loader.DeviceSplit on the GPU: batches assembled on the device from question ids (csrc/split.cu).

The arrays equal the host drop-ins element for element (loader.build_fact_mat(shuffle=False), GraftNet's
build_fact_mat_maxfacts under the identity permutation) with bit-equal fp32 weights, and every consumer gives the same
bits on the device tuple as on the host tuple: model(batch), ranking, GraphedStep (call and submit/collect), eager
training and GraphedTrainStep under torch.use_deterministic_algorithms, and Evaluator.evaluate."""
import json
import os

import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import evaluate, graphed, loader, ops, synthetic as S
from test_device_split_host import NE, NR, NW, GraftSplitLoader, SplitLoader, fake_cases

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
IDX = {torch.int32: np.int32, torch.int64: np.int64}


@pytest.fixture(autouse=True)
def _deterministic():
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        yield
    torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])


def _eq(host, devt, name):
    if host is None:
        assert devt is None, name
        return
    assert devt.is_cuda, name
    h = np.asarray(host)
    d = devt.cpu().numpy()
    assert d.shape == h.shape, (name, d.shape, h.shape)
    if h.dtype.kind == "f":
        np.testing.assert_array_equal(d.view(np.uint32), h.astype(np.float32).view(np.uint32), err_msg=name)
    else:
        np.testing.assert_array_equal(d, h, err_msg=name)


def _compare_tuples(hb, db, index_dtype, graft=False):
    assert len(hb) == len(db)
    le, qe, kb = db[0], db[1], db[2]
    assert le.dtype == torch.int64 and qe.dtype == torch.float32
    for i in (0, 1):
        _eq(hb[i], db[i], "tuple[%d]" % i)
    for k, (x, y) in enumerate(zip(hb[2], kb)):
        if k < 5:
            assert y.dtype == index_dtype, k
        _eq(x, y, "kb[%d]" % k)
    rest = (3, 4, 5, 6, 8) if graft else (3, 4, 6)
    for i in rest:
        if i == 3 and graft:
            for lh, ld in zip(hb[3], db[3]):
                for k, (x, y) in enumerate(zip(lh, ld)):
                    _eq(x, y, "graft[%d]" % k)
        else:
            _eq(hb[i], db[i], "tuple[%d]" % i)
    assert db[7 if graft else 5] is None
    if len(hb) > (9 if graft else 7):
        assert db[-1] is hb[-1] or list(db[-1]) == list(hb[-1])


# ---- arrays --------------------------------------------------------------------------------------------------------

def _with_order(L, ids):
    L.batches = np.asarray(ids)
    return L


@pytest.mark.parametrize("index_dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("case", sorted(fake_cases()))
def test_arrays_equal_the_host_drop_in(case, index_dtype):
    kw, ids = fake_cases()[case]
    L = _with_order(SplitLoader(**kw, index_dtype=IDX[index_dtype]), ids)
    split = loader.DeviceSplit(L, dev, index_dtype=index_dtype)
    for it, bs in ((0, len(ids)), (0, 2), (1, 2)):
        hb = L.get_batch(it, bs, 0.0, test=True)
        host_ids = list(L.sample_ids)
        db = split.get_batch(it, bs, 0.0, test=True)
        assert list(L.sample_ids) == host_ids
        _compare_tuples(hb, db, index_dtype)
    split.check()


@pytest.mark.parametrize("ids", [[3, 3, 0, 5, 3], [5, 4, 3, 2, 1, 0], [2]])
def test_repeated_and_out_of_order_ids(ids):
    L = _with_order(SplitLoader(seed=9, num_questions=6, max_local_entity=30, facts_hi=200), ids)
    split = loader.DeviceSplit(L, dev)
    _compare_tuples(L.get_batch(0, len(ids), 0.0), split.get_batch(0, len(ids), 0.0), torch.int32)


def test_hub_head_weights_are_bit_equal():
    """A head with thousands of facts over few relations, next to singleton rows: integer counts, one rounding."""
    L = SplitLoader(seed=4, num_questions=3, max_local_entity=500, facts_lo=100, facts_hi=300)
    rs = np.random.RandomState(0)
    n = 7000
    h = np.where(rs.rand(n) < 0.7, 3, rs.randint(0, 400, n))
    r = rs.randint(0, 3, n)
    L.kb_adj_mats[1] = (h, r, rs.randint(0, 400, n))
    L.global2local_entity_maps[1] = {k: k for k in range(400)}
    split = loader.DeviceSplit(L, dev, index_dtype=torch.int64)
    _compare_tuples(L.get_batch(0, 3, 0.0), split.get_batch(0, 3, 0.0), torch.int64)


@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("index_dtype", [torch.int32, torch.int64])
def test_graft_arrays_equal_the_host_drop_in(inverse, index_dtype):
    L = GraftSplitLoader(seed=12, num_questions=7, max_local_entity=25, use_inverse_relation=inverse,
                         index_dtype=IDX[index_dtype])
    L.kb_adj_mats[2] = tuple(np.zeros(0, dtype=int) for _ in range(3))          # an empty question
    L.kb_fact_rels[2] = L.create_kb_adj_mats_facts(2)[1]
    _with_order(L, [2, 6, 0, 0, 5, 1])
    split = loader.DeviceSplit(L, dev, index_dtype=index_dtype)
    for it, bs in ((0, 6), (1, 4), (2, 2)):
        _compare_tuples(L.get_batch(it, bs, 0.0, test=True), split.get_batch(it, bs, 0.0, test=True), index_dtype,
                        graft=True)
    split.check()


def test_weights_none_and_pass_throughs():
    L = SplitLoader(seed=2, num_questions=5, max_local_entity=10)
    split = loader.DeviceSplit(L, dev, weights="none")
    b = split.get_batch(0, 5, 0.0)
    assert b[2][5] is None and b[2][6] is None
    assert split.num_data == 5 and split.max_local_entity == 10
    assert split.get_quest() == ["question %d" % i for i in range(5)]
    split.reset_batches(is_sequential=False)
    assert sorted(L.batches.tolist()) == list(range(5))
    assert split.resident_bytes > 0 and split.build_seconds >= 0


def test_refusals():
    L = SplitLoader(seed=2, num_questions=5, max_local_entity=10)
    split = loader.DeviceSplit(L, dev)
    with pytest.raises(ValueError, match="fact_dropout must be 0"):
        split.get_batch(0, 2, 0.1)
    with pytest.raises(ValueError, match="q_type must be 'seq'"):
        split.get_batch(0, 2, 0.0, q_type="bert")
    L.batches = np.array([0, 7])
    with pytest.raises(ValueError, match=r"question ids outside \[0, 5\)"):
        split.get_batch(0, 2, 0.0)
    big = SplitLoader(seed=2, num_questions=2, max_local_entity=4)
    big.max_local_entity = 2 ** 30                       # B * N = 2^31: past int32 (the [num_q, N] tables stay small)
    s2 = loader.DeviceSplit(big, dev, weights="none")
    with pytest.raises(ValueError, match="overflows int32 indices"):
        s2.get_batch(0, 2, 0.0)


def test_out_of_range_question_id_sets_the_status_word():
    L = SplitLoader(seed=3, num_questions=4, max_local_entity=12)
    split = loader.DeviceSplit(L, dev)
    r = split._res
    count = split._count
    for bad, want in (([1, 4, 2], 1), ([-1, 0], 1), ([0, 1], 0)):
        ids = torch.tensor(bad, dtype=torch.int64, device=dev)
        F = int(sum(count[i] for i in bad if 0 <= i < 4))
        out = ops.split_assemble(r["q_off"], r["q_heads"], r["q_rels"], r["q_tails"], r["q_ents"], ids, 12, F,
                                 NR - 1, True, torch.int32)
        assert int(out[5].item()) == want
    ids = torch.tensor([0, 1, 2], dtype=torch.int64, device=dev)
    F = int(count[[0, 1, 2]].sum())
    out = ops.split_assemble(r["q_off"], r["q_heads"], r["q_rels"], r["q_tails"], r["q_ents"], ids, 12, F - 3,
                             NR - 1, True, torch.int32)
    assert int(out[5].item()) == 2                       # capacity too small: cut, flagged
    G_ = GraftSplitLoader(seed=5, num_questions=3, max_local_entity=9)
    gs = loader.DeviceSplit(G_, dev)
    r = gs._res
    _g, kfr, st = ops.split_assemble_graft(r["g_off"], r["g_e2f_f"], r["g_e2f_e"], r["g_f2e_e"], r["g_f2e_f"],
                                           r["r_off"], r["r_vals"], torch.tensor([0, 3], device=dev), gs.max_facts,
                                           gs.rel_pad, int(gs._graft_count[0]), torch.int32)
    assert int(st.item()) == 1 and bool((kfr[1] == gs.rel_pad).all())


# ---- consumers -------------------------------------------------------------------------------------------------------

def _model(name, L, D=50, eval_mode=True, **over):
    """A model over the stand-in loader ``L``'s vocabularies (relations: L.num_kb_relation, the self-loop included)."""
    torch.manual_seed(0)
    args = S.model_args(name, entity_dim=D, use_cuda=True, word_dim=64, linear_dropout=0.0, lm_dropout=0.0, **over)
    if name == "ReaRev":
        args.update(num_ins=2, num_iter=2, num_gnn=2)
    elif name == "NSM":
        args.update(num_step=2)
    else:
        args.update(num_layer=2)
    cls = {"ReaRev": G.ReaRev, "NSM": G.NSM, "GraftNet": G.GraftNet}[name]
    m = cls(dict(args), NE, L.num_kb_relation, NW).cuda()
    return m.eval() if eval_mode else m


def _loader(name, B=6, N=60, seed=21, **kw):
    cls = GraftSplitLoader if name == "GraftNet" else SplitLoader
    L = cls(seed=seed, num_questions=2 * B + 1, max_local_entity=N, facts_lo=20, facts_hi=150, **kw)
    return L


MODELS = ["ReaRev", "NSM", "GraftNet"]


def _bits(t):
    return t.detach().float().cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("name", MODELS)
def test_model_forward_and_ranking_are_bit_equal(name):
    L = _loader(name)
    m = _model(name, L, normalized_gnn=(name == "ReaRev"))
    split = loader.DeviceSplit(L, dev)
    for it in range(2):
        hb = L.get_batch(it, 6, 0.0)
        db = split.get_batch(it, 6, 0.0)
        lh, _ph, dh, _ = m(hb)
        rh, _ = evaluate.retrieve(dh, m.last_batch, NE, 0.95)
        ld, _pd, dd, _ = m(db)
        rd, _ = evaluate.retrieve(dd, m.last_batch, NE, 0.95)
        np.testing.assert_array_equal(_bits(dh), _bits(dd))
        assert _bits(lh).tolist() == _bits(ld).tolist()
        for a, b in zip(rh, rd):
            np.testing.assert_array_equal(a.ent, b.ent)
            np.testing.assert_array_equal(a.prob.view(np.uint32), b.prob.view(np.uint32))


@pytest.mark.parametrize("name", MODELS)
def test_graphed_step_call_and_pipeline_are_bit_equal(name):
    L = _loader(name, index_dtype=np.int32)
    m = _model(name, L)
    split = loader.DeviceSplit(L, dev)
    step = graphed.GraphedStep(m, NE)
    for it in range(2):
        hb, db = L.get_batch(it, 6, 0.0), split.get_batch(it, 6, 0.0)
        oh = step(hb)
        dh, rh = oh.pred_dist.clone(), step.retrieve(oh)[0]
        od = step(db)
        np.testing.assert_array_equal(_bits(dh), _bits(od.pred_dist))
        for a, b in zip(rh, step.retrieve(od)[0]):
            np.testing.assert_array_equal(a.ent, b.ent)
    got = {}
    for src in ("host", "device"):
        res = []
        tickets = []
        for it in range(2):
            b = L.get_batch(it, 6, 0.0) if src == "host" else split.get_batch(it, 6, 0.0)
            tickets.append(step.submit(b))
            if len(tickets) == 2:
                res.append(step.collect(tickets.pop(0)))
        res += [step.collect(t) for t in tickets]
        got[src] = res
    for (rh, _nh, lh, ph), (rd, _nd, ld, pd) in zip(got["host"], got["device"]):
        assert np.float32(lh).view(np.uint32) == np.float32(ld).view(np.uint32)
        np.testing.assert_array_equal(ph, pd)
        for a, b in zip(rh, rd):
            np.testing.assert_array_equal(a.idx, b.idx)
            np.testing.assert_array_equal(a.ent, b.ent)
            np.testing.assert_array_equal(a.prob.view(np.uint32), b.prob.view(np.uint32))


def _train_once(m, batch):
    m.zero_grad(set_to_none=True)
    loss, _pred, pred_dist, tp = m(batch, training=True)
    loss.backward()
    return (_bits(loss).tolist(), _bits(pred_dist), tp,
            {n: _bits(p.grad) for n, p in m.named_parameters() if p.grad is not None})


def _train_mode(m):
    m.train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.eval()
    return m


@pytest.mark.parametrize("name", MODELS)
def test_eager_training_is_bit_equal(name):
    torch.use_deterministic_algorithms(True, warn_only=True)
    over = dict(normalized_gnn=True) if name == "ReaRev" else dict(norm_rel=True) if name == "GraftNet" else {}
    L = _loader(name)
    m = _train_mode(_model(name, L, eval_mode=False, **over))
    split = loader.DeviceSplit(L, dev)
    h = _train_once(m, L.get_batch(0, 6, 0.0))
    d = _train_once(m, split.get_batch(0, 6, 0.0))
    assert h[0] == d[0]
    np.testing.assert_array_equal(h[1], d[1])
    assert h[2] == d[2]
    assert h[3].keys() == d[3].keys()
    for k in h[3]:
        np.testing.assert_array_equal(h[3][k], d[3][k], err_msg=k)


@pytest.mark.parametrize("name", ["ReaRev", "NSM"])
def test_graphed_train_step_is_bit_equal(name):
    torch.use_deterministic_algorithms(True, warn_only=True)
    L = _loader(name, index_dtype=np.int32)
    m = _train_mode(_model(name, L, eval_mode=False))
    split = loader.DeviceSplit(L, dev)
    step = graphed.GraphedTrainStep(m)
    outs = []
    for b in (L.get_batch(0, 6, 0.0), split.get_batch(0, 6, 0.0)):
        o = step.step(b)
        outs.append(([_bits(t) for t in o], {n: _bits(p.grad) for n, p in m.named_parameters()
                                              if p.grad is not None}))
        o.check()
    for x, y in zip(outs[0][0], outs[1][0]):
        np.testing.assert_array_equal(x, y)
    for k in outs[0][1]:
        np.testing.assert_array_equal(outs[0][1][k], outs[1][1][k], err_msg=k)


@pytest.mark.parametrize("name", ["ReaRev", "GraftNet"])
def test_get_batch_and_submit_do_not_synchronise(name):
    L = _loader(name)
    m = _model(name, L)
    split = loader.DeviceSplit(L, dev)
    step = graphed.GraphedStep(m, NE)
    for it in range(2):                                   # warm-up: capture, pipeline buffers
        step.collect(step.submit(split.get_batch(it, 6, 0.0)))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        t0 = step.submit(split.get_batch(0, 6, 0.0))
        t1 = step.submit(split.get_batch(1, 6, 0.0))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    step.collect(t0)
    step.collect(t1)


@pytest.mark.parametrize("name", ["ReaRev", "GraftNet"])
def test_evaluator_runs_on_a_split(name, tmp_path):
    L = _loader(name)
    m = _model(name, L)
    args = dict(S.model_args(name), checkpoint_dir=str(tmp_path), experiment_name="x", eps=0.95)
    ent = {"e%d" % i: i for i in range(NE + 1)}
    rel = {"r%d" % i: i for i in range(NR)}
    res = {}
    for src, data in (("host", L), ("device", loader.DeviceSplit(L, dev))):
        ev = evaluate.Evaluator(args, m, ent, rel, dev)
        res[src] = ev.evaluate(data, test_batch_size=5)
        res[src + "_rows"] = open(os.path.join(str(tmp_path), "x_test.info")).read()
    assert res["host"] == res["device"]
    assert res["host_rows"] == res["device_rows"] and json.loads(res["host_rows"].splitlines()[0])
