"""Host half of tests/test_gemm_layouts_gpu.py: the float64 layer references against the oracle modules run in
float64, the N > 256 column-slice arithmetic of ops.linear_tc_planes restated in numpy, and the weight pre-split
cache's key and version rules."""
import numpy as np
import pytest
import torch

from gnn_rag_b200 import ops
from oracle import graft_oracle as GO
from oracle import kgqa_oracle as O

import fp64_ref as R

F64 = torch.float64


def _facts(rs, B, N, E, R1):
    h = (rs.randint(0, N, size=(B, E)) + np.arange(B)[:, None] * N).ravel()
    t = (rs.randint(0, N, size=(B, E)) + np.arange(B)[:, None] * N).ravel()
    r = rs.randint(0, R1, size=len(h))
    t[:40] = 0                                                     # a hub row
    h[:40] = rs.randint(1, N, size=40)
    return h, r, t


def _mats(h, r, t, B, N, w):
    """oracle FactMats over (h, r, t) with weights ``w`` (or none), its COO operators in float64."""
    kb = (h, r, t, h // N, np.arange(len(h)), None if w is None else list(w), None)
    mats = O.FactMats(kb, B, N, w is not None)
    for name in ("fact2head", "head2fact", "fact2tail", "tail2fact"):
        setattr(mats, name, getattr(mats, name).to(F64))
    return mats


def _sd(rs, D, T, R1):
    d = lambda *s: torch.tensor(rs.randn(*s), dtype=F64)          # noqa: E731
    return {"reasoning.rel_linear0.weight": d(D, D) / np.sqrt(D), "reasoning.rel_linear0.bias": d(D) * 0.1,
            "reasoning.e2e_linear0.weight": d(D, T * D) / np.sqrt(T * D), "reasoning.e2e_linear0.bias": d(D) * 0.1,
            "reasoning.score_func.weight": d(1, D), "reasoning.score_func.bias": d(1)}


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("reason_kb", [False, True])
def test_nsm_layer_matches_oracle_step(reason_kb, weighted):
    rs = np.random.RandomState(2 * reason_kb + weighted)
    B, N, E, R1, D = 3, 30, 60, 7, 12
    h, r, t = _facts(rs, B, N, E, R1)
    w = rs.uniform(0.2, 1.5, size=len(h)).astype(np.float32) if weighted else None   # FactMats keeps fp32 values
    mats = _mats(h, r, t, B, N, w)
    sd = _sd(rs, D, 2, R1)
    rel_f = torch.tensor(rs.randn(R1, D), dtype=F64)
    hn = torch.tensor(rs.randn(B, N, D), dtype=F64)
    prior = torch.softmax(torch.tensor(rs.randn(B, N), dtype=F64), 1)
    prior[:, ::3] = 0
    ins = torch.tensor(rs.randn(B, D), dtype=F64)
    mask = torch.tensor((rs.rand(B, N) < 0.8).astype(np.float64))
    dist, h_new, poss = O.nsm_gnn_step(sd, mats, hn, prior, ins, rel_f, mask, 0, reason_kb)
    table = rel_f @ sd["reasoning.rel_linear0.weight"].t() + sd["reasoning.rel_linear0.bias"]
    facts = tuple(torch.as_tensor(a) for a in (h, r, t))
    y, s, p = R.nsm_layer(hn.view(B * N, D), prior, table, ins, sd["reasoning.e2e_linear0.weight"],
                          sd["reasoning.e2e_linear0.bias"], sd["reasoning.score_func.weight"].view(-1), facts,
                          None if w is None else torch.tensor(w))
    assert torch.allclose(y, h_new.view(B * N, D), rtol=1e-12, atol=1e-12)
    assert torch.equal(p, poss.view(-1))
    assert (p == 0).any() and (p == 1).any()
    m = mask * poss if reason_kb else mask
    z = s.view(B, N) + sd["reasoning.score_func.bias"] + (1 - m) * O.VERY_NEG_NUMBER
    assert torch.allclose(torch.softmax(z, 1), dist, rtol=1e-12, atol=1e-15)
    sc = R.nsm_layer_scale(hn.view(B * N, D), prior, table, ins, sd["reasoning.e2e_linear0.weight"],
                           sd["reasoning.e2e_linear0.bias"], facts, None if w is None else torch.tensor(w))
    assert (sc + 1e-12 >= (y - 0).abs()).all()


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("I", [1, 2, 3])
def test_rearev_layer_matches_oracle_step(I, weighted):
    rs = np.random.RandomState(10 * I + weighted)
    B, N, E, R1, D = 3, 25, 50, 6, 10
    h, r, t = _facts(rs, B, N, E, R1)
    w = rs.uniform(0.2, 1.5, size=len(h)).astype(np.float32) if weighted else None   # FactMats keeps fp32 values
    mats = _mats(h, r, t, B, N, w)
    sd = _sd(rs, D, 2 * I + 1, R1)
    rel_f, rel_fi = (torch.tensor(rs.randn(R1, D), dtype=F64) for _ in range(2))
    hn = torch.tensor(rs.randn(B, N, D), dtype=F64)
    prior = torch.softmax(torch.tensor(rs.randn(B, N), dtype=F64), 1)
    ins = torch.tensor(rs.randn(B, I, D), dtype=F64)
    mask = torch.ones(B, N, dtype=F64)
    _dist, h_new, score = O.rearev_gnn_step(sd, mats, hn, prior, ins, rel_f, rel_fi, mask, 0)
    Wr, br = sd["reasoning.rel_linear0.weight"], sd["reasoning.rel_linear0.bias"]
    y, s = R.rearev_layer(hn.view(B * N, D), prior, rel_f @ Wr.t() + br, rel_fi @ Wr.t() + br, ins,
                          sd["reasoning.e2e_linear0.weight"], sd["reasoning.e2e_linear0.bias"],
                          sd["reasoning.score_func.weight"].view(-1), tuple(torch.as_tensor(a) for a in (h, r, t)),
                          None if w is None else torch.tensor(w))
    assert torch.allclose(y, h_new.view(B * N, D), rtol=1e-12, atol=1e-12)
    assert torch.allclose(s + sd["reasoning.score_func.bias"], score.view(-1), rtol=1e-12, atol=1e-12)


# ---- N > 256: column slices -------------------------------------------------------------------------------------------

def _slices(N, max_n=256):
    """ops.linear_tc_planes' slicing of N > max_n output columns, restated."""
    nsl = -(-N // max_n)
    step = (-(-N // nsl) + 15) // 16 * 16
    return [(n0, min(N, n0 + step)) for n0 in range(0, N, step)]


def test_column_slices_arithmetic():
    """Every N the wide path admits: slices of at most 256 columns, starting on 16-column boundaries, tiling [0, N),
    as few as 256-column launches allow, and the planes each slice writes (to round16 of its width) end inside
    round16(N): no slice writes into another's columns or past the buffer a caller sized for N."""
    assert ops.TC_MAX_N == 256 and ops.TC_MAX_N_SPLIT == 512
    for N in range(ops.TC_MAX_N + 1, ops.TC_MAX_N_SPLIT + 1):
        sl = _slices(N)
        assert sl[0][0] == 0 and sl[-1][1] == N and len(sl) == -(-N // 256)
        assert all(a[1] == b[0] for a, b in zip(sl, sl[1:]))
        assert all(0 < n1 - n0 <= 256 and n0 % 16 == 0 for n0, n1 in sl)
        assert all(n0 + (n1 - n0 + 15) // 16 * 16 <= (N + 15) // 16 * 16 for n0, n1 in sl)
    assert _slices(300) == [(0, 160), (160, 300)] and _slices(400) == [(0, 208), (208, 400)]
    assert _slices(257) == [(0, 144), (144, 257)] and _slices(512) == [(0, 256), (256, 512)]


def test_column_slices_are_what_the_wrapper_launches(monkeypatch):
    """The launches ops.linear_tc_planes issues for N > 256 (recorded instead of run): one per slice of _slices, with
    the slice's W rows, bias, w_score, output columns and planes columns."""
    launched = []
    monkeypatch.setattr(ops, "_launch", lambda name, *a, **kw: launched.append(a))
    monkeypatch.setattr(ops, "_weight_ws", lambda W, N, K, k_seg, pitch, nbytes: (torch.empty(0), True))

    class _Lib:
        @staticmethod
        def gr_linear_tc_planes_workspace_bytes(N, K):
            return 0
    monkeypatch.setattr(ops, "_L", lambda: _Lib)
    M, K = 5, 64
    for N in (257, 300, 400, 512):
        launched.clear()
        hi = torch.zeros(M, K, dtype=torch.bfloat16)
        W, b, ws = torch.zeros(N, K), torch.zeros(N), torch.zeros(N)
        out = torch.zeros(M, N)
        ph, pl = torch.zeros(M, N + 16, dtype=torch.bfloat16), torch.zeros(M, N + 16, dtype=torch.bfloat16)
        dots = torch.zeros(2 * M)
        ops.linear_tc_planes(hi, hi, K, W, b, out=out, out_planes=(ph, pl), w_score=ws, dots=dots)
        want = _slices(N)
        assert len(launched) == len(want)
        for a, (n0, n1) in zip(launched, want):
            assert a[3].value == W[n0].data_ptr() and a[5].value == b[n0].data_ptr()
            assert a[6].value == out[0, n0].data_ptr() and a[8].value == ph[0, n0].data_ptr()
            assert a[11].value == ws[n0].data_ptr() and a[14] == n1 - n0
        assert launched[0][12].value == dots.data_ptr()
        assert all(a[12].value != dots.data_ptr() for a in launched[1:])


# ---- the weight pre-split cache ---------------------------------------------------------------------------------------

@pytest.fixture
def cache(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    ops.clear_weight_cache()
    yield
    ops.clear_weight_cache()


def test_cache_key_separates_views_and_layouts(cache):
    """``W`` and ``W[:, :D]`` share data_ptr and stride but differ in K; the plain, segmented, fused and K-order
    layouts of one W differ in k_seg / the layout tag: each gets buffers of its own."""
    D, T = 8, 5
    W = torch.randn(D, T * D)
    keys = [(W, D, T * D, 0, 0), (W[:, :D], D, 16, D, 16), (W, D, T * 16, D, 16), (W, D, T * D, "fused", 16),
            (W, D, T * D, "korder", 16)]
    bufs = [ops._weight_ws(Wv, N, K, ks, p, 64)[0] for Wv, N, K, ks, p in keys]
    assert len({b.data_ptr() for b in bufs}) == len(bufs)
    again = [ops._weight_ws(Wv, N, K, ks, p, 64) for Wv, N, K, ks, p in keys]
    assert all(cur and b.data_ptr() == a.data_ptr() for (b, cur), a in zip(again, bufs))


def test_cache_follows_versions_and_owners(cache):
    """An in-place update (on the tensor or on a view of it) makes the entry stale -- same buffers, re-formatted by
    the caller; another tensor object over the same storage is the same owner; a ``.data`` write does not bump the
    version (the documented case clear_weight_cache() is for).  A weight re-created at the same address is held on
    the GPU (test_gemm_layouts_gpu.py), where the caching allocator hands the address back."""
    W = torch.randn(8, 40)
    ws, cur = ops._weight_ws(W, 8, 40, 0, 0, 64)
    assert not cur
    assert ops._weight_ws(W, 8, 40, 0, 0, 64) == (ws, True)
    W.mul_(2)
    ws2, cur = ops._weight_ws(W, 8, 40, 0, 0, 64)
    assert ws2 is ws and not cur
    W[:, :8].add_(1)                                   # through a view: the shared version counter moves
    assert ops._weight_ws(W, 8, 40, 0, 0, 64)[1] is False
    assert ops._weight_ws(W[:, :8], 8, 8, 0, 0, 64)[1] is False      # the view's own first use
    W.data.mul_(2)
    assert ops._weight_ws(W, 8, 40, 0, 0, 64)[1] is True            # documented: .data writes are not seen
    ops.clear_weight_cache()
    assert ops._weight_ws(W, 8, 40, 0, 0, 64)[1] is False
    storage = torch.empty(8 * 40)
    A = storage.view(8, 40)
    ops._weight_ws(A, 8, 40, 0, 0, 64)
    Bv = storage.view(8, 40)                           # another tensor object over the same storage
    assert Bv.data_ptr() == A.data_ptr() and ops._weight_ws(Bv, 8, 40, 0, 0, 64)[1] is True   # same _base: same owner


# ---- GraftNet ---------------------------------------------------------------------------------------------------------

def graft_lin(layer, i):
    """name -> (W, b) of GraftLayer ``layer``'s linears of layer i, as fp64_ref.graft_layer takes them."""
    return {k: tuple(getattr(layer.lin(k + "_linear", i), a).detach().to(F64) for a in ("weight", "bias"))
            for k in ("q2e", "e2q", "e2e", "kb_head", "kb_tail", "kb_self")}


@pytest.mark.parametrize("name", ["graft_small", "graft_d50_sharp", "graft_hub_clamp"])
def test_graft_layer_matches_oracle(name):
    """fp64_ref.graft_layer, chained over every layer from the oracle's own layer-0 inputs (h, the attention W_tilde and
    E, the seed prior, query_node_emb), against oracle/graft_oracle.forward in fp32: each layer's PageRank prior and
    score softmax, so the query_emb handed from layer to layer is checked too."""
    from test_graftnet_host import load_model
    m, g = load_model(name)
    ref = GO.forward(m, g.batch)
    local_entity, _qe, kb, graft, q_input, kb_fact_rel, seed_dist = g.batch[:7]
    B, N = local_entity.shape
    D = m.entity_dim
    layer = m.reasoning
    with torch.no_grad():                              # graft_oracle.py:39-60, the layer-0 inputs
        le = torch.as_tensor(local_entity, dtype=torch.long)
        m.instruction.encode_question_train(torch.as_tensor(q_input, dtype=torch.long))
        qh, qnode, qmask = (m.instruction.query_hidden_emb, m.instruction.query_node_emb,
                            m.instruction.query_mask_train)
        rel = m.get_rel_feature_train()
        if m.encode_type:
            h = GO._type_layer(m.type_layer.kb_self_linear, kb, rel, B, N, m.norm_rel)
        else:
            h = m.entity_linear(m.entity_embedding(le))
        fact_emb = rel[torch.as_tensor(kb_fact_rel, dtype=torch.long)]
        div = float(np.sqrt(D))
        sim = torch.softmax(torch.bmm(qh, fact_emb.transpose(1, 2)) / div
                            + (1 - qmask.unsqueeze(2)) * GO.VERY_NEG_NUMBER, dim=1)
        W = torch.sum(torch.sum(sim.unsqueeze(3) * qh.unsqueeze(2), dim=1) * fact_emb, dim=2) / div
        W_tilde = torch.exp(W - torch.max(W, dim=1, keepdim=True)[0])
        (e2f_b, e2f_f, e2f_e, _v0), (f2e_b, f2e_e, f2e_f, _v1) = graft
        E = torch.zeros(B * N, dtype=F64).index_add_(
            0, torch.as_tensor(np.asarray(e2f_b) * N + np.asarray(e2f_e)),
            W_tilde.to(F64)[torch.as_tensor(e2f_b), torch.as_tensor(e2f_f)]).clamp(min=GO.VERY_SMALL_NUMBER)
        mask = (le != m.num_entity).to(F64)
        hh, d, q = h.reshape(B * N, D).to(F64), torch.as_tensor(seed_dist, dtype=F64), qnode.reshape(B, D).to(F64)
        sw, sb = layer.score_func.weight.detach().to(F64).view(-1), float(layer.score_func.bias)
        for i in range(m.num_layer):
            hh, s, d, q = R.graft_layer(hh, d, q, fact_emb.to(F64), W_tilde.to(F64), E, (e2f_b, e2f_f, e2f_e),
                                        (f2e_b, f2e_e, f2e_f), graft_lin(layer, i), sw, layer.pagerank_lambda,
                                        layer.fact_scale)
            pr = torch.as_tensor(ref["pagerank_history"][i], dtype=F64)
            assert (d - pr).abs().max() <= 1e-5 * pr.abs().max()
            dist = torch.softmax(s.view(B, N) + sb + (1 - mask) * GO.VERY_NEG_NUMBER, dim=1)
            want = torch.as_tensor(ref["dist_history"][i], dtype=F64)
            assert (dist - want).abs().max() <= 1e-4 * want.abs().max()
