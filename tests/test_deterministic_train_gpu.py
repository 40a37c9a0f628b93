"""Deterministic training backward under torch.use_deterministic_algorithms (csrc/aggregate_bwd.cu, csrc/graft.cu:
the *_det entry points and the fixed-window segmented sums of csrc/common.cuh).

* Against float64: the edge-shape tests of the atomic kernels (test_aggregate_backward_gpu, test_graftnet_train_gpu)
  run again with every wrapper forced to ``deterministic=True`` and the flag set; their per-element bounds count the
  terms summed into an element, which does not depend on the order.  No atomic entry point may run meanwhile.
* Repeat bit-identity on hub-heavy inputs, and the documented order restated in float32 numpy for the TypeLayer's
  grad_table, GraftNet's grad_self and the aggregation's dp: equal bit for bit, so the order is the data's.
* Which path runs, the flag captured at forward, nothing of shape [facts, D] saved, and the training goldens.
* Model level in child processes (CUBLAS_WORKSPACE_CONFIG must be set before cuBLAS starts): three Adam steps give
  bit-identical losses and state_dicts run to run and process to process."""
import functools
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from gnn_rag_b200 import autograd_path, batching, ops, synthetic as S

import test_aggregate_backward_gpu as AB
import test_graftnet_gpu as GG
import test_graftnet_train_gpu as GT
import test_training_path as TP

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ATOMIC = ("gr_aggregate_backward", "gr_type_layer_backward", "gr_graft_aggregate_backward",
          "gr_graft_attention_backward")
DET = tuple(n + "_det" for n in ATOMIC)
WRAPPERS = ("aggregate_backward", "type_layer_backward", "graft_aggregate_backward", "graft_attention_backward")
ROW_WIN, REL_WIN = 32, 64     # kRowWin, kRelWin / kFactWin of the kernels: part of the documented order


class _Spy:
    """Stands in for ops._L(): records the C entry points the wrappers call."""

    def __init__(self, real, calls):
        self._real, self._calls = real, calls

    def __getattr__(self, name):
        self._calls.append(name)
        return getattr(self._real, name)


@pytest.fixture
def calls(monkeypatch):
    """Entry points called through ops (list of names)."""
    seen = []
    real = ops._L
    monkeypatch.setattr(ops, "_L", lambda: _Spy(real(), seen))
    return seen


@pytest.fixture
def flag():
    """Restores torch's deterministic-algorithms setting after the test."""
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    yield
    torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])


@pytest.fixture
def det(monkeypatch, calls, flag):
    """The flag on (warn_only) and every backward wrapper forced to its deterministic kernels; afterwards, no atomic
    backward entry point may have run."""
    torch.use_deterministic_algorithms(True, warn_only=True)
    for name in WRAPPERS:
        monkeypatch.setattr(ops, name, functools.partial(getattr(ops, name), deterministic=True))
    yield calls
    assert not [n for n in calls if n in ATOMIC]


def _params(fn, argnames):
    """The parameter values ``fn`` is parametrized with for ``argnames``."""
    return [m.args[1] for m in getattr(fn, "pytestmark", []) if m.name == "parametrize" and m.args[0] == argnames][0]


# ---- against float64 ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("D,I,direction,weights", AB.CASES)
def test_aggregate_backward_vs_fp64(det, D, I, direction, weights):
    AB.test_backward_vs_fp64_autograd(D, I, direction, weights)
    assert "gr_aggregate_backward_det" in det


SHAPES = "kind,B,N,E,D,I,direction,weights"


@pytest.mark.parametrize(SHAPES, _params(AB.test_backward_graph_shapes, SHAPES))
def test_aggregate_backward_graph_shapes(det, kind, B, N, E, D, I, direction, weights):
    AB.test_backward_graph_shapes(kind, B, N, E, D, I, direction, weights)


def test_aggregate_backward_prefilled_and_f0(det):
    AB.test_backward_accumulates_into_buffers_and_f0_is_a_no_op()


def test_aggregate_backward_self_loop_relation_spans_many_windows(det):
    """One relation holding a self-loop fact for every real node (the self-loop relation at full Nt), spread over
    many windows of the dP pass, plus a source hub and a destination hub; relations 1 .. R1-2 stay empty."""
    rs = np.random.RandomState(3)
    B, N, D, I, R1 = 2, 700, 40, 2, 9
    Nt = B * N
    hub = 5
    h = np.concatenate([np.arange(Nt), np.full(900, hub), rs.randint(0, N, 900)])
    t = np.concatenate([np.arange(Nt), rs.randint(0, N, 900), np.full(900, hub + 1)])
    r = np.concatenate([np.full(Nt, R1 - 1), np.zeros(1800, dtype=np.int64)])
    case = AB._Case(0, D, I, "fwd", True, B=B, N=N, R1=R1)
    case.heads, case.rels, case.tails = h.astype(np.int64), r.astype(np.int64), t.astype(np.int64)
    case.F = len(h)
    d = lambda a: torch.from_numpy(a).to(dev)   # noqa: E731
    case.g = ops.csr_build(d(case.heads), d(case.rels), d(case.tails), B, N, R1)
    w = rs.uniform(0.1, 1.7, size=case.F).astype(np.float32)
    case.w = d(w)
    case.w_csr = ops.gather_f32(case.w, case.g.fact_t)
    case.G = d(rs.randn(Nt, I * D).astype(np.float32))
    AB._check(case, case.run())
    assert int(np.bincount(case.rels)[R1 - 1]) > 20 * REL_WIN


@pytest.mark.parametrize("D", _params(GT.test_aggregate_forward_and_backward_match_fp64, "D"))
def test_graft_aggregate_vs_fp64(det, D):
    GT.test_aggregate_forward_and_backward_match_fp64(D)
    assert "gr_graft_aggregate_backward_det" in det


@pytest.mark.parametrize("D", _params(GT.test_aggregate_with_dropout_matches_fp64_with_the_same_mask, "D"))
def test_graft_aggregate_with_dropout_vs_fp64(det, D):
    GT.test_aggregate_with_dropout_matches_fp64_with_the_same_mask(D)


@pytest.mark.parametrize("D", _params(GT.test_aggregate_with_no_staged_facts, "D"))
def test_graft_aggregate_without_staged_facts(det, D):
    GT.test_aggregate_with_no_staged_facts(D)


@pytest.mark.parametrize("D,Q", _params(GT.test_attention_backward_matches_fp64, "D,Q"))
def test_graft_attention_vs_fp64(det, D, Q):
    """Includes Q = 1, masked tokens and Q * D = 40 * 512 (too large for the atomic kernel's shared-memory path)."""
    GT.test_attention_backward_matches_fp64(D, Q)
    assert "gr_graft_attention_backward_det" in det


@pytest.mark.parametrize("D", _params(GT.test_type_layer_backward_matches_fp64, "D"))
@pytest.mark.parametrize("weighted", [False, True])
def test_type_layer_vs_fp64(det, D, weighted):
    GT.test_type_layer_backward_matches_fp64(D, weighted)
    assert "gr_type_layer_backward_det" in det


def test_type_layer_through_autograd_vs_fp64(det):
    GT.test_type_layer_through_autograd_matches_fp64()
    assert "gr_type_layer_backward_det" in det


# ---- repeat bit-identity --------------------------------------------------------------------------------------------

def _bits(ts):
    torch.cuda.synchronize()
    return [t.detach().contiguous().view(torch.int32).cpu().clone() for t in ts]


def _same_five_times(fn):
    first = _bits(fn())
    for _ in range(4):
        assert all(torch.equal(a, b) for a, b in zip(first, _bits(fn())))


@pytest.mark.parametrize("direction", ["fwd", "inv"])
def test_repeat_bit_identity_aggregate(direction):
    case = AB._Case(11, 200, 2, direction, True, kind="hub", B=2, N=300, E=400)

    def run():
        out = (torch.zeros(case.R1, case.D, device=dev), torch.zeros(case.B, case.I, case.D, device=dev),
               torch.zeros(case.B, case.N, device=dev))
        ops.aggregate_backward(case.g, direction, case.prior, case.table, case.ins, case.G, *out, w=case.w_csr,
                               deterministic=True)
        return out
    _same_five_times(run)


def _type_layer_case(D, seed=0, B=3, N=50, R1=13):
    rs = np.random.RandomState(seed)
    b = S.make_batch(seed, B=B, N=N, E=400, num_entity=500, num_relation=R1 - 1, num_word=20, powerlaw=True,
                     n_real="ragged", with_weights=True)
    g = batching.stage_batch(b, dev, R1, False, True).graph
    G_ = torch.tensor(rs.randn(B * N, D), dtype=torch.float32, device=dev)
    out = torch.tensor(rs.randn(B * N, D), dtype=torch.float32, device=dev)
    out[torch.as_tensor(rs.rand(B * N, D) < 0.2, device=dev)] = 0.0
    pre = torch.tensor(rs.randn(R1, D), dtype=torch.float32, device=dev)
    return g, G_, out, pre


def test_repeat_bit_identity_type_layer():
    g, G_, out, pre = _type_layer_case(200)

    def run():
        gt = pre.clone()
        ops.type_layer_backward(g, G_, out, gt, g.wr_t, g.wr_h, deterministic=True)
        return [gt]
    _same_five_times(run)


def _graft_case(D, p, seed=4):
    rs = np.random.RandomState(seed)
    B, N, R1, maxF = 3, 40, 9, 3600
    gg, kfr, st = GT._graft(B, N, maxF, R1, rs, [3400, 0, 70], head_hub=2500, tail_hub=2500)
    Nt, F_ = B * N, st["heads"].numel()
    t = lambda a: torch.tensor(a, dtype=torch.float32, device=dev)  # noqa: E731
    s = t(rs.rand(F_))
    s[torch.as_tensor(rs.rand(F_) < 0.3, device=dev)] = 0.0
    return dict(gg=gg, kfr=kfr, st=st, s=s, self_tab=t(rs.randn(R1, D)), head_tab=t(rs.randn(Nt, D)),
                G=t(rs.randn(Nt, D)), seed=torch.tensor([77], dtype=torch.int64, device=dev), p=p, R1=R1, D=D)


def test_repeat_bit_identity_graft_aggregate():
    c = _graft_case(200, 0.2)

    def run():
        gs, gself, ghead = (torch.zeros(c["s"].numel(), device=dev), torch.zeros(c["R1"], 200, device=dev),
                            torch.zeros_like(c["head_tab"]))
        ops.graft_aggregate_backward(c["gg"], c["s"], c["self_tab"], c["head_tab"], c["G"], gs, gself, ghead,
                                     c["seed"], c["p"], deterministic=True)
        return gs, gself, ghead
    _same_five_times(run)


def test_repeat_bit_identity_graft_attention():
    c = _graft_case(64, 0.0)
    rs = np.random.RandomState(5)
    B, Q, D = 3, 7, 64
    qh = torch.tensor(rs.randn(B, Q, D), dtype=torch.float32, device=dev)
    qmask = torch.tensor((rs.rand(B, Q) < 0.7).astype(np.float32), device=dev)
    qmask[:, 0] = 1
    rel = torch.tensor(rs.randn(c["R1"], D), dtype=torch.float32, device=dev)
    gW = torch.tensor(rs.randn(B * c["gg"].max_fact), dtype=torch.float32, device=dev)

    def run():
        gq, gr = torch.zeros(B, Q, D, device=dev), torch.zeros(c["R1"], D, device=dev)
        ops.graft_attention_backward(c["gg"], qh, qmask, rel, gW, gq, gr, deterministic=True)
        return gq, gr
    _same_five_times(run)


# ---- the order itself, restated in float32 --------------------------------------------------------------------------

def _segwin(segs, terms, W, out):
    """The fixed-window segmented sum of csrc/common.cuh in float32 numpy: ``segs`` (segment per list entry, sorted),
    ``terms`` (float32 row per entry), windows of W entries, ``out`` [segments, D] float32, added into in place."""
    L = len(segs)
    part = {}
    for a in range(0, L, W):
        b = min(L, a + W)
        i, first = a, True
        while i < b:
            s = segs[i]
            acc = np.zeros(out.shape[1], dtype=np.float32)
            while i < b and segs[i] == s:
                acc = acc + terms[i]
                i += 1
            before = first and a > 0 and segs[a - 1] == s
            after = b < L and segs[b] == s
            if before or after:
                part[(a // W, 0 if first else 1)] = acc
            else:
                out[s] = out[s] + acc
            first = False
    for s in np.unique(segs):
        idx = np.nonzero(segs == s)[0]
        beg, end = int(idx[0]), int(idx[-1]) + 1
        ws, we = beg // W, (end - 1) // W
        if ws != we:
            v = part[(ws, 0 if beg == ws * W else 1)]
            for w in range(ws + 1, we + 1):
                v = v + part[(w, 0)]
            out[s] = out[s] + v


def _rows(rowptr):
    return np.repeat(np.arange(len(rowptr) - 1), np.diff(rowptr))


def test_order_type_layer_grad_table_bit_exact():
    """grad_table[r] = (pre + tail-CSR sum) + head-CSR sum, each over the relation's slots in slot order, windows of
    64 entries: a 13-relation power-law batch puts several relations across window edges."""
    g, G_, out, pre = _type_layer_case(50, seed=1)
    gt = pre.clone()
    ops.type_layer_backward(g, G_, out, gt, g.wr_t, g.wr_h, deterministic=True)
    Gm = np.where(out.cpu().numpy() > 0, G_.cpu().numpy(), np.float32(0))
    want = pre.cpu().numpy().copy()
    F = g.F
    for rp, rel, w in ((g.rowptr_t, g.rel_t, g.wr_t), (g.rowptr_h, g.rel_h, g.wr_h)):
        rel, w = rel[:F].cpu().numpy(), w[:F].cpu().numpy()
        rows = _rows(rp[: g.B * g.N + 1].cpu().numpy())
        order = np.lexsort((np.arange(F), rel))
        _segwin(rel[order], [w[e] * Gm[rows[e]] for e in order], REL_WIN, want)
    assert np.bincount(g.rel_t[:F].cpu().numpy()).max() > REL_WIN
    np.testing.assert_array_equal(gt.cpu().numpy().view(np.int32), want.view(np.int32))


def test_order_graft_grad_self_bit_exact():
    """grad_self[r] += sum over the staged facts of r in slot order of g_f s_f [a_f > 0], with dropout p = 0.2."""
    c = _graft_case(40, 0.2, seed=6)
    st, D, R1 = c["st"], c["D"], c["R1"]
    pre = np.random.RandomState(2).randn(R1, D).astype(np.float32)
    gself = torch.tensor(pre, device=dev)
    ops.graft_aggregate_backward(c["gg"], c["s"], c["self_tab"], c["head_tab"], c["G"],
                                 torch.zeros(c["s"].numel(), device=dev), gself, torch.zeros_like(c["head_tab"]),
                                 c["seed"], c["p"], deterministic=True)
    mask = ops.graft_dropout_mask(c["seed"], c["p"], c["gg"].B * c["gg"].max_fact, D).cpu().numpy().astype(bool)
    scale = np.float32(1.0 / (1.0 - c["p"]))
    s, st_, ht, G_ = (c[k].cpu().numpy() for k in ("s", "self_tab", "head_tab", "G"))
    rels, heads, tails, slots = (st[k].numpy() for k in ("rels", "heads", "tails", "slot_of"))
    order = np.lexsort((np.arange(len(rels)), rels))
    terms = []
    for f in order:
        a = st_[rels[f]] + ht[heads[f]]
        g = np.where(mask[slots[f]], G_[tails[f]] * scale, np.float32(0))
        terms.append(np.where((a > 0) & (s[f] != 0), g * s[f], np.float32(0)).astype(np.float32))
    want = pre.copy()
    _segwin(rels[order], terms, REL_WIN, want)
    assert np.bincount(rels).max() > 5 * REL_WIN
    np.testing.assert_array_equal(gself.cpu().numpy().view(np.int32), want.view(np.int32))


@pytest.mark.parametrize("direction", ["fwd", "inv"])
def test_order_aggregate_dp_bit_exact(direction):
    """q_e = w_e^2 * dot_e (dot_e: each lane adds g * (P * x) over its columns c = lane + 32k, k then j, where
    P * x > 0; then a butterfly over the 32 lanes); dp[s] = pre + sum of q_e over the other CSR's row s in slot order."""
    case = AB._Case(21, 70, 2, direction, True, kind="hub", B=2, N=120, E=160)
    rs = np.random.RandomState(9)
    pre = rs.randn(case.B, case.N).astype(np.float32)
    gp = torch.tensor(pre, device=dev)
    ops.aggregate_backward(case.g, direction, case.prior, case.table, case.ins, case.G,
                           torch.zeros(case.R1, case.D, device=dev), torch.zeros(case.B, case.I, case.D, device=dev),
                           gp, w=case.w_csr, deterministic=True)
    g, F, D, I, N = case.g, case.F, case.D, case.I, case.N
    rp, src, rel, fact = (x.cpu().numpy() for x in ((g.rowptr_t, g.src_t, g.rel_t, g.fact_t) if direction == "fwd"
                                                    else (g.rowptr_h, g.src_h, g.rel_h, g.fact_h)))
    rp_o, fact_o = (x.cpu().numpy() for x in ((g.rowptr_h, g.fact_h) if direction == "fwd" else (g.rowptr_t, g.fact_t)))
    w, table, ins = case.w_csr.cpu().numpy(), case.table.cpu().numpy(), case.ins.cpu().numpy()
    G_ = case.G.cpu().numpy().reshape(-1, I, D)
    K = (D + 31) // 32
    cols = np.arange(32)[:, None] + 32 * np.arange(K)[None, :]                     # [lane, k]
    valid = cols < D
    cc = np.where(valid, cols, 0)
    q = np.zeros(F, dtype=np.float32)
    rows = _rows(rp[: case.Nt + 1])
    for e in range(F):
        n = rows[e]
        b = n // N
        pv = np.where(valid, table[rel[e]][cc], np.float32(0))
        lane = np.zeros(32, dtype=np.float32)
        for k in range(K):
            for j in range(I):
                x = np.where(valid[:, k], ins[b, j][cc[:, k]], np.float32(0))
                pre_ = pv[:, k] * x
                gv = np.where(valid[:, k], G_[n, j][cc[:, k]], np.float32(0))
                lane = np.where(pre_ > 0, lane + gv * pre_, lane)
        for o in (16, 8, 4, 2, 1):
            lane = lane + lane[np.arange(32) ^ o]
        q[fact[e]] = (w[e] * w[e]) * lane[0]
    want = pre.reshape(-1).copy()
    for s in range(case.Nt):
        if rp_o[s + 1] > rp_o[s]:
            v = np.float32(0)
            for e in range(rp_o[s], rp_o[s + 1]):
                v = np.float32(v + q[fact_o[e]])
            want[s] = np.float32(want[s] + v)
    np.testing.assert_array_equal(gp.cpu().numpy().reshape(-1).view(np.int32), want.view(np.int32))


# ---- which path runs ------------------------------------------------------------------------------------------------

def _graft_model(D, dropout=0.0):
    return GT._graft_model(D, dropout)


def _graft_batch():
    return S.make_graft_batch(3, B=3, N=40, E=150, num_entity=1000, num_relation=40, num_word=100)


def test_flag_off_runs_the_atomic_kernels(calls, flag):
    torch.use_deterministic_algorithms(False)
    m = _graft_model(64)
    m.train()
    m(_graft_batch(), training=True)[0].backward()
    assert set(ATOMIC[2:]) <= set(calls) and not set(DET) & set(calls)
    calls.clear()
    args = S.model_args("ReaRev", entity_dim=64, num_iter=1, num_ins=2, num_gnn=1, use_cuda=True)
    torch.manual_seed(0)
    import gnn_rag_b200 as G
    r = G.ReaRev(args, 1000, 40, 100).cuda().train()
    r(S.make_batch(1, B=2, N=40, E=120, num_entity=1000, num_relation=40, num_word=100), training=True)[0].backward()
    assert "gr_aggregate_backward" in calls and not set(DET) & set(calls)


def test_flag_on_runs_the_deterministic_kernels(calls, flag):
    torch.use_deterministic_algorithms(True, warn_only=True)
    m = _graft_model(64)
    m.train()
    m(_graft_batch(), training=True)[0].backward()
    assert set(DET[2:]) <= set(calls) and not set(ATOMIC) & set(calls)
    calls.clear()
    args = S.model_args("NSM", entity_dim=64, num_step=2, use_cuda=True)
    torch.manual_seed(0)
    import gnn_rag_b200 as G
    r = G.NSM(args, 1000, 40, 100).cuda().train()
    r(S.make_batch(1, B=2, N=40, E=120, num_entity=1000, num_relation=40, num_word=100), training=True)[0].backward()
    assert "gr_aggregate_backward_det" in calls and not set(ATOMIC) & set(calls)


def test_backward_follows_the_flag_captured_at_forward(calls, flag):
    m = _graft_model(64)
    m.train()
    b = _graft_batch()
    for fwd, names, other in ((True, DET[2:], ATOMIC), (False, ATOMIC[2:], DET)):
        calls.clear()
        torch.use_deterministic_algorithms(fwd, warn_only=True)
        loss = m(b, training=True)[0]
        torch.use_deterministic_algorithms(not fwd, warn_only=True)
        loss.backward()
        assert set(names) <= set(calls) and not set(other) & set(calls), (fwd, calls)


def test_no_per_fact_activation_is_saved_in_deterministic_mode(flag):
    torch.use_deterministic_algorithms(True, warn_only=True)
    GT.test_no_per_fact_activation_is_saved_for_backward()


# ---- goldens --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", TP.CASES)
def test_training_goldens_in_deterministic_mode(det, name):
    TP.test_training_on_gpu_through_the_aggregation_kernels(name)
    assert "gr_aggregate_backward_det" in det


@pytest.mark.parametrize("name", _params(GG.test_training_on_gpu_matches_reference_gradients, "name"))
def test_graftnet_golden_gradients_in_deterministic_mode(det, name):
    GG.test_training_on_gpu_matches_reference_gradients(name)
    assert "gr_graft_aggregate_backward_det" in det or "gr_graft_attention_backward_det" in det


# ---- model level, in child processes --------------------------------------------------------------------------------

CHILD = r'''
import hashlib, json, sys
import numpy as np
import torch
torch.use_deterministic_algorithms(True)
import gnn_rag_b200 as G
from gnn_rag_b200 import synthetic as S

def digest(ts):
    h = hashlib.sha256()
    for t in ts:
        h.update(t.detach().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()

CONFIGS = {
    "rearev_d50": ("ReaRev", dict(entity_dim=50, num_iter=2, num_ins=2, num_gnn=2)),
    "rearev_d200": ("ReaRev", dict(entity_dim=200, num_iter=2, num_ins=2, num_gnn=2)),
    "rearev_d264": ("ReaRev", dict(entity_dim=264, num_iter=1, num_ins=2, num_gnn=1)),
    "nsm_reason_kb": ("NSM", dict(entity_dim=64, num_step=3, reason_kb=True)),
    "graftnet_drop": ("GraftNet", dict(entity_dim=64, num_layer=3, linear_dropout=0.2)),
}

def batch_for(name, permute=False):
    if name == "GraftNet":
        b = S.make_graft_batch(5, B=6, N=120, E=600, num_entity=1000, num_relation=40, num_word=100, powerlaw=True,
                               n_real="ragged")
        if permute:
            (hb, hf, he, v0), (tb, te, tf, v1) = b[3]
            rs = np.random.RandomState(7)
            p, q = rs.permutation(len(hb)), rs.permutation(len(tb))
            b = list(b)
            b[3] = ((hb[p], hf[p], he[p], v0), (tb[q], te[q], tf[q], v1))
            b = tuple(b)
        return b
    return S.make_batch(5, B=6, N=120, E=600, num_entity=1000, num_relation=40, num_word=100, powerlaw=True,
                        n_real="ragged", with_weights=True)

def train(key, permute=False):
    name, over = CONFIGS[key]
    kw = dict(use_cuda=True, lm_dropout=0.0)
    kw.setdefault("linear_dropout", 0.0)
    kw.update(over)
    args = S.model_args(name, **kw)
    torch.manual_seed(0)
    np.random.seed(0)
    m = getattr(G, name)(args, 1000, 40, 100).cuda().train()
    b = batch_for(name, permute)
    opt = torch.optim.Adam([p for p in m.parameters() if p.requires_grad], lr=1e-3)
    losses = []
    for _ in range(3):
        opt.zero_grad()
        loss = m(b, training=True)[0]
        loss.backward()
        torch.nn.utils.clip_grad_norm_([p for p in m.parameters() if p.requires_grad], 1.0)
        opt.step()
        losses.append(loss.detach().reshape(1))
    return digest(losses + list(m.state_dict().values())), m, b

out = {}
for key in CONFIGS:
    d1, m, b = train(key)
    d2, _, _ = train(key)
    out[key] = [d1, d2]
    if key == "graftnet_drop":
        out["graftnet_permuted"] = train(key, permute=True)[0]
    m.eval()
    with torch.no_grad():
        on = m(b)[2].clone()
        torch.use_deterministic_algorithms(False)
        off = m(b)[2].clone()
        torch.use_deterministic_algorithms(True)
    out[key + "_inference_equal"] = bool(torch.equal(on.view(torch.int32), off.view(torch.int32)))
print("RESULT " + json.dumps(out))
'''


def _child():
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", CHILD]
    res = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stderr[-4000:]
    line = [ln for ln in res.stdout.splitlines() if ln.startswith("RESULT ")][-1]
    return json.loads(line[len("RESULT "):])


def test_three_adam_steps_are_bit_identical_across_runs_and_processes():
    """ReaRev at D = 50 / 200 (I = 2), ReaRev at D = 264 (the torch fallback), NSM with reason_kb, GraftNet with
    linear_dropout 0.2: three steps of forward, backward, clip_grad_norm_ and Adam, twice in one child and once more in
    a second child; losses and state_dicts bit-identical.  GraftNet with its graft lists permuted as the loader
    permutes them gives the same bits, and inference under the flag equals inference without it."""
    a, b = _child(), _child()
    keys = [k for k in a if isinstance(a[k], list)]
    assert len(keys) == 5
    for k in keys:
        assert a[k][0] == a[k][1] == b[k][0] == b[k][1], k
    assert a["graftnet_permuted"] == a["graftnet_drop"][0] == b["graftnet_permuted"]
    assert all(a[k] for k in a if k.endswith("_inference_equal"))
    assert hashlib.sha256(b"").hexdigest() not in a.values()
