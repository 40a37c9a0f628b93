"""CPU: fact dropout on a resident split (loader.DeviceSplit with shuffle=True, csrc/split.cu) -- header and binding
agreement for gr_split_fact_order and the ordered assembly entry points, their refusals and shape rules, the refusals
DeviceSplit makes before it touches a device, and the host's kept-count helper against the reference's expression.
Every entry-point call below is refused before any CUDA call, so the pointers are placeholders that are never
dereferenced."""
import ctypes

import numpy as np
import pytest
import torch

from gnn_rag_b200 import _lib, loader, ops
from test_device_split_host import SplitLoader

PTR = 0x1000
INVALID, WORKSPACE = -1, -3
INT_MAX = 2 ** 31 - 1
I64, I32, VP = ctypes.c_int64, ctypes.c_int, ctypes.c_void_p

EXPECTED = {
    "gr_split_fact_order_workspace_bytes": [I64],
    "gr_split_fact_order": [VP, I64, VP, VP, I32, VP, I32, I64, I64, VP, VP, VP, ctypes.c_size_t, VP],
    "gr_split_assemble_ordered": [VP] * 5 + [I64, VP, VP, VP, I64, I32, I64, I64, I32, I32, I64] + [VP] * 7,
    "gr_split_assemble_graft_ordered": [VP] * 7 + [I64, VP, VP, VP, I64, I32, I64, I64, I32, I64] + [VP] * 11,
}


@pytest.mark.parametrize("name", sorted(EXPECTED))
def test_header_prototypes_bind(name):
    res, args = _lib.SIGNATURES[name]
    assert args == EXPECTED[name]
    assert res == (ctypes.c_size_t if name.endswith("_bytes") else ctypes.c_int)
    assert getattr(_lib.load(), name).argtypes == EXPECTED[name]


# ---- entry-point refusals (before any CUDA call) -----------------------------------------------------------------------

def _call(name, a, over):
    a.update(over)
    lib = _lib.load()
    return getattr(lib, name)(*a.values()), lib.gr_last_error().decode()


def _order(**over):
    a = dict(off=PTR, num_q=3, ids=PTR, kept=PTR, B=2, seed=PTR, perm=0, n_total=20, K=10, order=PTR, status=PTR,
             workspace=PTR, workspace_bytes=1 << 20, stream=None)
    return _call("gr_split_fact_order", a, over)


@pytest.mark.parametrize("over,rc,msg", [
    (dict(off=None), INVALID, "invalid argument: null pointer"),
    (dict(kept=None), INVALID, "invalid argument: null pointer"),
    (dict(seed=None), INVALID, "invalid argument: null pointer"),
    (dict(status=None), INVALID, "invalid argument: null pointer"),
    (dict(B=0), INVALID, "invalid argument: need num_q >= 0, B > 0, n_total >= 0 and K >= 0"),
    (dict(num_q=-1), INVALID, "invalid argument: need num_q >= 0, B > 0, n_total >= 0 and K >= 0"),
    (dict(n_total=-1), INVALID, "invalid argument: need num_q >= 0, B > 0, n_total >= 0 and K >= 0"),
    (dict(K=-1), INVALID, "invalid argument: need num_q >= 0, B > 0, n_total >= 0 and K >= 0"),
    (dict(K=2 ** 31), INVALID, "invalid argument: K must fit int32"),
    (dict(perm=2), INVALID, "invalid argument: perm must be 0 (kb facts) or 1 (graft lists)"),
    (dict(order=None), INVALID, "invalid argument: null order"),
    (dict(workspace=None), WORKSPACE, "workspace too small"),
    (dict(workspace_bytes=16), WORKSPACE, "workspace too small"),
])
def test_split_fact_order_refusals(over, rc, msg):
    got_rc, got_msg = _order(**over)
    assert got_rc == rc and got_msg.startswith("gr_split_fact_order: " + msg), got_msg


def test_split_fact_order_workspace_holds_a_key_and_an_index_per_fact():
    ws = _lib.load().gr_split_fact_order_workspace_bytes
    assert ws(-1) == 0 and ws(0) > 0
    assert ws(10 ** 6) >= 12 * 10 ** 6 and ws(10 ** 6) > ws(10 ** 3)


def _ordered(**over):
    a = dict(q_off=PTR, q_heads=PTR, q_rels=PTR, q_tails=PTR, q_ents=PTR, num_q=3, ids=PTR, kept=PTR, order=PTR, K=6,
             B=2, N=5, self_rel=4, use_self_loop=1, idx_bytes=4, F=10, heads=PTR, rels=PTR, tails=PTR,
             batch_ids=PTR, fact_ids=PTR, status=PTR, stream=None)
    return _call("gr_split_assemble_ordered", a, over)


@pytest.mark.parametrize("over,msg", [
    (dict(q_off=None), "null pointer"),
    (dict(kept=None), "null pointer"),
    (dict(status=None), "null pointer"),
    (dict(B=0), "need num_q >= 0, B > 0, N > 0, F >= 0 and K >= 0"),
    (dict(N=0), "need num_q >= 0, B > 0, N > 0, F >= 0 and K >= 0"),
    (dict(F=-1), "need num_q >= 0, B > 0, N > 0, F >= 0 and K >= 0"),
    (dict(K=-1), "need num_q >= 0, B > 0, N > 0, F >= 0 and K >= 0"),
    (dict(idx_bytes=2), "idx_bytes must be 4 or 8"),
    (dict(B=2, N=2 ** 30), "the batch overflows int32 indices"),
    (dict(F=2 ** 31), "the batch overflows int32 indices"),
    (dict(self_rel=-1), "self_rel must be non-negative"),
    (dict(fact_ids=None), "null output arrays"),
    (dict(order=None), "null order"),
    (dict(q_tails=None), "null resident arrays"),
])
def test_split_assemble_ordered_refusals(over, msg):
    assert _ordered(**over) == (INVALID, "gr_split_assemble_ordered: invalid argument: " + msg)


def _graft_ordered(**over):
    a = dict(g_off=PTR, g_e2f_f=PTR, g_e2f_e=PTR, g_f2e_e=PTR, g_f2e_f=PTR, r_off=PTR, r_vals=PTR, num_q=3, ids=PTR,
             kept=PTR, order=PTR, K=10, B=2, max_facts=7, rel_pad=9, idx_bytes=4, G=10, e2f_b=PTR, e2f_f=PTR,
             e2f_e=PTR, e2f_v=PTR, f2e_b=PTR, f2e_e=PTR, f2e_f=PTR, f2e_v=PTR, kb_fact_rel=PTR, status=PTR,
             stream=None)
    return _call("gr_split_assemble_graft_ordered", a, over)


@pytest.mark.parametrize("over,msg", [
    (dict(g_off=None), "null pointer"),
    (dict(kept=None), "null pointer"),
    (dict(g_f2e_f=None), "null resident arrays"),
    (dict(B=0), "need num_q >= 0, B > 0, max_facts >= 0, G >= 0 and K >= 0"),
    (dict(K=-1), "need num_q >= 0, B > 0, max_facts >= 0, G >= 0 and K >= 0"),
    (dict(G=-1), "need num_q >= 0, B > 0, max_facts >= 0, G >= 0 and K >= 0"),
    (dict(idx_bytes=1), "idx_bytes must be 4 or 8"),
    (dict(G=2 ** 31), "the batch overflows int32 indices"),
    (dict(e2f_b=None), "null output arrays"),
    (dict(order=None), "null order"),
    (dict(kb_fact_rel=None), "null kb_fact_rel"),
])
def test_split_assemble_graft_ordered_refusals(over, msg):
    assert _graft_ordered(**over) == (INVALID, "gr_split_assemble_graft_ordered: invalid argument: " + msg)


def test_empty_orders_need_no_pointer():
    """K = 0 (every question drops all its facts): a null order passes the argument checks."""
    assert _order(K=0, order=None, workspace=None)[1].startswith("gr_split_fact_order: workspace too small")
    assert _ordered(K=0, order=None, tails=None)[1].endswith("null output arrays")
    assert _graft_ordered(K=0, order=None, f2e_v=None)[1].endswith("null output arrays")


# ---- shape rules agree with the entry points ---------------------------------------------------------------------------

@pytest.mark.parametrize("B,n_total,K", [(1, 0, 0), (3, 10 ** 9, INT_MAX), (3, 5, INT_MAX + 1), (0, 5, 1),
                                         (2, -1, 1), (2, 5, -1)])
def test_split_fact_order_ok_matches_the_entry_point(B, n_total, K):
    _rc, msg = _order(B=B, n_total=n_total, K=K, workspace=None)
    assert ops.split_fact_order_ok(B, n_total, K) == msg.startswith("gr_split_fact_order: workspace too small"), msg


@pytest.mark.parametrize("B,N,F,dt", [(1, 1, 1, torch.int32), (2, 2 ** 30 - 1, 5, torch.int32),
                                      (2, 2 ** 30, 5, torch.int32), (2, 2 ** 30, 5, torch.int64),
                                      (1, 5, INT_MAX, torch.int32), (1, 5, INT_MAX + 1, torch.int32),
                                      (0, 5, 1, torch.int64), (3, 0, 1, torch.int64), (3, 5, -1, torch.int64)])
def test_split_assemble_ordered_follows_split_assemble_ok(B, N, F, dt):
    _rc, msg = _ordered(B=B, N=N, F=F, idx_bytes=4 if dt == torch.int32 else 8, tails=None)
    assert ops.split_assemble_ok(B, N, F, dt) == msg.endswith("null output arrays"), msg


@pytest.mark.parametrize("B,M,G,dt", [(1, 0, 5, torch.int32), (2, 7, INT_MAX, torch.int32),
                                      (2, 7, INT_MAX + 1, torch.int32), (2, 7, INT_MAX + 1, torch.int64),
                                      (0, 7, 1, torch.int64), (2, -1, 1, torch.int64)])
def test_split_assemble_graft_ordered_follows_split_assemble_graft_ok(B, M, G, dt):
    _rc, msg = _graft_ordered(B=B, max_facts=M, G=G, idx_bytes=4 if dt == torch.int32 else 8, f2e_v=None)
    assert ops.split_assemble_graft_ok(B, M, G, dt) == msg.endswith("null output arrays"), msg


# ---- DeviceSplit refusals before the device ----------------------------------------------------------------------------

def _bare(shuffle, stored=None, ents=None, N=8):
    """A DeviceSplit with the host-side state get_batch reads before its first device call, and no device state."""
    L = SplitLoader(seed=1, num_questions=4, max_local_entity=N)
    s = object.__new__(loader.DeviceSplit)
    s.loader, s._res, s.device, s.shuffle, s.graft = L, {}, torch.device("cuda"), shuffle, False
    s.N, s.index_dtype, s.num_q = N, torch.int32, 4
    s._stored = np.array(stored if stored is not None else [len(m[0]) for m in L.kb_adj_mats], dtype=np.int64)
    s._ents = np.array(ents if ents is not None else [0] * 4, dtype=np.int64)
    s._count = s._stored + s._ents
    return s


@pytest.mark.parametrize("p", [-0.1, -1e-12, 1.0000001, 2.0, float("nan")])
def test_shuffle_refuses_a_dropout_outside_0_1(p):
    with pytest.raises(ValueError, match=r"fact_dropout must be in \[0, 1\]"):
        _bare(True).get_batch(0, 2, p)


def test_stored_order_keeps_its_refusal():
    with pytest.raises(ValueError, match=r"fact_dropout must be 0 \(facts come in stored order\), got 0.1"):
        _bare(False).get_batch(0, 2, 0.1)


def test_shuffle_refuses_data_eff_and_other_q_types():
    L = SplitLoader(seed=1, num_questions=4, max_local_entity=8)
    L.data_eff = True
    with pytest.raises(ValueError, match="data_eff"):
        loader.DeviceSplit(L, "cuda", shuffle=True)
    with pytest.raises(ValueError, match="q_type must be 'seq'"):
        _bare(True).get_batch(0, 2, 0.5, q_type="bert")


def test_int32_overflow_is_judged_on_the_kept_facts():
    s = _bare(True, stored=[2 ** 31, 2 ** 31, 1, 1])
    with pytest.raises(ValueError, match=r"overflows int32 indices \(B\*N = 16, 2147483648 facts\)"):
        s.get_batch(0, 2, 0.5)                 # 2^30 + 2^30 kept facts: one past INT_MAX


# ---- the kept count --------------------------------------------------------------------------------------------------

def test_kept_counts_equal_the_reference_expression():
    ns = list(range(0, 60)) + [99, 100, 101, 999, 1000, 6000, 7001, 50000, 2 ** 31 - 1, 2 ** 40 + 3]
    ps = [0.0, 0.1, 0.2, 0.25, 0.3, 1 / 3, 0.5, 0.7, 0.9, 0.95, 0.99, 1 - 1e-12, 1.0, 1e-12]
    ps += list(np.linspace(0, 1, 101))
    for p in ps:
        got = loader.kept_counts(np.array(ns, dtype=np.int64), p)
        assert got.dtype == np.int64
        assert got.tolist() == [int(np.floor(n * (1 - p))) for n in ns], p
    assert loader.kept_counts([10], 0.9).tolist() == [0]          # 10 * 0.09999999999999998 = 0.9999999999999998
    assert loader.kept_counts([10], 0.7).tolist() == [3]          # 10 * 0.30000000000000004
    assert loader.kept_counts([10], np.float64(0.7)).tolist() == [3]
