"""Exact restatements of the index kernels that build every batch, independent of every kernel and of the package:
gr_csr_build (csrc/csr_build.cu: both destination CSRs), the relation index the deterministic backward kernels sum in
(ops._relation_index / ops.csr_relation_index with gr_csr_row_of), gr_fact_weights (csrc/split.cu: the
normalized_gnn weights, gnn/dataset_load.py:507-517) and gr_graft_stage (csrc/graft.cu: GraftNet's two fact lists
paired by slot, gnn/dataset_load_graft.py:70-102 and base_gnn.py:56-75).

Everything here is integer work in numpy on the CPU, except the weights, which are 1 / count in float64 rounded once
to fp32.  tests/test_index_edges_gpu.py holds the kernels to these bit for bit; tests/test_index_edges_host.py pins
them to scipy.sparse, to the loader oracle and to the graft oracle's sparse matrices."""
import numpy as np

INT32_MAX = 2 ** 31 - 1
_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def pad4(n):
    return (n + 3) & ~3


def live_count(F, live):
    """The facts a kernel reads from an F-slot buffer: all of them, or clamp(live, 0, F)."""
    return F if live is None else min(max(int(live), 0), F)


# ---- gr_csr_build ------------------------------------------------------------------------------------------------------

def csr(heads, rels, tails, Nt, R1, live=None):
    """Both CSRs of the first ``live`` facts of (heads, rels, tails), as gr_csr_build documents them.

    -> dict with ``status`` (1 when a counted fact has a head or tail outside [0, Nt) or a relation outside [0, R1),
    else 0), ``live`` and, per direction d in 't' (rows = tails, src = heads) and 'h' (rows = heads, src = tails):
    ``rowptr_d`` [Nt + 1]; ``fact_d`` [live], the fact ids of each row in original fact order (a stable sort by the
    row); ``src_d`` / ``rel_d`` [pad4(F)], the clamped source and relation of each slot, with the pad slots
    [live, pad4(F)) zero.  Out-of-range ids are clamped into [0, Nt) and [0, R1).  Slots [live, F) of the kernel's
    fact array are unspecified and have no counterpart here."""
    heads, rels, tails = (np.asarray(a, dtype=np.int64).reshape(-1) for a in (heads, rels, tails))
    F = len(heads)
    L = live_count(F, live)
    h, r, t = heads[:L], rels[:L], tails[:L]
    bad = (h < 0) | (h >= Nt) | (t < 0) | (t >= Nt) | (r < 0) | (r >= R1)
    h, t, r = np.clip(h, 0, Nt - 1), np.clip(t, 0, Nt - 1), np.clip(r, 0, R1 - 1)
    out = dict(status=int(bad.any()), live=L)
    for d, key, other in (("t", t, h), ("h", h, t)):
        order = np.argsort(key, kind="stable")
        rowptr = np.zeros(Nt + 1, dtype=np.int64)
        rowptr[1:] = np.cumsum(np.bincount(key, minlength=Nt))
        src = np.zeros(pad4(F), dtype=np.int64)
        rel = np.zeros(pad4(F), dtype=np.int64)
        src[:L], rel[:L] = other[order], r[order]
        out.update({"rowptr_" + d: rowptr, "fact_" + d: order, "src_" + d: src, "rel_" + d: rel})
    return out


def relation_index(rel, R1, live=None):
    """(rix_ptr [R1 + 1], rix_slot [live]): the first ``live`` list positions grouped by relation, in increasing
    position inside each relation.  ``rel``: a relation in [0, R1) per position (a CSR's ``rel`` array)."""
    rel = np.asarray(rel, dtype=np.int64).reshape(-1)
    rel = rel[: live_count(len(rel), live)]
    ptr = np.zeros(R1 + 1, dtype=np.int64)
    ptr[1:] = np.cumsum(np.bincount(rel, minlength=R1))
    return ptr, np.argsort(rel, kind="stable")


def row_of(rowptr):
    """The row of every slot [0, rowptr[-1]) of a CSR (gr_csr_row_of)."""
    rowptr = np.asarray(rowptr, dtype=np.int64)
    return np.repeat(np.arange(len(rowptr) - 1), np.diff(rowptr))


# ---- gr_fact_weights ---------------------------------------------------------------------------------------------------

def fact_weights(heads, rels, Nt):
    """(weight fp32 [F], weight_rel fp32 [F], status): fp32(1.0 / outdeg(head)) and fp32(1.0 / count(head, rel)),
    each 1 / count in float64 rounded once.  A fact with a head outside [0, Nt) or a relation outside [0, 2^31 - 1] is
    refused: it counts nowhere, its weights are 0 and the status is 1."""
    h, r = np.asarray(heads, dtype=np.int64).reshape(-1), np.asarray(rels, dtype=np.int64).reshape(-1)
    ok = (h >= 0) & (h < Nt) & (r >= 0) & (r <= INT32_MAX)
    w = np.zeros(len(h), dtype=np.float32)
    wr = np.zeros(len(h), dtype=np.float32)
    hk, rk = h[ok], r[ok]
    deg = np.bincount(hk, minlength=int(Nt)) if len(hk) else np.zeros(1, dtype=np.int64)
    _, inv, cnt = np.unique((hk << 32) | rk, return_inverse=True, return_counts=True)
    w[ok] = (1.0 / deg[hk].astype(np.float64)).astype(np.float32)
    wr[ok] = (1.0 / cnt[inv.reshape(-1)].astype(np.float64)).astype(np.float32)
    return w, wr, int((~ok).any())


def mix64(x):
    """The splitmix64 finaliser, on a Python int or a numpy uint64 array (arithmetic mod 2^64)."""
    if isinstance(x, (int, np.integer)):
        return int(mix64(np.array([int(x) & 0xFFFFFFFFFFFFFFFF], dtype=np.uint64))[0])
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = x ^ (x >> np.uint64(30))
        x = (x * np.uint64(0xBF58476D1CE4E5B9)) & _M64
        x = x ^ (x >> np.uint64(27))
        x = (x * np.uint64(0x94D049BB133111EB)) & _M64
        return x ^ (x >> np.uint64(31))


def table_size(F):
    """Hash table slots gr_fact_weights uses for F facts: the power of two >= max(1024, 2F)."""
    T = 1024
    while T < 2 * F:
        T <<= 1
    return T


def home_slot(heads, rels, T):
    """The first probe of each (head, rel) key: mix64((head << 32) | rel) & (T - 1).  Only for constructing colliding
    keys: which slot a key ends in is not part of the kernel's contract."""
    h = np.asarray(heads, dtype=np.int64).astype(np.uint64)
    r = np.asarray(rels, dtype=np.int64).astype(np.uint64)
    return (mix64((h << np.uint64(32)) | r) & np.uint64(T - 1)).astype(np.int64)


def colliding_keys(n, slot, T, Nt, R):
    """(heads, rels): n distinct (head, rel) keys, head in [0, Nt) and rel in [0, R), whose home slot in a T-slot
    table is ``slot``: a probe chain of length n starting there."""
    h, r = np.divmod(np.arange(Nt * R, dtype=np.int64), R)
    pick = np.flatnonzero(home_slot(h, r, T) == slot)[:n]
    assert len(pick) == n, "not enough keys with home slot %d among %d x %d" % (slot, Nt, R)
    return h[pick], r[pick]


# ---- gr_graft_stage ----------------------------------------------------------------------------------------------------

BAD_ID, BAD_REL, DUP_SLOT, UNPAIRED = 1, 2, 4, 8


def graft_stage(e2f, f2e, kb_fact_rel, B, N, max_fact, R1, live=None):
    """GraftNet's facts paired by slot, as gr_graft_stage documents them.

    e2f = (b, f, head) and f2e = (b, tail, f), local ids; kb_fact_rel [B, max_fact]; ``live`` = (live head entries,
    live tail entries) or None.  -> dict with ``heads``, ``rels``, ``tails`` (global rows b*N + local) and ``slot_of``
    (b*max_fact + f) of every slot that has both a head and a tail, in slot order; ``nfacts`` = min(paired slots,
    len(e2f)); ``status``: bit 1 an entry with b, f or the node out of range (dropped), bit 2 a staged fact whose
    relation is outside [0, R1) (kept with relation 0), bit 4 a slot listed twice in one list, bit 8 a slot with a
    head but no tail or the reverse (dropped).  Of a slot listed twice the kernel keeps either node; the tests list a
    duplicate with the same node."""
    kb_fact_rel = np.asarray(kb_fact_rel, dtype=np.int64).reshape(B, max_fact)
    S = B * max_fact
    status = 0
    nodes = []
    for (bid, fid, nid), k in ((e2f, 0), ((f2e[0], f2e[2], f2e[1]), 1)):
        bid, fid, nid = (np.asarray(a, dtype=np.int64).reshape(-1) for a in (bid, fid, nid))
        L = live_count(len(bid), None if live is None else live[k])
        bid, fid, nid = bid[:L], fid[:L], nid[:L]
        ok = (bid >= 0) & (bid < B) & (fid >= 0) & (fid < max_fact) & (nid >= 0) & (nid < N)
        if not ok.all():
            status |= BAD_ID
        slot = bid[ok] * max_fact + fid[ok]
        if len(np.unique(slot)) != len(slot):
            status |= DUP_SLOT
        node_of = np.full(S, -1, dtype=np.int64)
        node_of[slot] = bid[ok] * N + nid[ok]
        nodes.append(node_of)
    head_of, tail_of = nodes
    if ((head_of >= 0) != (tail_of >= 0)).any():
        status |= UNPAIRED
    s = np.flatnonzero((head_of >= 0) & (tail_of >= 0))
    r = kb_fact_rel.reshape(-1)[s]
    if ((r < 0) | (r >= R1)).any():
        status |= BAD_REL
    r = np.where((r < 0) | (r >= R1), 0, r)
    return dict(heads=head_of[s], rels=r, tails=tail_of[s], slot_of=s, nfacts=min(len(s), len(np.asarray(e2f[0]))),
                status=status)
