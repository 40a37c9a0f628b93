"""CPU: the K-order layout of the dense layer's neighbour segments (GR_AGG_K_ORDER / GR_LINEAR_K_ORDER_PLANES)
restated in numpy -- the column map the aggregation writes, the k-block map the GEMM walks and the packed W planes --
and held to each other and to the grouped K order of fused_w_split_kernel: walking the K-order k-blocks must issue the
same k16 steps, in the same order, as the grouped walk over segment-layout planes, and give A W^T of the layer input.
Then the refusals of both entry points, which come before any CUDA call (the pointers are placeholders)."""
import ctypes

import numpy as np
import pytest

from gnn_rag_b200 import _lib, ops

PTR = ctypes.c_void_p(0x1000)
INVALID = -1


def seg(t, I):
    return 0 if t == 0 else 1 + 2 * ((t - 1) % I) + (t - 1) // I


def nb0(P):
    return (P + 31) // 32 * 32


def ko_col(u, c, P, I):
    """Column of column c of neighbour slot u (= direction d * I + instruction j) in the K-order layout."""
    Gf = P // 32
    if c < 32 * Gf:
        return nb0(P) + (c >> 5) * 32 * 2 * I + u * 32 + (c & 31)
    return nb0(P) + Gf * 32 * 2 * I + u * 16 + (c - 32 * Gf)


def grouped_steps(P, I):
    """k16 steps of the grouped walk: (segment, first column) in issue order, the k-block they belong to."""
    T, G = 2 * I + 1, (P + 31) // 32
    steps = []
    for g in range(G):
        for t in range(T):
            for k in range(min(2, (P - 32 * g) // 16)):
                steps.append((seg(t, I), 32 * g + 16 * k, g * T + t, k))
    return steps


def korder_kblocks(P, I):
    """K-order walk: [(A column of the 32-column box, k-steps)], as linear_tc_kernel's producer and consumer make it."""
    T, Gf, tail = 2 * I + 1, P // 32, P % 32 == 16
    nkb = Gf * T + (1 + I if tail else 0)
    out = []
    for kb in range(nkb):
        g = min(kb // T, Gf)
        t = kb - g * T
        col = 32 * g if t == 0 else nb0(P) + (kb - g - 1) * 32
        out.append((col, 1 if (tail and kb == Gf * T) else 2))
    return out


def packed_w_source(P, I):
    """Per packed W-plane column (k-block * 32 + c): the grouped W-plane column it copies, or -1 (zero)."""
    T, G = 2 * I + 1, (P + 31) // 32
    tail = P % 32 == 16
    nkb = (G - 1) * T + 1 + I if tail else G * T
    src = np.full(nkb * 32, -1)
    for blk in range(nkb):
        for c in range(32):
            b, cc = blk, c
            if tail and blk > (G - 1) * T:
                b = (G - 1) * T + 1 + 2 * (blk - (G - 1) * T - 1) + c // 16
                cc = c % 16
            src[blk * 32 + c] = b * 32 + cc
    return src


def w_planes(W, D, I, G):
    """Grouped-order planes of fused_w_split_kernel: block g*T + t = columns 32g.. of segment seg(t), zero past D."""
    T = 2 * I + 1
    out = np.zeros((W.shape[0], G * T * 32), W.dtype)
    for g in range(G):
        for t in range(T):
            n = max(0, min(32, D - 32 * g))
            out[:, (g * T + t) * 32:(g * T + t) * 32 + n] = W[:, seg(t, I) * D + 32 * g: seg(t, I) * D + 32 * g + n]
    return out


CASES = [(200, 2), (200, 1), (224, 2), (136, 1), (136, 3), (160, 3), (50, 3)]


@pytest.mark.parametrize("D,I", CASES)
def test_column_map_is_a_bijection_onto_the_region(D, I):
    P = (D + 15) // 16 * 16
    cols = [ko_col(u, c, P, I) for u in range(2 * I) for c in range(P)]
    assert sorted(cols) == list(range(nb0(P), nb0(P) + 2 * I * P))        # same width as the segment layout
    for u in range(2 * I):                                                # a lane's 4 columns stay contiguous
        for c in range(0, P, 4):
            assert [ko_col(u, c + i, P, I) for i in range(4)] == list(range(ko_col(u, c, P, I), ko_col(u, c, P, I) + 4))
    if D == 200:                                                          # fits the planes the model allocates
        assert nb0(P) + 2 * I * P <= ((2 * I + 1) * P + 63) // 64 * 64
        assert nb0(P) == 224 and nb0(P) + 2 * I * P == {1: 640, 2: 1056}[I]


@pytest.mark.parametrize("D,I", CASES)
def test_korder_walk_issues_the_grouped_k16_steps(D, I):
    rs = np.random.RandomState(D + I)
    P, T = (D + 15) // 16 * 16, 2 * I + 1
    G = (P + 31) // 32
    kbs = korder_kblocks(P, I)
    assert len(kbs) == (G * T if P % 32 == 0 else (G - 1) * T + 1 + I)
    assert all(col % 32 == 0 for col, _ in kbs)                           # every box 64-byte aligned
    if D == 200:
        assert len(kbs) == {1: 20, 2: 33}[I]             # 6 groups of T, the h tail, I packed blocks
    # which (segment, column) each issued k16 step reads, through the column map
    owner = {c: (0, c) for c in range(P)}                                 # plane column -> (segment, column)
    for s in range(1, T):
        for c in range(P):
            owner[ko_col(s2u(s, I), c, P, I)] = (s, c)
    steps = []
    for col, ks in kbs:
        for k in range(ks):
            s, c = owner[col + 16 * k]
            for i in range(16):                                           # a k16 step is 16 columns of one slot
                assert owner[col + 16 * k + i] == (s, c + i)
            steps.append((s, c))
    assert steps == [(s, c) for s, c, _, _ in grouped_steps(P, I)]
    # the packed W planes hold, per issued k16 step, the grouped planes' W columns of the same step
    Wg = w_planes(rs.randint(-9, 10, size=(5, T * D)), D, I, G)
    src = packed_w_source(P, I)
    gsteps = grouped_steps(P, I)
    n = 0
    for kb, (col, ks) in enumerate(kbs):
        for k in range(ks):
            _, _, gkb, gk = gsteps[n]
            assert list(src[kb * 32 + 16 * k: kb * 32 + 16 * k + 16]) == list(range(gkb * 32 + 16 * gk,
                                                                                    gkb * 32 + 16 * gk + 16))
            n += 1
    assert n == len(gsteps)
    # A W^T through the K-order layout and the packed planes (integers: every sum is exact)
    A = np.zeros((3, T, P), np.int64)
    A[:, :, :D] = rs.randint(-9, 10, size=(3, T, D))
    W = rs.randint(-9, 10, size=(5, T * D))
    Wg = w_planes(W, D, I, G)
    Wp = np.where(src >= 0, Wg[:, np.maximum(src, 0)], 0)
    width = nb0(P) + 2 * I * P
    a = np.full((3, width + 32), 10 ** 6, np.int64)                       # never-written columns must not enter
    a[:, :P] = A[:, 0]
    for s in range(1, T):
        for c in range(P):
            a[:, ko_col(s2u(s, I), c, P, I)] = A[:, s, c]
    acc = np.zeros((3, 5), np.int64)
    for kb, (col, ks) in enumerate(kbs):
        acc += a[:, col:col + 16 * ks] @ Wp[:, 32 * kb:32 * kb + 16 * ks].T
    assert (acc == A[:, :, :D].reshape(3, T * D) @ W.T).all()
    lib = _lib.load()
    plane = (5 * len(kbs) * 32 * 2 + 255) // 256 * 256
    assert lib.gr_fused_layer_workspace_bytes(D, P, I, 5) >= 2 * plane  # the workspace ops passes holds the packed planes


def s2u(s, I):
    """Neighbour slot u = d * I + j of segment s = 1 + 2j + d."""
    j, d = divmod(s - 1, 2)
    return d * I + j


def test_slot_order_is_the_fused_kernel_order():
    for I in (1, 2, 3):
        assert [s2u(seg(t, I), I) for t in range(1, 2 * I + 1)] == list(range(2 * I))


# ---- refusals ---------------------------------------------------------------------------------------------------------

def _agg_call(out_lo, I, D, P, flags):
    """A misaligned padded table: a call the argument checks admit is refused there, before any CUDA call."""
    lib = _lib.load()
    rc = lib.gr_aggregate_dual_abs_ex(PTR, PTR, PTR, None, PTR, PTR, PTR, None, PTR, ctypes.c_void_p(0x1008), PTR, 3,
                                      PTR, PTR, out_lo,
                                      2048, 224, P, 2, 64, D, I, 4, PTR, flags, None)
    return rc, lib.gr_last_error().decode()


@pytest.mark.parametrize("out_lo,I,D,P,msg", [
    (None, 2, 200, 208, "needs both planes"),                             # hi-only output (bf16 activation storage)
    (PTR, 3, 200, 208, "built for I <= 2"),
    (PTR, 2, 224, 224, "specialises D = 200"),                            # a width the aggregation does not specialise
    (PTR, 2, 200, 224, "specialises D = 200"),
])
def test_k_order_aggregation_refusals(out_lo, I, D, P, msg):
    rc, err = _agg_call(out_lo, I, D, P, ops.AGG_K_ORDER)
    assert rc == INVALID and msg in err, (rc, err)


def test_k_order_aggregation_admits_what_the_dense_layer_passes():
    # the same call with both planes is admitted up to the alignment of the (placeholder) padded tables
    rc, err = _agg_call(PTR, 2, 200, 208, ops.AGG_K_ORDER)
    assert rc == INVALID and "misaligned" in err, (rc, err)
    rc, err = _agg_call(PTR, 2, 200, 208, 2)
    assert rc == INVALID and "unknown flags" in err, (rc, err)


def _gemm_call(K, lda16, flags, k_seg=200, pitch=208):
    lib = _lib.load()
    rc = lib.gr_linear_tc_planes(PTR, PTR, lda16, PTR, 2048, None, PTR, 256, None, None, 0, None, None, 256, 200, K,
                                 k_seg, pitch, flags, PTR, 16, None)
    return rc, lib.gr_last_error().decode()


def test_k_order_gemm_refusals():
    G, KO = ops.LINEAR_K_GROUPED, ops.LINEAR_K_ORDER_PLANES
    for K, lda16, flags, msg in [
        (1040, 1088, KO, "needs it"),                                     # without GR_LINEAR_K_GROUPED
        (832, 1088, G | KO, "odd number of segments"),                    # an even segment count
        (1040, 1088, G | KO | ops.LINEAR_BF16_SINGLE, "does not combine"),    # the single-product mode
        (1040, 1048, G | KO, "cover the neighbour region"),               # planes end before 224 + 832 = 1056
    ]:
        rc, err = _gemm_call(K, lda16, flags)
        assert rc == INVALID and msg in err, (K, lda16, flags, rc, err)
    ops.set_option("tc_bk", 64)
    try:
        rc, err = _gemm_call(1040, 1088, G | KO)
        assert rc == INVALID and "32-column k-blocks" in err, (rc, err)
    finally:
        ops.set_option("tc_bk", 32)
    rc, _ = _gemm_call(1040, 1056, G | KO)                               # admitted: refused by the 16-byte workspace
    assert rc == -3
