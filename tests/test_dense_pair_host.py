"""CPU: the K map of the grouped order (GR_LINEAR_K_GROUPED, csrc/wgmma.cuh) restated in numpy and held to the W
layout of fused_w_split_kernel -- walking the k-blocks g*T + t over A columns seg(t)*pitch + 32g and W-plane columns
32 (g*T + t) must give A W^T of the segmented layer input --, the workspace size both entry points share, and the
refusals of gr_linear_tc_planes, which come before any CUDA call (the pointers are placeholders)."""
import ctypes

import numpy as np
import pytest

from gnn_rag_b200 import _lib, ops

PTR = ctypes.c_void_p(0x1000)
INVALID = -1


def seg(t, I):
    return 0 if t == 0 else 1 + 2 * ((t - 1) % I) + (t - 1) // I


def w_planes(W, D, I, G):
    """[N, G*T*32] planes of W [N, T*D] in grouped order: block g*T + t = columns 32g.. of segment seg(t), zero past D."""
    T = 2 * I + 1
    out = np.zeros((W.shape[0], G * T * 32), W.dtype)
    for g in range(G):
        for t in range(T):
            n = max(0, min(32, D - 32 * g))
            out[:, (g * T + t) * 32:(g * T + t) * 32 + n] = W[:, seg(t, I) * D + 32 * g: seg(t, I) * D + 32 * g + n]
    return out


@pytest.mark.parametrize("D,I", [(200, 2), (200, 1), (224, 2), (136, 1), (136, 3), (160, 3), (50, 3)])
def test_grouped_k_map_matches_the_w_layout(D, I):
    rs = np.random.RandomState(D + I)
    P, T = (D + 15) // 16 * 16, 2 * I + 1
    G = (P + 31) // 32
    ksteps_last = (P - 32 * (G - 1)) // 16
    assert ksteps_last in (1, 2)
    assert sorted(seg(t, I) for t in range(T)) == list(range(T))          # every segment once per group
    assert [seg(t, I) for t in range(1, I + 1)] == [1 + 2 * j for j in range(I)]      # direction 0 first (forward)
    A = np.zeros((3, T, P), np.int64)
    A[:, :, :D] = rs.randint(-9, 10, size=(3, T, D))                      # integers: every sum below is exact
    W = rs.randint(-9, 10, size=(5, T * D))
    Wp = w_planes(W, D, I, G)
    a = np.concatenate([A.reshape(3, T * P), np.full((3, 32), 10 ** 6)], 1)     # what lies past K must not enter
    acc = np.zeros((3, 5), np.int64)
    for kb in range(G * T):
        g, t = divmod(kb, T)
        cols = 16 * ksteps_last if g == G - 1 else 32                      # a 16-column last group is one k-step
        a0 = seg(t, I) * P + 32 * g
        acc += a[:, a0:a0 + cols] @ Wp[:, 32 * kb:32 * kb + cols].T
    want = A[:, :, :D].reshape(3, T * D) @ W.T
    assert (acc == want).all()
    lib = _lib.load()
    plane = (5 * G * T * 32 * 2 + 255) // 256 * 256
    assert lib.gr_fused_layer_workspace_bytes(D, P, I, 5) == 2 * plane


def _planes_call(K, k_seg, k_seg_pitch, flags, N=200):
    lib = _lib.load()
    rc = lib.gr_linear_tc_planes(PTR, PTR, 2048, PTR, 2048, None, PTR, 256, None, None, 0, None, None, 256, N, K, k_seg,
                                 k_seg_pitch, flags, PTR, 1 << 30, None)
    return rc, lib.gr_last_error().decode()


def test_grouped_flag_refusals():
    G = ops.LINEAR_K_GROUPED
    for K, k_seg, pitch, flags, msg in [
        (832, 200, 208, G, "odd number of segments"),                     # T = 4
        (1040, 0, 0, G, "needs segmented K"),                             # unsegmented K
        (1040, 200, 0, G, "needs segmented K"),
        (1000, 200, 200, G, "needs segmented K"),                         # pitch not a multiple of 16
        (1040, 200, 208, G | ops.LINEAR_BF16_SINGLE, "does not combine"),
    ]:
        rc, err = _planes_call(K, k_seg, pitch, flags)
        assert rc == INVALID and msg in err, (K, k_seg, pitch, flags, rc, err)
    ops.set_option("tc_bk", 64)
    try:
        rc, err = _planes_call(1040, 200, 208, G)
        assert rc == INVALID and "32-column k-blocks" in err, (rc, err)
    finally:
        ops.set_option("tc_bk", 32)
    # the same shapes pass the argument checks without the flag's conditions violated: the refusal that remains is the
    # workspace (a 16-byte workspace cannot hold the W planes)
    lib = _lib.load()
    rc = lib.gr_linear_tc_planes(PTR, PTR, 2048, PTR, 2048, None, PTR, 256, None, None, 0, None, None, 256, 200, 1040,
                                 200, 208, G, PTR, 16, None)
    assert rc == -3
