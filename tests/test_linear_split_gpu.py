"""GPU: the exact-fp32 SIMT linear (csrc/linear_simt.cu, ``gr_linear``) against float64 per element, and the split of
fp32 activations into bf16 hi/lo planes (``gr_split_bf16``) against a CPU restatement bit for bit.

``gr_linear`` accumulates K products with fmaf, then adds the bias and the addend row, then applies relu; relu is
1-Lipschitz, so each element is within (K + 4) u (|A| |W|^T + |b| + |addend|) of the float64 value (u = 2^-24).

``gr_split_bf16`` writes hi = bf16_rn(x), lo = bf16_rn(x - hi) to the first K columns of each plane row, zeros to
columns K .. round4(K) - 1 and nothing else.  Above the largest finite bf16 (|x| >= 0x7F7F8000) hi rounds to inf and
lo is -inf, so hi + lo is NaN: pinned as it is.
"""
import numpy as np
import pytest
import torch

from gnn_rag_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
F64 = torch.float64
SENT = -7.25


def _view(M, K, ld, off, gen):
    """[M, K] fp32 rows at leading dimension ld, starting `off` floats into a fresh allocation."""
    buf = torch.empty(off + M * ld + 8, device=DEV)
    buf.normal_(generator=gen)
    return buf[off:off + M * ld].view(M, ld)[:, :K]


def _r4(n):
    return (n + 3) // 4 * 4


# A layouts: "vec" (16-byte aligned rows at ld % 4 == 0, K % 4 may be != 0: float4 loads with a scalar tail),
# "lda" (lda % 4 != 0), "a_off" / "w_off" (A or W one float past a 16-byte boundary): the scalar path
LAYOUTS = {"vec": (0, 0, True), "lda": (0, 0, False), "a_off": (1, 0, True), "w_off": (0, 1, True)}

SHAPES = [(1, 1, 1), (127, 63, 3), (128, 64, 4), (129, 65, 15), (2050, 200, 16), (129, 257, 17), (128, 65, 300),
          (127, 200, 1027), (1, 257, 1027), (2050, 64, 17), (128, 1, 3), (129, 257, 4)]


def _check_linear(M, N, K, layout, bias, relu, addend_rows, seed):
    gen = torch.Generator(device=DEV)
    gen.manual_seed(seed)
    a_off, w_off, ld4 = LAYOUTS[layout]
    lda = _r4(K) + 4 if ld4 else _r4(K) + 5
    A = _view(M, K, lda, a_off, gen)
    W = _view(N, K, _r4(K) + 4 if ld4 else K, w_off, gen)
    if layout != "vec":
        assert (A.stride(0) % 4 or A.data_ptr() % 16 or W.data_ptr() % 16 or W.stride(0) % 4)
    else:
        assert A.stride(0) % 4 == 0 and W.stride(0) % 4 == 0 and A.data_ptr() % 16 == 0 and W.data_ptr() % 16 == 0
    b = torch.randn(N, device=DEV, generator=gen) if bias else None
    add = torch.randn(M, N + 5, device=DEV, generator=gen)[:, :N] if addend_rows is not None else None
    buf = torch.full((M, N + 7), SENT, device=DEV)
    out = buf[:, 3:3 + N]
    got = ops.linear(A, W, b, relu=relu, out=out, addend=add, addend_rows=addend_rows or 0)
    assert got.data_ptr() == out.data_ptr()
    A64, W64 = A.to(F64), W.to(F64)
    pre = A64 @ W64.T
    scale = A64.abs() @ W64.abs().T
    if b is not None:
        pre, scale = pre + b.to(F64), scale + b.to(F64).abs()
    if add is not None and addend_rows:
        pre[:addend_rows] += add[:addend_rows].to(F64)
        scale[:addend_rows] += add[:addend_rows].to(F64).abs()
    want = torch.relu(pre) if relu else pre
    bound = (K + 4) * U * scale
    err = (out.to(F64) - want).abs()
    assert (err <= bound).all(), (err / bound).max().item()
    if relu and M * N >= 64:
        assert (pre < 0).any() and (pre > 0).any()                              # pre-activations of both signs
    assert (buf[:, :3] == SENT).all() and (buf[:, 3 + N:] == SENT).all()      # nothing written past the window
    return (err / bound.clamp_min(1e-300)).max().item()


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_linear_vs_fp64(M, N, K):
    worst = 0.0
    for i, layout in enumerate(LAYOUTS):
        rows = (None, 0, 1, M - 1, M)[(i + K) % 5]
        worst = max(worst, _check_linear(M, N, K, layout, bias=(i + N) % 2 == 0, relu=i % 2 == 1,
                                         addend_rows=rows, seed=M * 7 + N * 3 + K + i))
    print("gr_linear max err/bound %s: %.3g" % ((M, N, K), worst))


@pytest.mark.parametrize("rows", ["0", "1", "M-1", "M"])
def test_linear_addend_rows(rows):
    M, N, K = 300, 65, 17
    n = {"0": 0, "1": 1, "M-1": M - 1, "M": M}[rows]
    for relu in (False, True):
        for bias in (False, True):
            _check_linear(M, N, K, "vec", bias, relu, n, seed=n + 2 * relu + bias)


@pytest.mark.parametrize("M,N,K,bias", [(4000, 50, 100, True), (4000, 200, 300, True), (2000, 400, 300, True),
                                        (16, 200, 200, True), (16, 200, 600, False)],
                         ids=["entity_d50", "entity_d200", "entity_d400", "graft_q2e", "graft_e2q"])
def test_linear_model_shapes(M, N, K, bias):
    """entity_linear at D = 50 / 200 / 400 (models.py), GraftNet's q2e [B, D] -> D and e2q [B, 3D] -> D (no bias)."""
    _check_linear(M, N, K, "vec", bias, relu=False, addend_rows=None, seed=N + K)


# ------------------------------------------------------------------ split_bf16 -------------------------------------
def _split_ref(x):
    """CPU restatement: hi = bf16_rn(x), lo = bf16_rn(x - hi) (torch rounds fp32 -> bf16 to nearest even)."""
    x = x.cpu()
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return hi, lo


def _same(got, want):
    """Bit equality of bf16 tensors, NaN compared by isnan."""
    got, want = got.cpu(), want.cpu()
    gn, wn = torch.isnan(got.float()), torch.isnan(want.float())
    return torch.equal(gn, wn) and torch.equal(got.view(torch.int16)[~gn], want.view(torch.int16)[~wn])


def _check_split(x, c0, ld):
    """split x [M, K] into hi[:, c0:], lo[:, c0:] of sentinel-filled [M, ld] planes and check every column."""
    M, K = x.shape
    assert c0 + _r4(K) <= ld
    hi = torch.full((M, ld), SENT, dtype=torch.bfloat16, device=DEV)
    lo = torch.full((M, ld), SENT, dtype=torch.bfloat16, device=DEV)
    ops.split_bf16(x, hi[:, c0:], lo[:, c0:])
    hw, lw = _split_ref(x)
    assert _same(hi[:, c0:c0 + K], hw) and _same(lo[:, c0:c0 + K], lw)
    for p in (hi, lo):
        assert (p[:, c0 + K:c0 + _r4(K)] == 0).all()                       # the tail up to round4(K) is zero
        assert (p[:, c0 + _r4(K):] == SENT).all() and (p[:, :c0] == SENT).all()


@pytest.mark.parametrize("K", [1, 2, 3, 4, 5, 6, 7, 8, 9, 63, 64, 65, 200, 1000])
def test_split_bf16_shapes(K):
    """Aligned rows (float4 loads), unaligned lda or base (scalar loads); plane windows at column offsets 0, 8 (as
    NSM's neighbour window hi[:, Dp:]), 4 and 2 (a base only 4-byte aligned: scalar stores)."""
    gen = torch.Generator(device=DEV)
    gen.manual_seed(K)
    M = 133
    for lda, off in ((_r4(K), 0), (_r4(K) + 4, 0), (K + 1, 0), (_r4(K), 1)):
        x = _view(M, K, lda, off, gen)
        ld = (K + 8 + 16 + 7) // 8 * 8
        for c0 in (0, 8, 4, 2):
            _check_split(x, c0, ld)


def _f32(bits):
    return torch.tensor(np.array(bits, dtype=np.uint32).view(np.int32)).view(torch.float32)


def test_split_bf16_values():
    """Exact bf16 values, round-half-even ties on even and odd mantissas, +-0, fp32 subnormals and values whose hi is
    subnormal, +-inf, NaN and |x| >= 0x7F7F8000 (hi = +-inf, lo = -+inf: hi + lo is NaN)."""
    rs = np.random.RandomState(0)
    exact = (rs.randint(0, 1 << 16, size=64) << 16).astype(np.uint32)                   # lo = 0
    hi16 = rs.randint(0, 0x7F7F, size=64).astype(np.uint32)
    ties = np.concatenate([((hi16 & 0xFFFE) << 16) | 0x8000, ((hi16 | 1) << 16) | 0x8000])  # even / odd mantissa
    near = (hi16 << 16) | rs.randint(0, 1 << 16, size=64).astype(np.uint32)
    sub = np.concatenate([np.arange(1, 40), rs.randint(1, 0x00800000, size=64),
                          [0x007FFFFF, 0x007F8000, 0x00008000, 0x00018000]]).astype(np.uint32)
    lowhi = (rs.randint(0, 0x0200, size=32) << 16 | rs.randint(0, 1 << 16, size=32)).astype(np.uint32)
    special = np.array([0, 0x7F800000, 0x7FC00000, 0x7F800001, 0x7F7F7FFF, 0x7F7F8000, 0x7F7FFFFF, 0x7F7F8001],
                       dtype=np.uint32)
    bits = np.concatenate([exact, ties, near, sub, lowhi, special]).astype(np.uint32)
    bits = np.concatenate([bits, bits | 0x80000000])                                      # both signs, -0 included
    vals = _f32(bits)
    K = 13
    pad = (-len(vals)) % K
    x = torch.cat([vals, torch.zeros(pad)]).view(-1, K).to(DEV)
    for c0 in (0, 2):
        _check_split(x, c0, 24)
    # the saturating values, spelled out
    big = _f32([0x7F7F8000, 0x7F7FFFFF, 0xFF7F8000]).to(DEV).view(1, 3)
    hi = torch.empty(1, 8, dtype=torch.bfloat16, device=DEV)
    lo = torch.empty(1, 8, dtype=torch.bfloat16, device=DEV)
    ops.split_bf16(big, hi, lo)
    assert hi[0, :3].tolist() == [float("inf"), float("inf"), float("-inf")]
    assert lo[0, :3].tolist() == [float("-inf"), float("-inf"), float("inf")]
    assert torch.isnan(hi[0, :3].float() + lo[0, :3].float()).all()
