"""GPU: the question-side training kernels (csrc/question.cu: gr_instructions_train, gr_instructions_backward,
gr_instructions_dropout_mask, gr_query_reform_ex, gr_query_reform_backward) and the autograd Functions that use them
(autograd_path._InstructionsFn, _QueryReformFn).

Every output buffer starts as NaN and the C entry points are called directly, so an unwritten element fails.  Bounds
(u = 2^-24, no fast-math):
  * instructions backward: the float64 restatement of tests/question_train_ref.py, conditioned on the kernel's own
    forward ri and attention (as tests/test_question_side_gpu.py conditions each step on the kernel's previous
    instruction), holds every output within K u mag, where mag is the same computation on absolute values and
    K = I (7 D + 3 Q + 64) counts the roundings on the longest chain into an element: per step the recomputed
    question_linear (D) and cq_linear (4D) rows, the token dot (D), the softmax sum and the token walk (2 Q), the
    transposed cq_linear and question_linear sums (D each), and a few element-wise operations;
  * query reform backward: a first-order forward error analysis of the kernel's operation order, written out in
    ``_reform_bounds`` (the seed walk, the GEMV rows, sigmoid as 1 / (1 + expf(-x)) within 8 u plus a quarter of its
    argument's error, the transposed sums).
A dropped or doubled term, a wrong mask, step or seed row moves an element by a sizeable fraction of its scale."""
import math

import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import _lib, autograd_path, ops, synthetic as S

import question_train_ref as QT
import test_amp_train_gpu as AMP
import test_question_side_gpu as QS
import test_training_path as TP

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
F64 = torch.float64
BF = torch.bfloat16
_p = ops._p


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def _bits_equal(a, b):
    torch.cuda.synchronize()
    assert a.dtype == b.dtype and a.shape == b.shape
    view = torch.int16 if a.dtype == BF else torch.int32
    eq = a.contiguous().view(view) == b.contiguous().view(view)
    assert bool(eq.all()), "%d of %d elements differ" % (int((~eq).sum()), eq.numel())


# --------------------------------------------------------------------------------------------------------------
# instructions
# --------------------------------------------------------------------------------------------------------------
def _seed(v):
    return torch.tensor([v], dtype=torch.int64, device=DEV)


def _ins_args(L):
    return [_p(L.hid), _p(L.qn), _p(L.text), L.PAD, ops._ptr_array(L.Wq), ops._ptr_array(L.bq), _p(L.Wcq), _p(L.bcq),
            _p(L.wca), _p(L.bca)]


def _ins_train(L, seed, p):
    out, at = _nan(L.B, L.I, L.D), _nan(L.B, L.I, L.Q)
    _lib.check(_lib.load().gr_instructions_train(*_ins_args(L), _p(seed), p, _p(out), _p(at), L.B, L.Q, L.D, L.I,
                                                  ops._stream()))
    return out, at


def _ins_backward(L, seed, p, out, at, Gout):
    B, Q, D, I = L.B, L.Q, L.D, L.I
    bufs = dict(grad_hidden=_nan(B, Q, D), grad_qnode=_nan(B, D), g_q=_nan(B, I, D), x_q=_nan(B, I, D),
                g_cq=_nan(B, I, D), x_cq=_nan(B, I, 4 * D), g_ca=_nan(B, I, Q), x_ca=_nan(B, I, Q, D))
    _lib.check(_lib.load().gr_instructions_backward(*_ins_args(L), _p(seed), p, _p(out), _p(at), _p(Gout),
                                                     *(_p(t) for t in bufs.values()), B, Q, D, I, ops._stream()))
    return bufs


def _masks(seed, p, L):
    if p == 0:
        return None
    m = ops.instructions_dropout_mask(seed, p, L.B, L.Q, L.D, L.I)
    return [t.bool().cpu().numpy() for t in m]


def _check(got, want, bound, what):
    err = (got.to(F64) - want).abs()
    ok = err <= bound
    assert ok.all(), "%s: %d bad, worst err/bound %g" % (what, int((~ok).sum()), (err / bound).max().item())


INS_CASES = [(3, 1, 1, 1), (3, 31, 33, 2), (3, 32, 200, 4), (3, 33, 256, 8), (2, 100, 400, 8), (3, 33, 1, 8),
             (4, 20, 50, 3), (3, 16, 64, 2)]


def _run_ins_case(B, Q, D, I, p, L=None):
    L = L or QS._Ins(Q * 100 + D + I + int(p * 10), B, Q, D, I)
    seed = _seed(1234 + D)
    out, at = _ins_train(L, seed, p)
    Gout = torch.from_numpy(np.random.RandomState(D + I).randn(B, I, D).astype(np.float32)).to(DEV)
    got = _ins_backward(L, seed, p, out, at, Gout)
    torch.cuda.synchronize()
    masks = _masks(seed, p, L)
    want, mag = QT.instructions_backward(L.hid, L.qn, L.Wq, L.bq, L.Wcq, L.bcq, L.wca, out, at, Gout, masks, p)
    K = I * (7 * D + 3 * Q + 64)
    for k, v in want.items():
        _check(got[k], v, K * U * mag[k] + 1e-30, k)
    return L, out, at


@pytest.mark.parametrize("B,Q,D,I", INS_CASES)
@pytest.mark.parametrize("p", [0.0, 0.3])
def test_instructions_backward_vs_fp64(B, Q, D, I, p):
    """grad_hidden, grad_qnode and every weight-gradient operand; a pad inside question 0, an all-pad last question,
    I = 1-8, D from 1 to 400; with and without dropout."""
    _run_ins_case(B, Q, D, I, p)


@pytest.mark.parametrize("D,I", [(200, 2), (33, 1), (400, 8)])
def test_instructions_backward_at_the_largest_admitted_question(D, I):
    Q = QS._q_max(D, I)
    _run_ins_case(2, Q, D, I, 0.2)
    L2 = QS._Ins(D + I, 2, Q + 1, D, I)
    with pytest.raises(_lib.GrError, match="gr_instructions_train: invalid argument.*too large"):
        _ins_train(L2, _seed(1), 0.2)
    with pytest.raises(_lib.GrError, match="gr_instructions_backward: invalid argument.*too large"):
        _ins_backward(L2, _seed(1), 0.2, _nan(2, I, D), _nan(2, I, Q + 1), _nan(2, I, D))


@pytest.mark.parametrize("B,Q,D,I", INS_CASES)
def test_instructions_train_without_dropout_is_gr_instructions_bit_for_bit(B, Q, D, I):
    L = QS._Ins(Q * 100 + D + I, B, Q, D, I)
    want, wat = L.run()
    got, gat = _ins_train(L, _seed(5), 0.0)
    _bits_equal(got, want)
    _bits_equal(gat, wat)


@pytest.mark.parametrize("B,Q,D,I", [(3, 31, 33, 2), (3, 33, 256, 8), (4, 20, 50, 3)])
def test_instructions_train_with_dropout_vs_fp64(B, Q, D, I):
    """The forward with dropout against the float64 restatement with the kernel's masks, each step from the kernel's
    previous instruction.  A plain tolerance (1e-4 of the instruction scale, 1e-4 on the attention): the per-element
    bounds of the dropout-free kernel are in test_question_side_gpu, and p = 0 is that kernel bit for bit (above); a
    wrong mask or scale moves an element by a sizeable fraction of its scale."""
    L = QS._Ins(Q + D + I, B, Q, D, I)
    seed, p = _seed(99), 0.25
    out, at = _ins_train(L, seed, p)
    torch.cuda.synchronize()
    masks = _masks(seed, p, L)
    mask = (L.text != L.PAD).to(F64)
    for i in range(I):
        sub = [m[:, i:i + 1] for m in masks]
        ri0 = out[:, i - 1].to(F64) if i > 0 else torch.zeros(B, D, dtype=F64, device=DEV)
        ri, att = _fwd_from(L, i, ri0, sub, p, mask)
        _check(out[:, i], ri[:, 0], 1e-4 * (1 + ri.abs().max()), "ri step %d" % i)
        _check(at[:, i], att[:, 0], 1e-4, "attn step %d" % i)


def _fwd_from(L, i, ri0, masks, p, mask):
    s = [torch.as_tensor(m, dtype=F64, device=DEV) / (1 - p) for m in masks]
    hid, qn = L.hid.to(F64), L.qn.to(F64)
    q = (qn * s[0][:, 0]) @ L.Wq[i].to(F64).t() + L.bq[i].to(F64)
    z = torch.cat([ri0, q, q - ri0, q * ri0], 1) * s[1][:, 0]
    cq = z @ L.Wcq.to(F64).t() + L.bcq.to(F64)
    ca = (cq.unsqueeze(1) * hid * s[2][:, 0]) @ L.wca.to(F64) + L.bca.to(F64)
    attn = torch.softmax(torch.where(mask > 0, ca, torch.full_like(ca, QT.VERY_NEG)), 1)
    return (attn.unsqueeze(2) * hid).sum(1).unsqueeze(1), attn.unsqueeze(1)


def test_dropout_mask_equals_the_numpy_restatement():
    B, Q, D, I = 3, 7, 37, 4
    for sv, p in ((12345, 0.3), ((1 << 61) + 977, 0.55), (7, 0.05)):
        got = ops.instructions_dropout_mask(_seed(sv), p, B, Q, D, I)
        want = QT.ins_masks(sv, p, B, Q, D, I)
        for g, w in zip(got, want):
            assert np.array_equal(g.cpu().numpy().astype(bool), w)


def test_dropout_kept_fraction_is_within_the_binomial_bound():
    """n Bernoulli(1 - p) draws: the kept fraction is within 6 standard deviations of 1 - p (a false failure has
    probability below 1e-8), for each site."""
    B, Q, D, I = 64, 40, 200, 4
    for p in (0.1, 0.5):
        for m in ops.instructions_dropout_mask(_seed(31), p, B, Q, D, I):
            n = m.numel()
            frac = float(m.double().mean())
            assert abs(frac - (1 - p)) <= 6 * math.sqrt(p * (1 - p) / n), (p, frac, n)


def test_instructions_dropout_refusals():
    L = QS._Ins(3, 2, 5, 16, 2)
    with pytest.raises(_lib.GrError, match="null seed"):
        _ins_train(L, None, 0.3)
    with pytest.raises(_lib.GrError, match="outside"):
        _ins_train(L, _seed(1), 1.0)
    L9 = QS._Ins(9, 2, 5, 16, 9)
    with pytest.raises(_lib.GrError, match="gr_instructions_train: invalid argument"):
        _ins_train(L9, _seed(1), 0.1)


# --------------------------------------------------------------------------------------------------------------
# query reform
# --------------------------------------------------------------------------------------------------------------
def _reform_bwd(L, Gout, grad_h, io=0, h=None):
    B, I, D = L.B, L.I, L.D
    h = L.h if h is None else h
    bufs = dict(grad_ins=_nan(B, I, D), g_r=_nan(B, I, D), g_g=_nan(B, I, D), x_z=_nan(B, I, 3 * D))
    _lib.check(_lib.load().gr_query_reform_backward(
        _p(L.seed), _p(h), h.stride(0), _p(L.ins), ops._ptr_array(L.Wr), ops._ptr_array(L.Wg), _p(Gout),
        _p(bufs["grad_ins"]), _p(grad_h), grad_h.stride(0), _p(bufs["g_r"]), _p(bufs["g_g"]), _p(bufs["x_z"]), B, L.N,
        D, I, io, ops._stream()))
    return bufs


def _gam(n):
    return (n + 8) * U


def _reform_bounds(L, Gout, ref):
    """First-order bounds of every output of gr_query_reform_backward (module docstring)."""
    B, N, D, I = L.B, L.N, L.D, L.I
    ey = QS._seed_bound(L.seed, L.h, B, N)
    G_ = Gout.to(F64).abs()
    x = L.ins.to(F64)
    b = {k: [] for k in ("grad_ins", "g_r", "g_g", "x_z")}
    egy = torch.zeros_like(ey)
    for j in range(I):
        xj, y = x[:, j], ref["y"]
        z = ref["x_z"][:, j]
        ez = torch.cat([torch.zeros_like(ey), ey, ey + U * (xj - y).abs()], 1)
        Wr, Wg = L.Wr[j].to(F64).abs(), L.Wg[j].to(F64).abs()
        r, g = ref["r"][:, j], ref["g"][:, j]
        er = _gam(3 * D) * (z.abs() @ Wr.t()) + ez @ Wr.t()
        eg = (_gam(3 * D) * (z.abs() @ Wg.t()) + ez @ Wg.t()) / 4 + 8 * U
        gr, gg = ref["g_r"][:, j], ref["g_g"][:, j]
        e_gr = G_[:, j] * eg + U * gr.abs()
        e_gg = G_[:, j] * (g * (1 - g) * er + (r - xj).abs() * eg) + 6 * U * gg.abs()
        gxd = G_[:, j] * (1 - g)
        e_gxd = G_[:, j] * eg + 2 * U * gxd
        mz = gr.abs() @ Wr + gg.abs() @ Wg
        gz = gr @ L.Wr[j].to(F64) + gg @ L.Wg[j].to(F64)
        e_gz = _gam(D) * mz + e_gr @ Wr + e_gg @ Wg + U * mz
        e0, e1, e2 = e_gz.split(D, 1)
        g0, g1, g2 = gz.abs().split(D, 1)
        b["grad_ins"].append(e_gxd + e0 + e2 + 2 * U * (gxd + g0 + g2))
        egy = egy + e1 + e2 + 2 * I * U * (g1 + g2)
        b["g_r"].append(e_gr)
        b["g_g"].append(e_gg)
        b["x_z"].append(ez)
    out = {k: torch.stack(v, 1) for k, v in b.items()}
    s = L.seed.to(F64).abs()
    out["grad_h"] = (s.view(B, N, 1) * (egy + U * ref["grad_y"].abs()).view(B, 1, D)).reshape(B * N, D)
    return out


REFORM_CASES = [(1, 1, 1), (63, 3, 1023), (64, 8, 1024), (65, 2, 1025), (128, 4, 1024), (200, 2, 3000),
                (1024, 1, 1025), (65, 8, 1), (50, 3, 500)]


@pytest.mark.parametrize("D,I,N", REFORM_CASES)
@pytest.mark.parametrize("ldh_pad", [0, 3])
def test_query_reform_backward_vs_fp64(D, I, N, ldh_pad):
    """grad_ins, the operands and the seed rows of grad_h, for seeds none / one / across the 1024-node chunk edges /
    dense, h plain or strided; every other row of the (pre-filled) grad_h unchanged bit for bit."""
    L = QS._Reform(D * 10 + I + N, 4, N, D, I, ldh_pad)
    rs = np.random.RandomState(D + I)
    Gout = torch.from_numpy(rs.randn(L.B, I, D).astype(np.float32)).to(DEV)
    pre = torch.from_numpy(rs.randn(L.B * N, D + 2).astype(np.float32)).to(DEV)[:, :D]   # strided grad_h
    grad_h = pre.clone()
    got = _reform_bwd(L, Gout, grad_h)
    torch.cuda.synchronize()
    ref = QT.reform_backward(L.seed, L.h, L.ins, L.Wr, L.Wg, L.B, N, Gout)
    bound = _reform_bounds(L, Gout, ref)
    for k in ("grad_ins", "g_r", "g_g", "x_z"):
        _check(got[k], ref[k], bound[k] + 1e-30, k)
    seeded = (L.seed != 0).reshape(-1)
    _bits_equal(grad_h[~seeded], pre[~seeded])
    want_h = pre.to(F64) + ref["grad_h"]
    _check(grad_h[seeded], want_h[seeded], (bound["grad_h"] + U * want_h.abs())[seeded] + 1e-30, "grad_h")


@pytest.mark.parametrize("I", [1, 3, 8])
def test_query_reform_backward_at_the_widest_admitted_width(I):
    D = QS._reform_d_max(I)
    L = QS._Reform(I, 2, 300, D, I, ldh_pad=1)
    Gout = torch.randn(2, I, D, device=DEV)
    grad_h = torch.zeros(2 * 300, D, device=DEV)
    got = _reform_bwd(L, Gout, grad_h)
    torch.cuda.synchronize()
    ref = QT.reform_backward(L.seed, L.h, L.ins, L.Wr, L.Wg, 2, 300, Gout)
    bound = _reform_bounds(L, Gout, ref)
    _check(got["grad_ins"], ref["grad_ins"], bound["grad_ins"] + 1e-30, "grad_ins")
    _check(grad_h, ref["grad_h"], bound["grad_h"] + 1e-30, "grad_h")
    L2 = QS._Reform(I, 2, 8, D + 1, I)
    with pytest.raises(_lib.GrError, match="gr_query_reform_backward: invalid argument"):
        _reform_bwd(L2, torch.zeros(2, I, D + 1, device=DEV), torch.zeros(16, D + 1, device=DEV))


@pytest.mark.parametrize("D,I,N", [(50, 3, 500), (200, 2, 1025), (1024, 1, 300)])
def test_query_reform_bf16_h_equals_the_fp32_kernel_on_the_upcast_h(D, I, N):
    """GR_IO_BF16: forward and backward equal the fp32 calls on h.float(); the bf16 grad_h holds the fp32 result
    rounded to nearest even (pre-filled bf16 rows widened, the seed term added, rounded once)."""
    L = QS._Reform(D + I, 4, N, D, I)
    h16 = L.h.to(BF)
    out16 = ops.query_reform(L.seed, h16, L.ins, L.Wr, L.Wg, L.B, N)
    out32 = ops.query_reform(L.seed, h16.float(), L.ins, L.Wr, L.Wg, L.B, N)
    _bits_equal(out16, out32)
    Gout = torch.randn(L.B, I, D, device=DEV)
    pre16 = torch.randn(L.B * N, D, device=DEV).to(BF)
    g16, g32 = pre16.clone(), pre16.float()
    a = _reform_bwd(L, Gout, g16, io=ops.IO_BF16, h=h16)
    b = _reform_bwd(L, Gout, g32, io=0, h=h16.float())
    for k in a:
        _bits_equal(a[k], b[k])
    _bits_equal(g16, g32.to(BF))


def test_query_reform_fp32_equals_gr_query_reform_ex_with_io_0():
    """The fp32 wrapper and gr_query_reform_ex with io = 0 give the bits of gr_query_reform."""
    L = QS._Reform(7, 4, 1025, 130, 3, ldh_pad=3)
    out, _ = L.run()
    _bits_equal(ops.query_reform(L.seed, L.h, L.ins, L.Wr, L.Wg, L.B, L.N), out)
    ex = _nan(L.B, L.I, L.D)
    _lib.check(_lib.load().gr_query_reform_ex(_p(L.seed), _p(L.h), L.h.stride(0), _p(L.ins), ops._ptr_array(L.Wr),
                                              ops._ptr_array(L.Wg), _p(ex), None, L.B, L.N, L.D, L.I, 0,
                                              ops._stream()))
    _bits_equal(ex, out)


# --------------------------------------------------------------------------------------------------------------
# end to end
# --------------------------------------------------------------------------------------------------------------
def _model(name, seed=0, **over):
    kw = dict(use_cuda=True, lm_dropout=0.0, linear_dropout=0.0)
    kw.update(over)
    torch.manual_seed(seed)
    return getattr(G, name)(S.model_args(name, **kw), 1000, 40, 100).cuda()


def _batch(seed=5, B=6, N=120, E=600):
    return S.make_batch(seed, B=B, N=N, E=E, num_entity=1000, num_relation=40, num_word=100, powerlaw=True,
                        n_real="ragged", with_weights=True)


def _grads(m, b, kernels, monkeypatch, amp=False):
    """Loss and parameter gradients of one step with the question-side kernels on or off (the rest unchanged)."""
    with monkeypatch.context() as mp:
        if not kernels:
            mp.setattr(autograd_path, "_instruction_kernels", lambda *a: False)
            mp.setattr(autograd_path, "_reform_kernels", lambda *a: False)
        m.zero_grad()
        torch.manual_seed(11)
        with torch.autocast("cuda", dtype=BF, enabled=amp), torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            loss = m(b, training=True)[0]
            loss.backward()
    return float(loss), {k: p.grad.detach().float().clone() for k, p in m.named_parameters() if p.grad is not None}


def _agree(ga, gb, tol=2e-4):
    """Per tensor: max |a - b| <= tol * max|b| + 1e-6 * (largest gradient in the model).  The score bias is left out:
    softmax is shift invariant, so its exact gradient is zero and both paths hold rounding noise there."""
    assert set(ga) == set(gb)
    gmax = max(float(g.abs().max()) for g in gb.values())
    for k in gb:
        if k.endswith("score_func.bias"):
            continue
        err = float((ga[k] - gb[k]).abs().max())
        assert err <= tol * float(gb[k].abs().max()) + 1e-6 * gmax, (k, err, float(gb[k].abs().max()))


E2E = {"rearev_lstm": ("ReaRev", dict(entity_dim=50, num_iter=3, num_ins=2, num_gnn=2)),
       "rearev_cwq": ("ReaRev", dict(entity_dim=50, num_iter=2, num_ins=3, num_gnn=2)),
       "nsm": ("NSM", dict(entity_dim=64, num_step=3, reason_kb=True))}


@pytest.mark.parametrize("key", list(E2E))
def test_gradients_agree_with_the_torch_question_side(key, monkeypatch):
    """p = 0, kernels on and off: the loss within 1e-5 relative and every parameter gradient within 2e-4 of its
    tensor's scale plus 1e-6 of the model's largest gradient (fp32 rounding of two summation orders)."""
    name, over = E2E[key]
    m = _model(name, **over).train()
    b = _batch()
    calls = []
    with monkeypatch.context() as mp:
        for fn in ("_InstructionsFn", "_QueryReformFn"):
            cls = getattr(autograd_path, fn)
            mp.setattr(cls, "apply", (lambda f, n: lambda *a: calls.append(n) or f(*a))(cls.apply, fn))
        la, ga = _grads(m, b, True, monkeypatch)
    assert "_InstructionsFn" in calls and (name != "ReaRev" or "_QueryReformFn" in calls)
    lb, gb = _grads(m, b, False, monkeypatch)
    assert abs(la - lb) <= 1e-5 * abs(lb)
    _agree(ga, gb)


def test_gradients_agree_on_the_sbert_reltext_golden(monkeypatch):
    m, batch, _t = TP._load("rearev_sbert_reltext", device="cuda")
    m = m.cuda().train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.eval()
    m.instruction.node_encoder.eval()
    la, ga = _grads(m, batch, True, monkeypatch)
    lb, gb = _grads(m, batch, False, monkeypatch)
    assert abs(la - lb) <= 1e-5 * abs(lb)
    _agree(ga, gb)


def test_dropout_is_drawn_from_the_torch_seed(monkeypatch):
    """The forward with dropout is a function of torch.manual_seed: the same seed gives the same loss, another seed
    another loss.  (Gradients repeat bit for bit only under use_deterministic_algorithms: the default aggregation
    backward sums with fp32 atomics; see the deterministic test below.)"""
    m = _model("ReaRev", linear_dropout=0.3, entity_dim=50, num_iter=2, num_ins=2, num_gnn=2).train()
    b = _batch()
    la, _ = _grads(m, b, True, monkeypatch)
    lb, _ = _grads(m, b, True, monkeypatch)
    assert la == lb
    m.zero_grad()
    torch.manual_seed(12)
    assert float(m(b, training=True)[0]) != la


def test_bf16_autocast_gradients_meet_the_cosine_bound(monkeypatch):
    """The models and bound of test_amp_train_gpu (ReaRev D = 50 and 200, NSM with reason_kb), here with the question
    side asserted to run in the kernels: dropout layers off, every gradient above 1e-6 of the largest has cosine
    >= 0.98 with fp32, and the loss agrees within 2e-2."""
    assert autograd_path._instruction_kernels(torch.device(DEV), 10, 200, 2)
    for name, over in [v for v in AMP.MODELS.values() if v[0] != "GraftNet"]:
        m = _model(name, **over).train()
        for mod in m.modules():
            if isinstance(mod, torch.nn.Dropout):
                mod.eval()
        b = _batch()
        l32, g32 = _grads(m, b, True, monkeypatch)
        l16, g16 = _grads(m, b, True, monkeypatch, amp=True)
        assert abs(l16 - l32) <= 2e-2 * abs(l32)
        gmax = max(float(g.norm()) for g in g32.values())
        for k, g in g32.items():
            if float(g.norm()) > 1e-6 * gmax and not k.endswith("score_func.bias"):
                cos = float(torch.nn.functional.cosine_similarity(g16[k].flatten(), g.flatten(), dim=0, eps=1e-30))
                assert cos >= 0.98, (name, k, cos)


def test_deterministic_mode_with_dropout_is_bit_identical(monkeypatch):
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        for name, over in E2E.values():
            m = _model(name, linear_dropout=0.2, **over).train()
            b = _batch()
            la, ga = _grads(m, b, True, monkeypatch)
            lb, gb = _grads(m, b, True, monkeypatch)
            assert la == lb and all(torch.equal(ga[k], gb[k]) for k in ga), name
    finally:
        torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])


def test_three_adam_steps_through_the_train_epoch_call_sequence():
    """zero_grad, model(batch, training=True), backward, clip_grad_norm_, step (train_model.py:209-233), dropout on."""
    for name, over in E2E.values():
        m = _model(name, linear_dropout=0.2, **over).train()
        b = _batch()
        params = [p for p in m.parameters() if p.requires_grad]
        opt = torch.optim.Adam(params, lr=1e-3)
        for _ in range(3):
            opt.zero_grad()
            loss, _pred, _dist, tp_list = m(b, training=True)
            loss.backward()
            torch.nn.utils.clip_grad_norm_(params, 1.0)
            opt.step()
            assert torch.isfinite(loss).all()
        assert all(torch.isfinite(p).all() for p in m.parameters())
        assert m.instruction.question_linear0.weight.grad is not None
