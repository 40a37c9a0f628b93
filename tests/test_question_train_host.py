"""Host side of the question-side training kernels: the float64 restatements of their backward
(tests/question_train_ref.py) against torch.autograd, the numpy Philox restatement of the dropout key, and which path
``autograd_path`` dispatches to."""
import numpy as np
import pytest
import torch

from gnn_rag_b200 import autograd_path

import question_train_ref as QT

F64 = torch.float64


def _ins_case(seed, B, Q, D, I, p):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, sc=1.0: (torch.randn(*s, generator=g, dtype=F64) * sc).requires_grad_(True)   # noqa: E731
    t = dict(hidden=r(B, Q, D, sc=0.5), qnode=r(B, D, sc=0.5), Wq=[r(D, D, sc=D ** -0.5) for _ in range(I)],
             bq=[r(D, sc=0.1) for _ in range(I)], Wcq=r(D, 4 * D, sc=(4 * D) ** -0.5), bcq=r(D, sc=0.1),
             wca=r(1, D, sc=D ** -0.5), bca=r(1, sc=0.1))
    qmask = torch.ones(B, Q, dtype=F64)
    if Q > 2:
        qmask[0, Q // 2] = 0.0
    if B > 1:
        qmask[B - 1] = 0.0                                                   # an all-pad question
    masks = None
    if p > 0:
        rs = np.random.RandomState(seed)
        masks = [rs.rand(B, I, D) >= p, rs.rand(B, I, 4 * D) >= p, rs.rand(B, I, Q, D) >= p]
    return t, qmask, masks


@pytest.mark.parametrize("B,Q,D,I,p", [(3, 5, 4, 1, 0.0), (3, 7, 6, 3, 0.0), (2, 4, 5, 2, 0.3), (3, 6, 3, 4, 0.5)])
def test_instructions_backward_restatement_matches_autograd(B, Q, D, I, p):
    t, qmask, masks = _ins_case(B * 100 + Q * 10 + D + I, B, Q, D, I, p)
    ri, attn = QT.instructions_fwd(t["hidden"], t["qnode"], qmask, t["Wq"], t["bq"], t["Wcq"], t["bcq"], t["wca"],
                                   t["bca"], masks, p)
    G = torch.randn(B, I, D, dtype=F64, generator=torch.Generator().manual_seed(1))
    (ri * G).sum().backward()
    vals, mag = QT.instructions_backward(t["hidden"].detach(), t["qnode"].detach(), [w.detach() for w in t["Wq"]],
                                         [b.detach() for b in t["bq"]], t["Wcq"].detach(), t["bcq"].detach(),
                                         t["wca"].detach(), ri.detach(), attn.detach(), G, masks, p)
    close = lambda a, b: torch.testing.assert_close(a, b, rtol=1e-10, atol=1e-12)   # noqa: E731
    close(vals["grad_hidden"], t["hidden"].grad)
    close(vals["grad_qnode"], t["qnode"].grad)
    for i in range(I):                                                   # grad_W = G^T X, grad_b = sum G
        close(vals["g_q"][:, i].t() @ vals["x_q"][:, i], t["Wq"][i].grad)
        close(vals["g_q"][:, i].sum(0), t["bq"][i].grad)
    close(vals["g_cq"].reshape(-1, D).t() @ vals["x_cq"].reshape(-1, 4 * D), t["Wcq"].grad)
    close(vals["g_cq"].reshape(-1, D).sum(0), t["bcq"].grad)
    close(vals["g_ca"].reshape(1, -1) @ vals["x_ca"].reshape(-1, D), t["wca"].grad)
    close(vals["g_ca"].sum().reshape(1), t["bca"].grad)
    for k, v in vals.items():                                            # the magnitude bounds every value
        assert (v.abs() <= mag[k] * (1 + 1e-12) + 1e-300).all(), k


@pytest.mark.parametrize("B,N,D,I", [(3, 7, 4, 1), (4, 9, 5, 3), (2, 3, 2, 8)])
def test_reform_backward_restatement_matches_autograd(B, N, D, I):
    g = torch.Generator().manual_seed(B * 100 + N + D + I)
    seed = torch.zeros(B, N, dtype=F64)
    seed[0, 1] = 1.0
    seed[1, [0, N - 1]] = torch.tensor([0.3, 0.7], dtype=F64)
    if B > 2:
        seed[2] = torch.rand(N, generator=g, dtype=F64)                  # dense
    h = torch.randn(B * N, D, generator=g, dtype=F64).requires_grad_(True)
    ins = torch.randn(B, I, D, generator=g, dtype=F64).requires_grad_(True)
    Wr = [(torch.randn(D, 3 * D, generator=g, dtype=F64) * 0.3).requires_grad_(True) for _ in range(I)]
    Wg = [(torch.randn(D, 3 * D, generator=g, dtype=F64) * 0.3).requires_grad_(True) for _ in range(I)]
    G = torch.randn(B, I, D, generator=g, dtype=F64)
    (QT.reform_fwd(seed, h, ins, Wr, Wg, B, N) * G).sum().backward()
    res = QT.reform_backward(seed, h.detach(), ins.detach(), [w.detach() for w in Wr], [w.detach() for w in Wg], B, N, G)
    close = lambda a, b: torch.testing.assert_close(a, b, rtol=1e-10, atol=1e-12)   # noqa: E731
    close(res["grad_ins"], ins.grad)
    close(res["grad_h"], h.grad)
    assert (res["grad_h"].view(B, N, D)[seed == 0] == 0).all()             # only seed rows
    for j in range(I):
        close(res["g_r"][:, j].t() @ res["x_z"][:, j], Wr[j].grad)
        close(res["g_g"][:, j].t() @ res["x_z"][:, j], Wg[j].grad)


def test_philox_restatement_known_answers():
    """Philox4x32-10 known-answer vectors of the Random123 distribution (kat_vectors)."""
    cases = [((0, 0), (0, 0, 0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
             ((0xFFFFFFFF, 0xFFFFFFFF), (0xFFFFFFFF,) * 4, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
             ((0xA4093822, 0x299F31D0), (0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344),
              (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for key, ctr, want in cases:
        assert tuple(int(x) for x in QT.philox4x32_10(key, ctr)) == want


def test_dropout_key_follows_the_documented_formula():
    """ins_keep is the header's formula: counter (b, 4 i + site, q, c), key = the 64-bit seed split low / high, the
    first word's top 24 bits as u in [0, 1), kept iff u >= p; the masks index it as documented."""
    seed = (0x1234567 << 32) | 0x89ABCDEF
    x0 = QT.philox4x32_10((0x89ABCDEF, 0x1234567), (2, 4 * 3 + 1, 0, 17))[0]
    u = float(np.float32(int(x0) >> 8) * np.float32(2.0 ** -24))
    for p in (0.1, 0.5, u, np.nextafter(np.float32(u), np.float32(1))):
        assert bool(QT.ins_keep(seed, p, 2, 3, 1, 0, 17)) == (np.float32(u) >= np.float32(p))
    m0, m1, m2 = QT.ins_masks(seed, 0.4, 3, 5, 7, 4)
    assert m0.shape == (3, 4, 7) and m1.shape == (3, 4, 28) and m2.shape == (3, 4, 5, 7)
    assert m1[2, 3, 17] == QT.ins_keep(seed, 0.4, 2, 3, 1, 0, 17)
    assert m2[1, 2, 4, 6] == QT.ins_keep(seed, 0.4, 1, 2, 2, 4, 6)
    assert m0[0, 1, 5] == QT.ins_keep(seed, 0.4, 0, 1, 0, 0, 5)
    assert abs(m2.mean() - 0.6) < 0.05


def test_dispatch_takes_the_torch_path_for_cpu_refused_shapes_and_use_kernels_off(monkeypatch):
    cuda, cpu = torch.device("cuda"), torch.device("cpu")
    assert autograd_path._instruction_kernels(cuda, 20, 50, 3)
    assert autograd_path._reform_kernels(cuda, 50, 3)
    assert not autograd_path._instruction_kernels(cpu, 20, 50, 3)
    assert not autograd_path._reform_kernels(cpu, 50, 3)
    assert not autograd_path._instruction_kernels(cuda, 20, 50, 9)             # I <= 8
    assert not autograd_path._reform_kernels(cuda, 50, 9)
    D, I = 200, 2
    q_max = (200 * 1024 // 4 - (I + 7) * D) // (D + 2)                           # gr_instructions' 200 KB check
    assert autograd_path._instruction_kernels(cuda, q_max, D, I)
    assert not autograd_path._instruction_kernels(cuda, q_max + 1, D, I)
    assert autograd_path._reform_kernels(cuda, 1024, 1) and not autograd_path._reform_kernels(cuda, 1025, 1)
    d_max = 48 * 1024 // (4 * (5 * 3 + 1))                                        # (5I+1) D floats <= 48 KB
    assert autograd_path._reform_kernels(cuda, d_max, 3) and not autograd_path._reform_kernels(cuda, d_max + 1, 3)
    monkeypatch.setattr(autograd_path, "USE_KERNELS", False)
    assert not autograd_path._instruction_kernels(cuda, 20, 50, 3)
    assert not autograd_path._reform_kernels(cuda, 50, 3)


def test_cpu_model_under_host_check_runs_the_torch_question_side(monkeypatch):
    """A CPU model (HOST_CHECK) never reaches the kernel Functions."""
    import gnn_rag_b200 as G
    from gnn_rag_b200 import synthetic as S
    monkeypatch.setattr(autograd_path, "HOST_CHECK", True)
    called = []
    monkeypatch.setattr(autograd_path._InstructionsFn, "apply", lambda *a: called.append(1))
    monkeypatch.setattr(autograd_path._QueryReformFn, "apply", lambda *a: called.append(2))
    torch.manual_seed(0)
    m = G.ReaRev(S.model_args("ReaRev", entity_dim=16, num_iter=2, num_ins=2, num_gnn=1, word_dim=8,
                              use_cuda=False, linear_dropout=0.2), 200, 10, 30).train()
    b = S.make_batch(1, B=2, N=20, E=40, num_entity=200, num_relation=10, num_word=30)
    loss = m(b, training=True)[0]
    loss.backward()
    assert not called
