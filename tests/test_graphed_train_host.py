"""CPU: the C declaration and ctypes binding of gr_train_metrics and its refusals, the capture key and the refusals of
graphed.GraphedTrainStep, and a numpy restatement of what gr_train_metrics computes (csrc/rank.cu) held against
autograd_path.eval_metric on CPU tensors (``HOST_CHECK``).  The GPU half is tests/test_graphed_train_gpu.py."""
import ctypes

import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import _lib, autograd_path, graphed, ops, synthetic as S

NE, NR, NW = 3000, 40, 100


# ---- the entry point --------------------------------------------------------------------------------------------------

def test_header_declaration_and_binding():
    res, args = _lib.SIGNATURES["gr_train_metrics"]
    P, I64, I = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    assert res is ctypes.c_int
    assert args == [P, P, P, P, I64, P, P, P, P, I, I, P]
    assert _lib.load().gr_train_metrics.argtypes == args


def _call(**over):
    lib = _lib.load()
    a = dict(pred_dist=0x1000, answer_dist=0x1000, seed_dist=0x1000, local_entity=0x1000, pad_id=7, cand_idx=0x1000,
             cand_count=0x1000, h1=0x1000, f1=0x1000, B=2, N=3, stream=None)
    a.update(over)
    rc = lib.gr_train_metrics(*a.values())
    return rc, lib.gr_last_error().decode()


@pytest.mark.parametrize("over,msg", [
    (dict(pred_dist=None), "null pointer"), (dict(cand_count=None), "null pointer"), (dict(f1=None), "null pointer"),
    (dict(B=0), "B and N must be positive"), (dict(N=0), "B and N must be positive"),
    (dict(N=-1), "B and N must be positive")])
def test_entry_point_refusals(over, msg):
    assert _call(**over) == (-1, "gr_train_metrics: invalid argument: " + msg)


def test_shape_rule_matches_the_entry_point():
    for B, N in [(1, 1), (0, 3), (2, 0), (64, 2000)]:
        assert ops.train_metrics_ok(B, N) == (B > 0 and N > 0)


def test_wrapper_refuses_cpu_tensors():
    z = torch.zeros(2, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.train_metrics(z, z, z, z.long(), z.int(), torch.zeros(2, dtype=torch.int32), 7)


# ---- GraphedTrainStep: refusals and the capture key --------------------------------------------------------------------

def test_refuses_graftnet_and_cpu_models():
    graft = G.GraftNet(dict(S.model_args("GraftNet", entity_dim=16, use_cuda=False)), NE, NR, NW)
    with pytest.raises(ValueError, match="covers ReaRev and NSM; GraftNet"):
        graphed.GraphedTrainStep(graft)
    cpu = G.ReaRev(dict(S.model_args("ReaRev", entity_dim=16, use_cuda=False)), NE, NR, NW)
    with pytest.raises(ValueError, match="needs a model on a CUDA device"):
        graphed.GraphedTrainStep(cpu)


def _unbuilt_step(model, device="cpu"):
    """A GraphedTrainStep over a CPU model, built past the constructor's device refusal: its key and refusal logic run
    on the host and capture nothing."""
    st = object.__new__(graphed.GraphedTrainStep)
    st.model, st._params, st.device = model, list(model.parameters()), torch.device(device)
    st.max_graphs, st._cache = 8, {}
    st._layout = graphed._KbLayout(st)
    return st


def _model(D=16, name="ReaRev", **over):
    torch.manual_seed(0)
    cls = G.ReaRev if name == "ReaRev" else G.NSM
    return cls(dict(S.model_args(name, entity_dim=D, use_cuda=False, **over)), NE, NR, NW).train()


def _batch(seed=1, E=300, Q=12):
    return S.make_batch(seed, B=3, N=60, E=E, num_entity=NE, num_relation=NR, num_word=NW, Q=Q,
                        with_weights=False)[:7]


def test_refusal_names_the_kernel_condition():
    assert _unbuilt_step(_model(16), "cuda").refusal(12) is None
    assert _unbuilt_step(_model(16, "NSM"), "cuda").refusal(12) is None
    why = _unbuilt_step(_model(264), "cuda").refusal(12)
    assert why.startswith("_kernel_graph is None: entity_dim 264 with 2 instruction(s)")
    why = _unbuilt_step(_model(16, num_ins=5), "cuda").refusal(12)
    assert why.startswith("_kernel_graph is None: entity_dim 16 with 5 instruction(s)")
    why = _unbuilt_step(_model(200), "cuda").refusal(300)
    assert why.startswith("_instruction_kernels is false: 300 question tokens")
    old = autograd_path.USE_KERNELS
    autograd_path.USE_KERNELS = False
    try:
        assert "USE_KERNELS is off" in _unbuilt_step(_model(16), "cuda").refusal(12)
    finally:
        autograd_path.USE_KERNELS = old


def test_capture_key_rules():
    m = _model()
    st = _unbuilt_step(m)
    b = _batch()
    k0 = st.key(b)
    assert st.key(_batch(2, E=300)) == k0                     # another batch of the same bucket: the same graph
    assert st.key(_batch(2, E=1000)) != k0                    # another fact-capacity bucket
    assert st.key(_batch(2, Q=9)) != k0                       # another question length
    opt = torch.optim.Adam(m.parameters(), lr=1e-2)          # in-place updates keep the key ...
    for p in m.parameters():
        p.grad = torch.ones_like(p)
    opt.step()
    m.load_state_dict({k: v + 1 for k, v in m.state_dict().items()})
    assert st.key(b) == k0
    p = m.entity_linear.weight                                # ... a replaced storage changes it
    p.data = p.data.clone()
    k1 = st.key(b)
    assert k1 != k0
    m.eval()
    assert st.key(b) != k1
    m.train()
    assert st.key(b) == k1
    m.reasoning.linear_drop_train.p = 0.5 if m.reasoning.linear_drop_train.p != 0.5 else 0.25
    k2 = st.key(b)
    assert k2 != k1
    m.entity_linear.bias.requires_grad_(False)               # another set of trainable parameters: recapture
    assert st.key(b) != k2
    m.entity_linear.bias.requires_grad_(True)
    assert st.key(b) == k2
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(not prev, warn_only=True)
    try:
        assert st.key(b) != k2
    finally:
        torch.use_deterministic_algorithms(prev)
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=not torch.backends.cudnn.allow_tf32):
        assert st.key(b) != k2
    m.add_module("extra", torch.nn.Linear(2, 2))
    with pytest.raises(ValueError, match="parameters changed"):
        st.key(b)


# ---- the metric semantics ----------------------------------------------------------------------------------------------

def metrics_np(pred_dist, answer_dist, seed_dist, local_entity, cand_idx, cand_count, pad_id):
    """What gr_train_metrics computes, per question: hit@1 at the first maximal index (NaN counts as maximal), and for
    hit@1 questions the F1 of the first cand_count candidates against the answer list matched by entity id."""
    B, N = pred_dist.shape
    h1, f1 = np.zeros(B, np.float32), np.zeros(B, np.float32)
    for b in range(B):
        p = pred_dist[b]
        nan = np.isnan(p)
        top = int(np.argmax(nan)) if nan.any() else int(np.argmax(p))
        if not answer_dist[b, top] > np.float32(1e-10):
            continue
        h1[b] = 1.0
        ok = (answer_dist[b] > 0) & ~(seed_dist[b] > 0) & (local_entity[b] != pad_id)
        answers = local_entity[b][ok]
        c = int(cand_count[b])
        k = sum(int(local_entity[b, i] in set(answers.tolist())) for i in cand_idx[b, :c])
        if len(answers) == 0:
            v = 1.0 if c == 0 else 0.0
        elif c == 0 or k == 0:
            v = 0.0
        else:
            v = 2.0 / (1.0 / (k / c) + 1.0 / (k / len(answers)))
        f1[b] = np.float32(v)
    return h1, f1


def edge_batch():
    """Eight questions of N = 8 (pad id 99), each one edge case of get_eval_metric:
    (pred_dist, answer_dist, seed_dist, local_entity, pad)."""
    B, N, pad = 8, 8, 99
    le = np.tile(np.arange(10, 10 + N), (B, 1)).astype(np.int64)
    sd = np.zeros((B, N), np.float32)
    sd[:, 0] = 1.0
    ad = np.zeros((B, N), np.float32)
    pd = np.full((B, N), 0.01, np.float32)
    ad[0, [2, 5]] = 0.5; pd[0, 2] = 0.9                       # hit, one of two answers retrieved
    ad[1, 0] = 1.0; pd[1, 0] = 0.9                            # answer mass on the seed only: candidates, no answers
    ad[2, 1:] = 1.0 / (N - 1); pd[2, 1:] = 1.0 / (N - 1); pd[2, 0] = 0.0   # every candidate correct
    ad[3, 4] = 1.0; pd[3, 6] = 0.9                            # hit@1 = 0
    ad[4, 3] = 1.0; pd[4, 3] = 0.4; pd[4, 6] = 0.4            # tie at the maximum: the first index (an answer)
    le[5, 6] = le[5, 2]; ad[5, 2] = 1.0; pd[5, 2] = 0.45; pd[5, 6] = 0.45  # a repeated entity id, both retrieved
    le[6, 3] = pad; ad[6, 3] = 1.0; pd[6] = 0.0; pd[6, 3] = 1.0  # all mass on a pad answer: no answers, no candidates
    ad[7, [0, 4]] = 0.5; pd[7, 4] = 0.9                       # the other answer node is a seed
    return pd, ad, sd, le, pad


EDGE_H1 = [1.0, 1.0, 1.0, 0.0, 1.0, 1.0, 1.0, 1.0]


def _check_host(pd, ad, sd, le, pad, eps=0.95):
    old = autograd_path.HOST_CHECK
    autograd_path.HOST_CHECK = True
    try:
        t = torch.from_numpy
        h1, f1 = autograd_path.eval_metric(type("M", (), dict(num_entity=pad, eps=eps)), t(pd), t(ad), t(sd), t(le))
        ci, cc = autograd_path._retrieved_sets_host(t(pd), t(le), (t(sd) > 0).float(), pad, eps)
    finally:
        autograd_path.HOST_CHECK = old
    h1n, f1n = metrics_np(pd, ad, sd, le, ci.numpy(), cc.numpy(), pad)
    assert h1.numpy().tobytes() == h1n.tobytes()
    assert f1.numpy().tobytes() == f1n.tobytes()
    return h1n.tolist(), f1n.tolist()


def test_restatement_matches_eval_metric_on_the_edge_cases():
    pd, ad, sd, le, pad = edge_batch()
    h1, f1 = _check_host(pd, ad, sd, le, pad)
    assert h1 == EDGE_H1
    assert f1[1] == 0.0 and f1[2] == 1.0 and f1[3] == 0.0 and f1[6] == 1.0
    for b in range(len(h1)):                                  # B = 1
        _check_host(pd[b:b + 1], ad[b:b + 1], sd[b:b + 1], le[b:b + 1], pad)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_restatement_matches_eval_metric_on_random_batches(seed):
    rs = np.random.RandomState(seed)
    B, N, pad = 16, 120, 500
    le = rs.randint(0, 60, size=(B, N)).astype(np.int64)     # repeated ids
    le[rs.rand(B, N) < 0.2] = pad
    sd = (rs.rand(B, N) < 0.03).astype(np.float32)
    ad = (rs.rand(B, N) < 0.1).astype(np.float32) * rs.rand(B, N).astype(np.float32)
    logits = rs.randn(B, N).astype(np.float32) * 2 + 3 * (ad > 0)
    pd = np.exp(logits - logits.max(1, keepdims=True)).astype(np.float32)
    pd /= pd.sum(1, keepdims=True)
    h1, _ = _check_host(pd, ad, sd, le, pad)
    assert 0 < sum(h1)
