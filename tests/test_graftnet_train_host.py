"""GraftNet training without a GPU: the float64 restatement the GPU kernel tests hold the kernels against
(tests/graft_train_ref.py) agrees with ``model(batch, training=True)``'s per-fact restatement on a reference golden,
and the new training entry points refuse null pointers and bad sizes with status codes."""
import numpy as np
import pytest
import torch

from gnn_rag_b200 import _lib, autograd_path
from graft_train_ref import graftnet_fp64
from test_graftnet_host import load_model


@pytest.fixture
def host_check():
    old = autograd_path.HOST_CHECK
    autograd_path.HOST_CHECK = True
    yield
    autograd_path.HOST_CHECK = old


@pytest.mark.parametrize("name", ["graft_small", "graft_hub_clamp"])
def test_fp64_restatement_agrees_with_the_training_forward(name, host_check):
    """Same logits' softmax, PageRank history and parameter gradients (of a fixed functional of pred_dist) as
    graftnet_forward, to fp32 rounding: the restatement moves kb_tail_linear after the per-node sum by linearity."""
    m, g = load_model(name)
    rs = np.random.RandomState(0)
    _loss, _pred, pred_dist, _tp = m(g.batch, training=True)
    wsum = torch.tensor(rs.randn(*pred_dist.shape), dtype=torch.float32)
    (pred_dist * wsum).sum().backward()
    got = {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}
    pr_got = torch.stack(m.pagerank_history[1:])
    m.zero_grad()
    logit, pr = graftnet_fp64(m, g.batch)
    mask = torch.as_tensor(g.batch[0] != 1000).double()
    ref = torch.softmax(logit + (1 - mask) * -1e11, dim=1)
    (ref * wsum.double()).sum().backward()
    assert (pred_dist.detach().double() - ref.detach()).abs().max() <= 1e-5 * ref.detach().abs().max()
    assert (pr_got.detach().double() - pr.detach()).abs().max() <= 1e-5 * pr.detach().abs().max()
    # 1e-4 of the tensor's scale plus 1e-6 of the model's largest gradient: the score bias has a mathematically zero
    # gradient (softmax is shift invariant), both sides hold rounding noise there
    gmax = max(float(p.grad.abs().max()) for p in m.parameters() if p.grad is not None)
    checked = 0
    for k, p in m.named_parameters():
        if k not in got:
            continue
        want = p.grad
        assert want is not None, k
        assert (got[k] - want).abs().max() <= 1e-4 * want.abs().max() + 1e-6 * gmax, k
        checked += 1
    assert checked >= 15


def test_fact_kernels_cover_d_up_to_512_on_cuda_only():
    """Wider models and CPU tensors keep the per-fact torch ops of the training path."""
    cuda, cpu = torch.device("cuda"), torch.device("cpu")
    assert autograd_path._fact_kernels(cuda, 1) and autograd_path._fact_kernels(cuda, 512)
    assert not autograd_path._fact_kernels(cuda, 513) and not autograd_path._fact_kernels(cpu, 64)
    old = autograd_path.USE_KERNELS
    autograd_path.USE_KERNELS = False
    try:
        assert not autograd_path._fact_kernels(cuda, 64)
    finally:
        autograd_path.USE_KERNELS = old


def test_training_on_a_batch_without_graft_facts_on_the_host(host_check):
    """The per-fact restatement trains on a batch without graft facts (the GPU test holds the kernel path to it)."""
    import gnn_rag_b200 as G
    from gnn_rag_b200 import synthetic as S
    m = G.GraftNet(S.model_args("GraftNet", entity_dim=16, num_layer=2, linear_dropout=0.0), 100, 10, 20)
    b = list(S.make_graft_batch(4, B=3, N=20, E=60, num_entity=100, num_relation=10, num_word=20))
    z = np.zeros(0, dtype=np.int64)
    b[3] = ((z, z, z, np.ones(0)), (z, z, z, np.ones(0)))
    loss = m(tuple(b), training=True)[0]
    loss.backward()
    assert torch.isfinite(loss) and float(loss) > 0


def test_training_entry_points_refuse_bad_arguments():
    L = _lib.load()
    x = 256        # a non-null address: every call below must be refused before anything is dereferenced
    assert L.gr_graft_dropout_mask(None, 0.5, 10, 8, x, None) == -1 and b"seed" in L.gr_last_error()
    assert L.gr_graft_dropout_mask(x, 1.0, 10, 8, x, None) == -1
    assert L.gr_graft_dropout_mask(x, 0.5, 10, 0, x, None) == -1
    assert L.gr_graft_dropout_mask(x, 0.5, 10, 8, None, None) == -1
    assert L.gr_graft_dropout_mask(None, 0.0, 0, 8, None, None) == 0                      # nothing to do
    args = [x] * 7 + [8, x, 8, None, 0.0, x, 8, 1, 2, 8, None]
    for i in range(7):
        bad = list(args)
        bad[i] = None
        assert L.gr_graft_aggregate_train(*bad) == -1 and b"null" in L.gr_last_error()
    for i, v in ((7, 4), (9, 4), (13, 4), (16, 513), (16, 0), (14, 0), (11, -0.1), (11, 1.0)):
        bad = list(args)
        bad[i] = v
        assert L.gr_graft_aggregate_train(*bad) == -1, (i, v)
    bad = list(args)
    bad[11] = 0.2                                                                          # p > 0 without a seed
    assert L.gr_graft_aggregate_train(*bad) == -1 and b"seed" in L.gr_last_error()
    bargs = [x] * 7 + [8, x, 8, None, 0.0, x, 8, x, x, 8, x, 8, 1, 2, 8, None]
    for i in (0, 1, 2, 3, 4, 5, 6, 8, 12, 14, 15, 17):
        bad = list(bargs)
        bad[i] = None
        assert L.gr_graft_aggregate_backward(*bad) == -1, i
    for i, v in ((7, 4), (13, 4), (16, 4), (18, 4), (21, 600)):
        bad = list(bargs)
        bad[i] = v
        assert L.gr_graft_aggregate_backward(*bad) == -1, (i, v)
    aargs = [x, x, 4, x, 8, 3, x, 1, 5, 8, x, x, x, 8, None]
    for i in (0, 1, 3, 6, 10, 11, 12):
        bad = list(aargs)
        bad[i] = None
        assert L.gr_graft_attention_backward(*bad) == -1, i
    for i, v in ((2, 0), (4, 4), (5, 0), (7, 0), (7, 70000), (9, 513), (13, 4)):
        bad = list(aargs)
        bad[i] = v
        assert L.gr_graft_attention_backward(*bad) == -1, (i, v)
    targs = [x, x, None, x, x, None, x, 8, x, 8, x, 8, 1, 2, 8, 5, None]
    for i in (0, 1, 3, 4, 6, 8, 10):
        bad = list(targs)
        bad[i] = None
        assert L.gr_type_layer_backward(*bad) == -1, i
    for i, v in ((7, 4), (9, 4), (11, 4), (14, 0), (14, 513), (15, -1), (12, 0)):
        bad = list(targs)
        bad[i] = v
        assert L.gr_type_layer_backward(*bad) == -1, (i, v)
