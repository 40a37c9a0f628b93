"""CPU: the capture key and the refusals of graphed.GraphedGraftTrainStep, and that GraphedTrainStep keeps refusing
GraftNet.  The GPU half is tests/test_graphed_graft_train_gpu.py."""
import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import autograd_path, graphed, synthetic as S

NE, NR, NW = 3000, 40, 100


def _unbuilt_step(model, device="cpu"):
    """A GraphedGraftTrainStep over a CPU model, built past the constructor's device refusal: its key and refusal
    logic run on the host and capture nothing."""
    st = object.__new__(graphed.GraphedGraftTrainStep)
    st.model, st._params, st.device = model, list(model.parameters()), torch.device(device)
    st.max_graphs, st._cache = 8, {}
    st._layout = graphed._GraftLayout(st)
    return st


def _model(D=16, **over):
    torch.manual_seed(0)
    return G.GraftNet(dict(S.model_args("GraftNet", entity_dim=D, use_cuda=False, **over)), NE, NR, NW).train()


def _batch(seed=1, E=300, Q=12, N=60):
    return S.make_graft_batch(seed, B=3, N=N, E=E, num_entity=NE, num_relation=NR, num_word=NW, Q=Q)


def test_exported_beside_graphed_train_step():
    assert G.GraphedGraftTrainStep is graphed.GraphedGraftTrainStep
    assert "GraphedGraftTrainStep" in G.__all__
    assert issubclass(graphed.GraphedGraftTrainStep, graphed.GraphedTrainStep)


def test_constructor_refusals():
    with pytest.raises(ValueError, match="covers ReaRev and NSM; GraftNet"):
        graphed.GraphedTrainStep(_model())
    with pytest.raises(ValueError, match="GraphedGraftTrainStep needs a model on a CUDA device"):
        graphed.GraphedGraftTrainStep(_model())
    rearev = G.ReaRev(dict(S.model_args("ReaRev", entity_dim=16, use_cuda=False)), NE, NR, NW)
    with pytest.raises(ValueError, match="GraphedGraftTrainStep covers GraftNet"):
        graphed.GraphedGraftTrainStep(rearev)


def test_refusal_names_the_kernel_condition():
    assert _unbuilt_step(_model(16), "cuda").refusal(12) is None
    assert _unbuilt_step(_model(512), "cuda").refusal(300) is None      # the question length does not matter
    why = _unbuilt_step(_model(513), "cuda").refusal(12)
    assert why == "_fact_kernels is false: entity_dim 513 is outside the GraftNet training kernels (D <= 512)"
    assert _unbuilt_step(_model(16), "cpu").refusal(12).startswith("_fact_kernels is false")
    old = autograd_path.USE_KERNELS
    autograd_path.USE_KERNELS = False
    try:
        assert "USE_KERNELS is off" in _unbuilt_step(_model(16), "cuda").refusal(12)
    finally:
        autograd_path.USE_KERNELS = old


def test_a_kb_tuple_is_refused():
    st = _unbuilt_step(_model())
    kb = S.make_batch(1, B=3, N=60, E=300, num_entity=NE, num_relation=NR, num_word=NW)[:7]
    with pytest.raises(ValueError, match="9/10-tuple of GraftSingleDataLoader.get_batch, not a 7-tuple"):
        st.key(kb)


def _trim_graft(batch, n):
    """``batch`` with only the first n head-list graft facts and their tail-list partners (same kb facts, same
    ``kb_fact_rel`` shape)."""
    (hb, hf, he, hv), (tb, te, tf, tv) = batch[3]
    slots = set(zip(hb[:n].tolist(), hf[:n].tolist()))
    tk = np.array([(b, f) in slots for b, f in zip(tb.tolist(), tf.tolist())], dtype=bool)
    out = list(batch)
    out[3] = ((hb[:n], hf[:n], he[:n], np.asarray(hv)[:n]), (tb[tk], te[tk], tf[tk], np.asarray(tv)[tk]))
    return tuple(out)


def test_capture_key_rules():
    m = _model()
    st = _unbuilt_step(m)
    b = _batch(E=2000)
    k0 = st.key(b)
    n = len(b[3][0][0])
    assert n > 2048
    assert st.key(_trim_graft(b, n - 10)) == k0                 # another graft count of the same bucket
    assert st.key(_trim_graft(b, n // 3)) != k0                 # another graft-capacity bucket
    assert st.key(b + (None,)) == k0                            # the 10-tuple of get_batch(test=True)
    assert st.key(_batch(2, E=2000, N=70)) != k0                # another max_fact / N
    assert st.key(_batch(1, E=2000, Q=9)) != k0                 # another question length
    layer = m.reasoning
    layer.pagerank_lambda = 0.5
    k1 = st.key(b)
    assert k1 != k0
    layer.fact_scale = 2
    assert st.key(b) != k1
    layer.pagerank_lambda, layer.fact_scale = 0.8, 3
    assert st.key(b) == k0
    m.reasoning.linear_drop_train.p = 0.5
    assert st.key(b) != k0
    m.reasoning.linear_drop_train.p = 0.2
    assert st.key(b) == k0
    p = m.type_layer.kb_self_linear.weight                      # a replaced storage recaptures
    p.data = p.data.clone()
    assert st.key(b) != k0
    m.eval()
    assert st.key(b)[7] is False
    m.add_module("extra", torch.nn.Linear(2, 2))
    with pytest.raises(ValueError, match="parameters changed"):
        st.key(b)
