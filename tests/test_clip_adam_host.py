"""optim's host side without a GPU: what the fused clip + Adam step refuses, the per-step scalars against a restatement
of torch's host arithmetic in ``_multi_tensor_adam``, the state it creates against ``Adam._init_group``, and the
state key ``load_state_dict`` changes."""
import copy
import math

import numpy as np
import pytest
import torch

from gnn_rag_b200 import graphed, optim


def _params(n=3, dtype=torch.float32):
    torch.manual_seed(0)
    return [torch.nn.Parameter(torch.randn(4 + i, 3, dtype=dtype)) for i in range(n)]


@pytest.mark.parametrize("make,msg", [
    (lambda ps: torch.optim.SGD(ps, lr=0.1), "torch.optim.Adam"),
    (lambda ps: torch.optim.AdamW(ps), "torch.optim.Adam"),
    (lambda ps: torch.optim.Adamax(ps), "torch.optim.Adam"),
    (lambda ps: torch.optim.Adam(ps, amsgrad=True), "amsgrad"),
    (lambda ps: torch.optim.Adam(ps, maximize=True), "maximize"),
    (lambda ps: torch.optim.Adam(ps, decoupled_weight_decay=True), "decoupled_weight_decay"),
    (lambda ps: torch.optim.Adam(ps, capturable=True), "capturable"),
    (lambda ps: torch.optim.Adam(ps, differentiable=True), "differentiable"),
    (lambda ps: torch.optim.Adam(ps, lr=torch.tensor(1e-3)), "float lr"),
    (lambda ps: torch.optim.Adam([ps[0], torch.nn.Parameter(torch.zeros(2))]), "not the model's"),
])
def test_optimizer_refusals(make, msg):
    ps = _params()
    with pytest.raises(ValueError, match=msg):
        optim.check_optimizer(make(ps), ps, 1.0)


def test_fused_adam_is_refused():
    ps = _params()
    opt = torch.optim.Adam(ps)
    opt.param_groups[0]["fused"] = True          # a CPU Adam(fused=True) cannot be built without a GPU
    with pytest.raises(ValueError, match="fused"):
        optim.check_optimizer(opt, ps, None)


def test_non_fp32_parameters_are_refused():
    ps = _params(dtype=torch.float64)
    with pytest.raises(ValueError, match="fp32"):
        optim.check_optimizer(torch.optim.Adam(ps), ps, None)


@pytest.mark.parametrize("max_norm", [0.0, -1.0, float("nan")])
def test_max_norm_must_be_positive(max_norm):
    ps = _params()
    with pytest.raises(ValueError, match="max_norm"):
        optim.check_optimizer(torch.optim.Adam(ps), ps, max_norm)


def test_max_norm_needs_an_optimizer():
    with pytest.raises(ValueError, match="needs an optimizer"):
        optim.check_optimizer(None, _params(), 1.0)


def test_admitted_configurations():
    ps = _params()
    optim.check_optimizer(None, ps, None)
    optim.check_optimizer(torch.optim.Adam(ps), ps, None)
    optim.check_optimizer(torch.optim.Adam(ps[:2], weight_decay=0.01, foreach=True), ps, 1.0)
    optim.check_optimizer(torch.optim.Adam([dict(params=ps[:1]), dict(params=ps[1:], lr=1e-2, betas=(0.8, 0.9))]),
                          ps, 0.5)


def test_graphed_steps_refuse_a_cpu_model_before_the_optimizer():
    m = torch.nn.Linear(3, 3)
    with pytest.raises(ValueError, match="CUDA device"):
        graphed.GraphedTrainStep(m, optimizer=torch.optim.Adam(m.parameters()), max_norm=1.0)


def _torch_host_scalars(lr, beta1, beta2, eps, wd, step_t):
    """_multi_tensor_adam's host arithmetic restated (non-capturable branch, one CPU step tensor), and the fp32 value
    each scalar becomes in its foreach kernel (c10::Scalar -> opmath float)."""
    step = torch.tensor(float(step_t - 1), dtype=torch.float32)
    torch._foreach_add_([step], torch.tensor(1.0), alpha=1.0)
    t = step.item()
    bc1 = 1 - math.pow(beta1, t)
    bc2 = 1 - math.pow(beta2, t)
    f = lambda x: float(np.float32(x))      # noqa: E731
    return [f(1 - beta1), f(beta2), f(1 - beta2), f(eps), f(wd), f(-(lr / bc1)), f(math.pow(bc2, 0.5)), 0.0]


@pytest.mark.parametrize("lr,betas,eps,wd", [(5e-3, (0.9, 0.999), 1e-8, 0.0), (1e-3 * 0.7 ** 5, (0.8, 0.99), 1e-6, 0.01),
                                             (0.1, (0.5, 0.5), 1e-3, 1.0), (3e-4, (0.0, 0.0), 1e-8, 0.0)])
def test_per_step_scalars_match_torchs_host_arithmetic(lr, betas, eps, wd):
    for t in [1, 2, 3, 10, 1000, 123457]:
        got = optim.adam_scalars(lr, betas[0], betas[1], eps, wd, float(t))
        assert got.dtype == np.float32
        assert got.tolist() == _torch_host_scalars(lr, betas[0], betas[1], eps, wd, t), t


def test_init_state_matches_adams_init_group():
    ps = _params()
    for p in ps:
        p.grad = torch.ones_like(p)
    ref = torch.optim.Adam(ps)
    ref._init_group(ref.param_groups[0], [], [], [], [], [], [])
    mine = torch.optim.Adam(ps)
    optim.init_state(mine, ps[:2])
    assert ps[2] not in mine.state
    for p in ps[:2]:
        a, b = mine.state[p], ref.state[p]
        assert a.keys() == b.keys()
        for k in a:
            assert a[k].dtype == b[k].dtype and a[k].device == b[k].device and a[k].shape == b[k].shape, k
            assert torch.equal(a[k], b[k]), k


def test_state_key_changes_when_the_state_is_replaced():
    ps = _params()
    opt = torch.optim.Adam(ps)
    empty = optim.state_key(opt)
    assert empty == (None, None, None)
    optim.init_state(opt, ps)
    key = optim.state_key(opt)
    assert key != empty and optim.state_key(opt) == key
    opt.load_state_dict(copy.deepcopy(opt.state_dict()))
    assert optim.state_key(opt) != key
