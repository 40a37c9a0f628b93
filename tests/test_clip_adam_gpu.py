"""Gradient clipping + Adam as two kernels (csrc/optim.cu, optim.ClipAdam) and inside the graphed training steps.

On tensor lists outside any model the kernels are bit-equal to torch: with clipping inactive to
``clip_grad_norm_`` + ``torch.optim.Adam(foreach=True)``; with clipping active to ``clip_grads_with_norm_`` given the
kernels' norm (itself within 1 fp32 ulp of a float64 restatement) + ``Adam.step()``; over two param groups, weight
decay, an ExponentialLR schedule, empty / odd-sized / unaligned / 1.5 M-element tensors, and inf / NaN gradients.
Through the models, under the deterministic flag, the graphed step with ``optimizer`` and ``max_norm`` is bit-equal
to the eager loop that clips with the graphed norm and steps the same Adam."""
import copy

import numpy as np
import pytest
import torch

from gnn_rag_b200 import batching, graphed, loader, optim, synthetic as S

from test_device_split_gpu import _loader, _model, _train_mode
from test_graphed_train_gpu import _det, _fp32_cudnn, _synthetic  # noqa: F401
import test_graphed_graft_train_gpu as GG

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")

NE, NR, NW = 3000, 40, 100
WORD_EMB = 1_500_000


def _shapes(n):
    """n tensor shapes: the first 7 cover 1.5 M elements (the word embedding), 0, 1 and 3 elements and sizes that are
    not a multiple of 4; the rest are layer-sized."""
    base = [(WORD_EMB // 50, 50), (0,), (1,), (3,), (50, 50), (7, 13), (200,)]
    more = [(50 + 3 * i, 37 + (i % 5)) if i % 3 else (201 + i,) for i in range(max(n - len(base), 0))]
    return (base + more)[:n]


def _lists(n, seed, unaligned=False):
    """Two identical parameter lists (ours, torch's) and the per-step gradients.  ``unaligned``: the fifth tensor is
    a view one element into its storage (the kernels' scalar path)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    shapes = _shapes(n)
    vals = [torch.randn(s, generator=g) * 0.5 for s in shapes]
    ours, ref = [], []
    for i, v in enumerate(vals):
        if unaligned and i == 4:
            base = torch.zeros(v.numel() + 1, device=dev)
            base[1:].copy_(v.reshape(-1))
            ours.append(torch.nn.Parameter(base[1:].view(v.shape)))
        else:
            ours.append(torch.nn.Parameter(v.to(dev)))
        ref.append(torch.nn.Parameter(v.to(dev)))
    if unaligned:
        assert ours[4].data_ptr() % 16 != 0
    return ours, ref, g


def _grads(shapes, g, scale):
    return [(torch.randn(s, generator=g) * scale).to(dev) for s in shapes]


def _adam(params, lr=3e-3):
    """Two param groups with their own lr, betas, eps and weight decay (0 and 0.01)."""
    half = (len(params) + 1) // 2
    groups = [dict(params=params[:half], lr=lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0)]
    if params[half:]:
        groups.append(dict(params=params[half:], lr=2 * lr, betas=(0.8, 0.99), eps=1e-6, weight_decay=0.01))
    return torch.optim.Adam(groups, foreach=True)


def _bits_equal(a, b):
    """Equal bit patterns, NaN where NaN (the NaN payload aside)."""
    if not torch.equal(torch.isnan(a), torch.isnan(b)):
        return False
    keep = ~torch.isnan(a)
    return torch.equal(a[keep].view(torch.int32), b[keep].view(torch.int32))


def _norm64(grads):
    return float(torch.stack([g.double().pow(2).sum() for g in grads]).sum().sqrt().float())


def _within_one_ulp(x, ref):
    r = torch.tensor(ref, dtype=torch.float32)
    lo, hi = torch.nextafter(r, torch.tensor(-np.inf)), torch.nextafter(r, torch.tensor(np.inf))
    return float(lo) <= x <= float(hi)


def _run_lists(n, max_norm, clip_active, steps=5, seed=0, unaligned=False, poison=None):
    ours, ref, gen = _lists(n, seed, unaligned)
    shapes = [p.shape for p in ours]
    opt_a, opt_b = _adam(ours), _adam(ref)
    sch_a = torch.optim.lr_scheduler.ExponentialLR(opt_a, gamma=0.7)
    sch_b = torch.optim.lr_scheduler.ExponentialLR(opt_b, gamma=0.7)
    bufs = [torch.zeros(s, device=dev) for s in shapes]
    fused = optim.ClipAdam(opt_a, ours, bufs, max_norm)
    for p, b in zip(ours, bufs):
        p.grad = b
    for it in range(steps):
        grads = _grads(shapes, gen, 0.05 if clip_active else 1e-3)
        if poison is not None and it == steps - 1:
            grads[4].view(-1)[5] = poison
        for b, x in zip(bufs, grads):
            b.copy_(x)
        fused.step()
        torch.cuda.synchronize()
        for p, x in zip(ref, grads):
            p.grad = x.clone()
        if clip_active or poison is not None:
            norm = float(fused.grad_norm)
            if poison is None:
                assert _within_one_ulp(norm, _norm64(grads)), (norm, _norm64(grads))
            torch.nn.utils.clip_grads_with_norm_(ref, max_norm, fused.grad_norm.clone(), foreach=True)
        else:
            torch.nn.utils.clip_grad_norm_(ref, max_norm, foreach=True)
            assert float(fused.grad_norm) <= max_norm
        opt_b.step()
        sch_a.step()
        sch_b.step()
        for i, (a, b) in enumerate(zip(ours, ref)):
            assert _bits_equal(a.grad, b.grad), ("grad", it, i)
            assert _bits_equal(a.detach(), b.detach()), ("param", it, i)
            for k in ("exp_avg", "exp_avg_sq"):
                assert _bits_equal(opt_a.state[a][k], opt_b.state[b][k]), (k, it, i)
    sa, sb = opt_a.state_dict(), opt_b.state_dict()
    assert [s["step"].item() for s in sa["state"].values()] == [s["step"].item() for s in sb["state"].values()]
    assert [g["lr"] for g in sa["param_groups"]] == [g["lr"] for g in sb["param_groups"]]
    return ours, ref, opt_a


@pytest.mark.parametrize("n", [1, 7, 60])
def test_clip_inactive_bit_equal_to_torch(n):
    _run_lists(n, max_norm=1e6, clip_active=False)


@pytest.mark.parametrize("n", [1, 7, 60])
def test_clip_active_bit_equal_to_torch_given_the_norm(n):
    _run_lists(n, max_norm=1.0, clip_active=True, seed=1)


def test_unaligned_tensor_takes_the_scalar_path():
    _run_lists(7, max_norm=1.0, clip_active=True, seed=2, unaligned=True)


@pytest.mark.parametrize("poison", [float("inf"), float("nan")])
def test_non_finite_gradients_reproduce_torch(poison):
    ours, _ref, opt = _run_lists(7, max_norm=1.0, clip_active=True, steps=2, seed=3, poison=poison)
    g = ours[4].grad.view(-1)
    assert torch.isnan(g[5])
    if poison == float("inf"):                   # coef 0: the other gradients become 0, inf * 0 NaN
        assert (ours[0].grad == 0).all()
    else:                                        # a NaN norm makes every gradient NaN
        assert torch.isnan(ours[0].grad).all()


def test_without_max_norm_only_adam_runs():
    ours, ref, gen = _lists(7, 4)
    shapes = [p.shape for p in ours]
    opt_a, opt_b = _adam(ours), _adam(ref)
    bufs = [torch.zeros(s, device=dev) for s in shapes]
    fused = optim.ClipAdam(opt_a, ours, bufs)
    assert fused.grad_norm is None
    for p, b in zip(ours, bufs):
        p.grad = b
    for _ in range(3):
        grads = _grads(shapes, gen, 10.0)
        for b, x in zip(bufs, grads):
            b.copy_(x)
        fused.step()
        for p, x in zip(ref, grads):
            p.grad = x.clone()
        opt_b.step()
    for a, b in zip(ours, ref):
        assert torch.equal(a.grad, b.grad) and torch.equal(a.detach(), b.detach())


# ---- through the models ---------------------------------------------------------------------------------------------

def _rearev_batches():
    m, b1 = _synthetic(D=50, num_ins=3, num_iter=2, num_gnn=3)
    b2 = S.make_batch(8, B=4, N=200, E=1400, num_entity=NE, num_relation=NR, num_word=NW, with_weights=False)[:7]
    assert graphed.fact_capacity(len(b1[2][0])) != graphed.fact_capacity(len(b2[2][0]))
    return m, [b1, b2, b1]


def _nsm_batches():
    m, b1 = _synthetic("NSM", D=50)
    b2 = S.make_batch(9, B=4, N=200, E=1400, num_entity=NE, num_relation=NR, num_word=NW, with_weights=False)[:7]
    return m, [b1, b2, b1]


def _graftnet_batches():
    m, b1 = GG._synthetic(D=50)
    b2 = S.make_graft_batch(9, B=4, N=200, E=1400, num_entity=NE, num_relation=NR, num_word=NW, n_real="ragged")
    assert graphed.fact_capacity(len(b1[2][0])) != graphed.fact_capacity(len(b2[2][0]))
    return m, [b1, b2, b1]


def _trainable(m):
    return [p for p in m.parameters() if p.requires_grad]


def _steps(m, max_norm, wd=0.0):
    m2 = copy.deepcopy(m)
    opt_e = torch.optim.Adam(_trainable(m), lr=5e-3, weight_decay=wd)
    opt_g = torch.optim.Adam(_trainable(m2), lr=5e-3, weight_decay=wd)
    cls = graphed.GraphedGraftTrainStep if type(m).__name__ == "GraftNet" else graphed.GraphedTrainStep
    return m2, opt_e, opt_g, cls(m2, optimizer=opt_g, max_norm=max_norm)


def _eager_iteration(m, opt, b, max_norm, grad_norm, autocast=None):
    opt.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=autocast, enabled=autocast is not None):
        loss = m(b, training=True)[0]
    loss.backward()
    if grad_norm is not None:
        torch.nn.utils.clip_grads_with_norm_(m.parameters(), max_norm, grad_norm)
    else:
        torch.nn.utils.clip_grad_norm_(m.parameters(), max_norm)
    opt.step()
    return loss.detach().clone()


def _assert_same_training(m, m2, opt_e, opt_g):
    for (k, a), b in zip(m.named_parameters(), m2.parameters()):
        assert torch.equal(a.detach(), b.detach()), k
        if a.grad is not None:
            assert torch.equal(a.grad, b.grad), k
    for a, b in zip(_trainable(m), _trainable(m2)):
        sa, sb = opt_e.state.get(a, {}), opt_g.state.get(b, {})
        assert sa.keys() == sb.keys()
        for k in sa:
            assert torch.equal(sa[k], sb[k]), k


def _train_both(m, batches, max_norm=1.0, wd=0.0, autocast=None):
    m2, opt_e, opt_g, step = _steps(m, max_norm, wd)
    norms = []
    for b in batches:
        with torch.autocast("cuda", dtype=autocast, enabled=autocast is not None):
            out = step.step(b)
        out.check()
        loss_g = out[0].clone()
        norms.append(float(out.grad_norm))
        loss_e = _eager_iteration(m, opt_e, b, max_norm, out.grad_norm.clone(), autocast)
        assert torch.equal(loss_e, loss_g)
        _assert_same_training(m, m2, opt_e, opt_g)
    return step, norms


# max_norm sits between the cases' gradient norms, so that some steps clip and others do not
@pytest.mark.parametrize("case,max_norm", [("rearev_d50_lstm", 1e-3), ("nsm", 0.11), ("graftnet_d50", 100.0)])
def test_models_bit_equal_to_the_eager_loop_under_the_deterministic_flag(case, max_norm):
    m, batches = {"rearev_d50_lstm": _rearev_batches, "nsm": _nsm_batches, "graftnet_d50": _graftnet_batches}[case]()
    _det(True)
    step, norms = _train_both(m, batches, max_norm=max_norm, wd=0.01 if case == "nsm" else 0.0)
    assert len(step._cache) == 2
    print("%s: gradient norms %s, max_norm %g" % (case, norms, max_norm))


def test_bf16_autocast_bit_equal_to_the_eager_loop():
    m, batches = _rearev_batches()
    _det(True)
    _train_both(m, batches, max_norm=1e-3, autocast=torch.bfloat16)


def test_device_split_shuffle_bit_equal_to_the_eager_loop():
    L = _loader("ReaRev")
    m = _train_mode(_model("ReaRev", L, eval_mode=False))
    split = loader.DeviceSplit(L, dev, shuffle=True)
    _det(True)
    m2, opt_e, opt_g, step = _steps(m, 1.0)
    for it in (0, 1, 0):
        b = split.get_batch(it, 6, 0.1)
        out = step.step(b)
        loss_e = _eager_iteration(m, opt_e, b, 1.0, out.grad_norm.clone())
        assert torch.equal(loss_e, out[0])
        _assert_same_training(m, m2, opt_e, opt_g)
    split.check()


def _normwise(xs, ys):
    """The largest difference of a tensor relative to its largest entry, over paired tensor lists."""
    with torch.no_grad():
        return max(float((a - b).abs().max() / b.abs().max()) for a, b in zip(xs, ys) if a.numel() and b.abs().max() > 0)


@pytest.mark.parametrize("case,max_norm", [("rearev_d50_lstm", 1e-3), ("graftnet_d50", 100.0)])
def test_close_to_plain_clip_and_adam_without_the_deterministic_flag(case, max_norm):
    """The same gradients -- each step's, from the graphed backward with fp32 atomics -- through the fused kernels
    and through plain ``clip_grad_norm_`` (torch's own norm) + Adam: only the norm differs (by at most an ulp or so)."""
    m, batches = {"rearev_d50_lstm": _rearev_batches, "graftnet_d50": _graftnet_batches}[case]()
    _det(False)
    cls = graphed.GraphedGraftTrainStep if case == "graftnet_d50" else graphed.GraphedTrainStep
    step = cls(m)
    ours = _trainable(m)
    ref = [torch.nn.Parameter(p.detach().clone()) for p in ours]
    opt_a, opt_b = torch.optim.Adam(ours, lr=5e-3), torch.optim.Adam(ref, lr=5e-3)
    bufs = [torch.zeros_like(p) for p in ours]
    fused = None
    for b in batches:
        step.step(b)
        grads = [p.grad.clone() if p.grad is not None else torch.zeros_like(p) for p in ours]
        if fused is None:
            fused = optim.ClipAdam(opt_a, ours, bufs, max_norm)
        for p, buf, g in zip(ours, bufs, grads):
            buf.copy_(g)
            p.grad = buf
        fused.step()
        for p, g in zip(ref, grads):
            p.grad = g
        torch.nn.utils.clip_grad_norm_(ref, max_norm)
        opt_b.step()
    worst = _normwise(ours, ref)
    print("%s: largest relative parameter difference %.3g" % (case, worst))
    assert worst <= 1e-5


@pytest.mark.parametrize("case,max_norm", [("rearev_d50_lstm", 1e-3), ("graftnet_d50", 100.0)])
def test_graphed_loop_against_the_eager_loop_without_the_deterministic_flag(case, max_norm):
    """End to end, graphed fused step against the eager loop with plain clip + Adam, both with fp32 atomics in the
    backward.  Adam divides each gradient entry by its own running scale, so an entry whose gradient is near zero
    (where the atomics' rounding decides its sign or size) moves by up to lr either way: the difference is of the order
    of lr relative to the tensor's scale, not of the gradients' rounding."""
    m, batches = {"rearev_d50_lstm": _rearev_batches, "graftnet_d50": _graftnet_batches}[case]()
    _det(False)
    m2, opt_e, opt_g, step = _steps(m, max_norm)
    for b in batches:
        step.step(b)
        _eager_iteration(m, opt_e, b, max_norm, None)
    worst = _normwise(list(m2.parameters()), list(m.parameters()))
    print("%s: largest relative parameter difference, end to end %.3g" % (case, worst))
    assert worst <= 2 * 5e-3 * len(batches)


def test_state_dict_after_two_graphed_steps_continues_bit_equal():
    m, batches = _rearev_batches()
    m_b = copy.deepcopy(m)
    _det(True)
    opt = torch.optim.Adam(_trainable(m), lr=5e-3)
    step = graphed.GraphedTrainStep(m, optimizer=opt, max_norm=1.0)
    for b in batches[:2]:
        step.step(b)
    sd = copy.deepcopy(opt.state_dict())
    m_b.load_state_dict(m.state_dict())
    graphs = len(step._cache)
    out = step.step(batches[2])                    # continuing in the graph
    assert len(step._cache) == graphs
    opt_b = torch.optim.Adam(_trainable(m_b), lr=5e-3)
    opt_b.load_state_dict(sd)
    _eager_iteration(m_b, opt_b, batches[2], 1.0, out.grad_norm.clone())
    _assert_same_training(m_b, m, opt_b, opt)
    assert opt_b.state_dict()["state"][0]["step"].item() == 3.0


def test_load_state_dict_recaptures():
    m, batches = _rearev_batches()
    opt = torch.optim.Adam(_trainable(m), lr=5e-3)
    step = graphed.GraphedTrainStep(m, optimizer=opt, max_norm=1.0)
    step.step(batches[0])
    step.step(batches[0])
    assert len(step._cache) == 1
    key = step.key(batches[0])
    opt.load_state_dict(copy.deepcopy(opt.state_dict()))
    assert step.key(batches[0]) != key
    step.step(batches[0])
    assert len(step._cache) == 2
    assert opt.state[_trainable(m)[0]]["step"].item() == 3.0


def test_lr_schedule_needs_no_recapture():
    m, batches = _rearev_batches()
    opt = torch.optim.Adam(_trainable(m), lr=5e-3)
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=0.5)
    step = graphed.GraphedTrainStep(m, optimizer=opt)
    for _ in range(3):
        out = step.step(batches[0])
        assert out.grad_norm is None
        sched.step()
    assert len(step._cache) == 1


def test_replay_does_not_synchronise_with_the_host():
    m, batch = _synthetic(D=50, num_ins=3, num_iter=2, num_gnn=3)
    pinned = batching.pin_batch(batch)
    opt = torch.optim.Adam(_trainable(m), lr=5e-3, weight_decay=0.01)
    step = graphed.GraphedTrainStep(m, optimizer=opt, max_norm=1.0)
    step.step(pinned)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = step.step(pinned)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    out.check()
    assert torch.isfinite(out.grad_norm).item()


def test_graftnet_replay_does_not_synchronise_with_the_host():
    m, batch = GG._synthetic(D=50)
    pinned = batching.pin_graft_batch(batch)
    opt = torch.optim.Adam(_trainable(m), lr=5e-3)
    step = graphed.GraphedGraftTrainStep(m, optimizer=opt, max_norm=1.0)
    step.step(pinned)
    out = GG._step_without_sync(step, pinned)
    out.check()
    assert torch.isfinite(out.grad_norm).item()


def test_refusals_on_the_device():
    m, _b = _synthetic(D=50, num_ins=2, num_iter=2, num_gnn=2)
    other = torch.nn.Parameter(torch.zeros(3, device=dev))
    for opt, max_norm, msg in [
            (torch.optim.SGD(m.parameters(), lr=1e-3), None, "torch.optim.Adam"),
            (torch.optim.AdamW(m.parameters(), lr=1e-3), None, "torch.optim.Adam"),
            (torch.optim.Adam(m.parameters(), amsgrad=True), None, "amsgrad"),
            (torch.optim.Adam(m.parameters(), fused=True), None, "fused"),
            (torch.optim.Adam(m.parameters(), capturable=True), None, "capturable"),
            (torch.optim.Adam(m.parameters(), maximize=True), None, "maximize"),
            (torch.optim.Adam(m.parameters(), decoupled_weight_decay=True), None, "decoupled_weight_decay"),
            (torch.optim.Adam(m.parameters(), differentiable=True), None, "differentiable"),
            (torch.optim.Adam(m.parameters(), lr=torch.tensor(1e-3)), None, "float lr"),
            (torch.optim.Adam(list(m.parameters()) + [other]), None, "not the model's"),
            (None, 1.0, "needs an optimizer"),
            (torch.optim.Adam(m.parameters()), 0.0, "max_norm"),
            (torch.optim.Adam(m.parameters()), -1.0, "max_norm")]:
        with pytest.raises(ValueError, match=msg):
            graphed.GraphedTrainStep(m, optimizer=opt, max_norm=max_norm)
    with pytest.raises(ValueError, match="not the model's"):
        graphed.GraphedGraftTrainStep(GG._synthetic(D=50)[0], optimizer=torch.optim.Adam([other]))
