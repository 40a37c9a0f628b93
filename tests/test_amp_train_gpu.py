"""Mixed-precision training under torch.autocast(bfloat16): the bf16 node-tensor I/O of the training kernels
(csrc/aggregate.cu, csrc/aggregate_bwd.cu, csrc/graft.cu: the *_ex entry points with GR_IO_BF16) and the autograd
Functions and models that select it.

* Rounding contract: the forward kernels and every deterministic backward kernel in bf16 mode equal the fp32 kernel on
  the upcast inputs followed by ``.to(torch.bfloat16)``, bit for bit, over the edge shapes of the fp32 tests.  The
  atomic backward kernels meet the fp32 kernels' per-element float64 bounds on the upcast inputs; their one bf16
  store, GraftNet's grad_head, is an owned sum and is checked bit for bit as well.
* The four autograd Functions: bf16 node-sized outputs, fp32 and bf16 grad_out give the same gradients, the node-sized
  tensors they save are bf16 and nothing of shape [facts, D] is saved.
* Models: one step under autocast against fp32, three Adam steps, the torch fallbacks, fp16 autocast, inference and
  Evaluator unchanged by autocast, and bit-reproducible steps under use_deterministic_algorithms + bf16 autocast."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import autograd_path, batching, ops, synthetic as S
from graft_train_ref import ref_aggregate

import test_aggregate_backward_gpu as AB
import test_configs_gpu as CG
import test_graftnet_train_gpu as GT

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
BF = torch.bfloat16
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bits_equal(a, b):
    torch.cuda.synchronize()
    assert a.dtype == b.dtype and a.shape == b.shape
    view = torch.int16 if a.dtype == BF else torch.int32
    eq = a.contiguous().view(view) == b.contiguous().view(view)
    assert bool(eq.all()), "%d of %d elements differ" % (int((~eq).sum()), eq.numel())


def _bf(t):
    """t rounded to bf16, and that value widened back to fp32 (the upcast input of the contract)."""
    t16 = t.to(BF)
    return t16, t16.float()


@pytest.fixture
def flag():
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    yield
    torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])


# ---- aggregation ----------------------------------------------------------------------------------------------------

SHAPE_CASES = AB.CASES + [(33, 2, "fwd", True, "hub", 2, 300, 400), (31, 4, "inv", False, "random", 20000, 5, 6),
                          (8, 1, "fwd", True, "random", 1, 1, 3)]


def _agg_case(params):
    if len(params) == 4:
        D, I, direction, weights = params
        return AB._Case(D * 7 + I, D, I, direction, weights)
    D, I, direction, weights, kind, B, N, E = params
    return AB._Case(B + N + D, D, I, direction, weights, kind=kind, B=B, N=N, E=E)


@pytest.mark.parametrize("params", SHAPE_CASES, ids=str)
def test_aggregate_forward_bf16_is_the_rounded_fp32_output(params):
    c = _agg_case(params)
    out32 = ops.aggregate(c.g, c.direction, c.prior, c.table, c.ins, w=c.w_csr)
    out16 = ops.aggregate(c.g, c.direction, c.prior, c.table, c.ins, w=c.w_csr, dtype=BF)
    assert out16.dtype == BF
    _bits_equal(out16, out32.to(BF))


def _agg_bwd(c, G, deterministic, pre):
    bufs = [p.clone() for p in pre]
    ops.aggregate_backward(c.g, c.direction, c.prior, c.table, c.ins, G, *bufs, w=c.w_csr, deterministic=deterministic)
    return bufs


def _prefill(c, seed):
    rs = np.random.RandomState(seed)
    return [torch.from_numpy(rs.randn(*s).astype(np.float32)).to(dev)
            for s in ((c.R1, c.D), (c.B, c.I, c.D), (c.B, c.N))]


@pytest.mark.parametrize("params", SHAPE_CASES, ids=str)
def test_aggregate_backward_det_bf16_equals_fp32_on_the_upcast_gradient(params):
    """Pre-filled accumulators; a bf16 grad_out read with the wrong row stride or summed in another order shows here."""
    c = _agg_case(params)
    G16, G32 = _bf(c.G)
    pre = _prefill(c, 1)
    for a, b in zip(_agg_bwd(c, G16, True, pre), _agg_bwd(c, G32, True, pre)):
        _bits_equal(a, b)


@pytest.mark.parametrize("params", SHAPE_CASES, ids=str)
def test_aggregate_backward_atomic_bf16_within_the_fp64_bound(params):
    """The atomic kernel reading bf16 grad_out: the fp32 kernels' per-element bound against float64 autograd on the
    upcast gradient (its accumulators stay fp32, so no bf16 rounding is added)."""
    c = _agg_case(params)
    G16, c.G = _bf(c.G)
    zeros = [torch.zeros_like(p) for p in _prefill(c, 0)]
    AB._check(c, _agg_bwd(c, G16, False, zeros))


def test_aggregate_backward_bf16_without_facts_is_a_no_op():
    c = AB._Case(5, 33, 2, "inv", True)
    g0 = ops.csr_build(*(torch.zeros(0, dtype=torch.int64, device=dev) for _ in range(3)), c.B, c.N, c.R1)
    pre = _prefill(c, 2)
    for det in (False, True):
        bufs = [p.clone() for p in pre]
        ops.aggregate_backward(g0, "fwd", c.prior, c.table, c.ins, c.G.to(BF), *bufs, deterministic=det)
        for a, b in zip(bufs, pre):
            _bits_equal(a, b)


# ---- TypeLayer ------------------------------------------------------------------------------------------------------

def _type_case(D, weighted):
    R1 = 13
    b = S.make_batch(D, B=3, N=50, E=400, num_entity=500, num_relation=R1 - 1, num_word=20, powerlaw=True,
                     n_real="ragged", with_weights=True)
    g = batching.stage_batch(b, dev, R1, False, weighted).graph
    w = (g.wr_t, g.wr_h) if weighted else (None, None)
    rs = np.random.RandomState(D + weighted)
    table = torch.from_numpy(rs.randn(R1, D).astype(np.float32)).to(dev)
    table[torch.from_numpy(rs.rand(R1, D) < 0.2).to(dev)] = 0.0        # exact zeros in out: the relu mask is closed
    return b, g, w, table, rs


@pytest.mark.parametrize("D", [1, 31, 50, 200, 256, 512])
@pytest.mark.parametrize("weighted", [False, True])
def test_type_layer_bf16_forward_and_det_backward_are_bit_exact(flag, D, weighted):
    _b, g, w, table, rs = _type_case(D, weighted)
    Nt = g.B * g.N
    out32 = torch.empty(Nt, D, device=dev)
    out16 = torch.empty(Nt, D, device=dev, dtype=BF)
    ops.type_layer(g, table, out32, *w)
    ops.type_layer(g, table, out16, *w)
    _bits_equal(out16, out32.to(BF))
    assert bool((out16 == 0).any()) and bool((out16 > 0).any())
    G16, G32 = _bf(torch.from_numpy(rs.randn(Nt, D).astype(np.float32)).to(dev))
    pre = torch.from_numpy(rs.randn(g.R1, D).astype(np.float32)).to(dev)
    got, want = pre.clone(), pre.clone()
    # the mask comes from the bf16 out the bf16 forward wrote: a mask from any other buffer differs here
    ops.type_layer_backward(g, G16, out16, got, *w, deterministic=True)
    ops.type_layer_backward(g, G32, out16.float(), want, *w, deterministic=True)
    _bits_equal(got, want)


@pytest.mark.parametrize("D", [1, 31, 200, 512])
def test_type_layer_atomic_backward_bf16_within_the_fp64_bound(D):
    b, g, w, table, rs = _type_case(D, True)
    Nt = g.B * g.N
    out16 = torch.empty(Nt, D, device=dev, dtype=BF)
    ops.type_layer(g, table, out16, *w)
    G16, G32 = _bf(torch.from_numpy(rs.randn(Nt, D).astype(np.float32)).to(dev))
    got = torch.zeros(g.R1, D, device=dev)
    ops.type_layer_backward(g, G16, out16, got, *w)
    heads, rels, tails = (torch.as_tensor(np.asarray(x, dtype=np.int64)) for x in b[2][:3])
    wf = torch.as_tensor(np.asarray(b[2][6], dtype=np.float64)).unsqueeze(1)
    Gm = G32.cpu().double() * (out16.float().cpu() > 0)
    want = torch.zeros(g.R1, D, dtype=torch.float64).index_add(0, rels, (Gm[tails] + Gm[heads]) * wf)
    scale = torch.zeros(g.R1, D, dtype=torch.float64).index_add(0, rels, (Gm[tails].abs() + Gm[heads].abs()) * wf)
    cnt = 2 * torch.bincount(rels, minlength=g.R1).double().unsqueeze(1)
    GT._check(got, want, cnt + 2, scale, "grad_table")


# ---- GraftNet fact messages -----------------------------------------------------------------------------------------

def _graft_case(D, with_facts=True):
    rs = np.random.RandomState(D)
    B, N, R1, maxF = 3, 40, 9, 3600
    per_q = [3400, 0, 70] if with_facts else [0, 0, 0]
    gg, _kfr, st = GT._graft(B, N, maxF, R1, rs, per_q, head_hub=2500 if with_facts else 0,
                             tail_hub=2500 if with_facts else 0)
    Nt, F_ = B * N, st["heads"].numel()
    self_tab = torch.from_numpy(rs.randn(R1, D).astype(np.float32)).to(dev)
    head16, head32 = _bf(torch.from_numpy(rs.randn(Nt, D).astype(np.float32)).to(dev))
    if F_:                                               # self + head == 0 exactly at one fact
        h0, r0 = int(st["heads"][0]), int(st["rels"][0])
        self_tab[r0, : (D + 1) // 2] = -head32[h0, : (D + 1) // 2]
    s = torch.from_numpy(rs.rand(F_).astype(np.float32)).to(dev)
    s[torch.from_numpy(rs.rand(F_) < 0.3).to(dev)] = 0.0
    G16, G32 = _bf(torch.from_numpy(rs.randn(Nt, D).astype(np.float32)).to(dev))
    pre = [torch.from_numpy(rs.randn(*sh).astype(np.float32)).to(dev) for sh in ((F_,), (R1, D), (Nt, D))]
    return dict(gg=gg, st=st, self_tab=self_tab, head16=head16, head32=head32, s=s, G16=G16, G32=G32, pre=pre)


def _graft_bwd(c, head, G, ghead_dtype, seed, p, deterministic):
    gs, gself = c["pre"][0].clone(), c["pre"][1].clone()
    ghead = c["pre"][2].to(ghead_dtype, copy=True)
    ops.graft_aggregate_backward(c["gg"], c["s"], c["self_tab"], head, G, gs, gself, ghead, seed, p,
                                 deterministic=deterministic)
    return gs, gself, ghead


@pytest.mark.parametrize("D", [1, 31, 50, 200, 256, 512])
@pytest.mark.parametrize("p", [0.0, 0.2])
def test_graft_aggregate_bf16_forward_and_backward_bit_exact(flag, D, p):
    """Forward and the deterministic backward: bit-exact to fp32 on the upcast inputs, grad_head rounded from the fp32
    value (the bf16 pre-filled buffer widened, the sum added, rounded once).  The atomic backward: grad_s and grad_head
    are owned sums, bit-exact too; grad_self (fp32 atomics) within the fp64 bound of the fp32 test."""
    c = _graft_case(D)
    seed = torch.tensor([77], dtype=torch.int64, device=dev)
    out16 = ops.graft_aggregate_train(c["gg"], c["s"], c["self_tab"], c["head16"], seed, p)
    out32 = ops.graft_aggregate_train(c["gg"], c["s"], c["self_tab"], c["head32"], seed, p)
    assert out16.dtype == BF
    _bits_equal(out16, out32.to(BF))
    c["pre"][2] = c["pre"][2].to(BF).float()             # a bf16 accumulator holds bf16 values
    for det in (True, False):
        gs16, gself16, gh16 = _graft_bwd(c, c["head16"], c["G16"], BF, seed, p, det)
        gs32, gself32, gh32 = _graft_bwd(c, c["head32"], c["G32"], torch.float32, seed, p, det)
        _bits_equal(gs16, gs32)
        _bits_equal(gh16, gh32.to(BF))
        if det:
            _bits_equal(gself16, gself32)
    # grad_self of the atomic kernel against float64
    st = c["st"]
    mask = ops.graft_dropout_mask(seed, p, c["gg"].B * c["gg"].max_fact, D).cpu() if p > 0 else None
    lt = c["self_tab"].cpu().double().requires_grad_(True)
    ref = ref_aggregate(lt, c["head32"].cpu().double(), c["s"].cpu().double(), st, c["gg"].B * c["gg"].N, mask, p)
    (ref * c["G32"].cpu().double()).sum().backward()
    keep = (mask[st["slot_of"]].double() / (1 - p)) if mask is not None else 1.0
    a = c["self_tab"].cpu().double()[st["rels"]] + c["head32"].cpu().double()[st["heads"]]
    gterm = (c["G32"].cpu().double()[st["tails"]] * keep).abs() * c["s"].cpu().double().unsqueeze(1) * (a > 0)
    R1 = c["self_tab"].shape[0]
    deg_r = torch.bincount(st["rels"], minlength=R1).double().unsqueeze(1)
    pre_self = c["pre"][1].cpu().double()
    GT._check(gself16, pre_self + lt.grad, deg_r + 3,
              torch.zeros(R1, D, dtype=torch.float64).index_add(0, st["rels"], gterm) + pre_self.abs(), "grad_self")


@pytest.mark.parametrize("D", [1, 200])
def test_graft_aggregate_bf16_without_staged_facts(D):
    c = _graft_case(D, with_facts=False)
    out = ops.graft_aggregate_train(c["gg"], c["s"], c["self_tab"], c["head16"])
    assert out.dtype == BF and float(out.float().abs().max()) == 0.0
    for det in (False, True):
        gs, gself, gh = _graft_bwd(c, c["head16"], c["G16"], BF, None, 0.0, det)
        _bits_equal(gself, c["pre"][1])
        _bits_equal(gh, c["pre"][2].to(BF))


# ---- autograd Functions ---------------------------------------------------------------------------------------------

def _graft_model(D, dropout, **over):
    return GT._graft_model(D, dropout, **over)


def _graft_batch(seed=3, **kw):
    kw = dict(dict(B=3, N=40, E=150, num_entity=1000, num_relation=40, num_word=100), **kw)
    return S.make_graft_batch(seed, **kw)


def test_functions_return_bf16_node_outputs_and_take_either_gradient_dtype(flag):
    """Under bf16 autocast each Function's node-sized output is bf16 (the attention's W [B, max_fact] stays fp32).
    Their backward, called with the bf16 gradient or with the same values in fp32, gives identical gradients
    (deterministic kernels, so equal means bit-equal), returned in each input's dtype."""
    torch.use_deterministic_algorithms(True, warn_only=True)
    c = AB._Case(21, 40, 2, "fwd", True)
    table = c.table.to(BF).requires_grad_(True)
    ins = c.ins.clone().requires_grad_(True)
    prior = c.prior.clone().requires_grad_(True)
    b, g, w, ttab, _rs = _type_case(48, True)
    ttab = ttab.to(BF).requires_grad_(True)
    gc = _graft_case(50)
    gs = [gc["self_tab"].to(BF).requires_grad_(True), gc["head16"].clone().requires_grad_(True),
          gc["s"].clone().requires_grad_(True)]
    B, maxF = gc["gg"].B, gc["gg"].max_fact
    qh = torch.randn(B, 5, 50, device=dev).to(BF).requires_grad_(True)
    rel = torch.randn(9, 50, device=dev).to(BF).requires_grad_(True)
    qmask = torch.ones(B, 5, device=dev)
    with torch.autocast("cuda", dtype=BF):
        outs = [autograd_path._AggregateFn.apply(table, ins, prior, c.g, "fwd", c.w_csr),
                autograd_path._TypeLayerFn.apply(ttab, g, *w),
                autograd_path._GraftAggregateFn.apply(*gs, gc["gg"], None, 0.0),
                autograd_path._GraftAttentionFn.apply(qh, rel, qmask, gc["gg"])]
    assert [o.dtype for o in outs] == [BF, BF, BF, torch.float32]
    assert outs[3].shape == (B, maxF)
    for o in outs:
        g16 = torch.randn(o.shape, device=dev).to(o.dtype)
        a = o.grad_fn.apply(g16)                            # the Function's backward itself, no dtype cast by the engine
        r = o.grad_fn.apply(g16.float())
        for x, y in zip(a, r):
            if x is not None:
                _bits_equal(x, y)
    gt16 = torch.randn(outs[1].shape, device=dev).to(BF)      # the relu mask is the forward's bf16 output
    want = torch.zeros(ttab.shape, device=dev)
    ops.type_layer_backward(g, gt16, outs[1].detach(), want, *w, deterministic=True)
    _bits_equal(outs[1].grad_fn.apply(gt16)[0], want.to(BF))
    ga = outs[0].grad_fn.apply(torch.randn(outs[0].shape, device=dev).to(BF))
    assert [t.dtype for t in ga[:3]] == [BF, torch.float32, torch.float32]
    gg_ = outs[2].grad_fn.apply(torch.randn(outs[2].shape, device=dev).to(BF))
    assert [t.dtype for t in gg_[:3]] == [BF, BF, torch.float32]


def test_saved_node_tensors_are_bf16_and_no_fact_tensor_is_saved():
    """GraftNet with dropout and ReaRev, one training forward under bf16 autocast: every tensor our Functions save
    with B*N*D elements is bf16, and nothing with facts x D elements is saved anywhere."""
    D = 64
    m = _graft_model(D, 0.2, num_relation=40, num_word=50, num_entity=600)
    m.train()
    b = S.make_graft_batch(2, B=4, N=500, E=8000, num_entity=600, num_relation=40, num_word=50)
    thresh = min(len(b[2][0]), len(b[3][0][0]), b[5].size) * D // 2
    saved = []

    def pack(t):
        saved.append((t.numel(), t.dtype, t.shape))
        return t
    fn_saved = []
    orig = torch.autograd.function.FunctionCtx.save_for_backward

    def spy(ctx, *ts):
        fn_saved.extend(t for t in ts if t is not None)
        return orig(ctx, *ts)
    torch.autograd.function.FunctionCtx.save_for_backward = spy
    try:
        with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t), torch.autocast("cuda", dtype=BF):
            loss = m(b, training=True)[0]
    finally:
        torch.autograd.function.FunctionCtx.save_for_backward = orig
    loss.backward()
    assert not [s for s in saved if s[0] >= thresh], thresh
    node = [t for t in fn_saved if t.dim() == 2 and t.shape[0] == 4 * 500]
    assert node and all(t.dtype == BF for t in node), [(t.shape, t.dtype) for t in node]


# ---- models ---------------------------------------------------------------------------------------------------------

def _model(name, seed=0, **over):
    kw = dict(use_cuda=True, lm_dropout=0.0, linear_dropout=0.0)
    kw.update(over)
    args = S.model_args(name, **kw)
    torch.manual_seed(seed)
    return getattr(G, name)(args, 1000, 40, 100).cuda()


def _batch(name, seed=5, B=6, N=120, E=600):
    if name == "GraftNet":
        return S.make_graft_batch(seed, B=B, N=N, E=E, num_entity=1000, num_relation=40, num_word=100, powerlaw=True,
                                  n_real="ragged")
    return S.make_batch(seed, B=B, N=N, E=E, num_entity=1000, num_relation=40, num_word=100, powerlaw=True,
                        n_real="ragged", with_weights=True)


MODELS = {
    "rearev_d50": ("ReaRev", dict(entity_dim=50, num_iter=2, num_ins=2, num_gnn=2)),
    "rearev_d200": ("ReaRev", dict(entity_dim=200, num_iter=2, num_ins=2, num_gnn=2)),
    "nsm_reason_kb": ("NSM", dict(entity_dim=64, num_step=3, reason_kb=True)),
    "graftnet_drop": ("GraftNet", dict(entity_dim=64, num_layer=3, linear_dropout=0.2)),
}


def _step(m, b, amp_dtype=None):
    m.zero_grad()
    torch.manual_seed(11)
    with torch.autocast("cuda", dtype=amp_dtype or BF, enabled=amp_dtype is not None):
        loss = m(b, training=True)[0]
    loss.backward()
    return loss.detach().float(), {k: p.grad.detach().float().clone() for k, p in m.named_parameters()
                                   if p.grad is not None}


@pytest.mark.parametrize("key", list(MODELS))
def test_one_step_under_autocast_agrees_with_fp32(key):
    """Same weights and batch, dropout layers in eval mode (torch draws different dropout masks for bf16 and fp32
    tensors): the loss within 2e-2 relative, and every parameter gradient whose norm exceeds 1e-6 of the largest has
    cosine similarity >= 0.98 with its fp32 counterpart.  The observed values are printed; on an H100 the losses agreed
    within 2e-4 and the cosines were >= 0.993 except ReaRev D = 50's e2e_linear1.bias at 0.990: a bias gradient is a
    sum over all B*N rows of the bf16 gradient rows torch's autocast GEMM backward reduces, with cancellation, so 0.99
    leaves no margin there.  The score bias is left out: softmax is shift invariant, so its exact gradient is zero and
    both runs hold rounding noise there."""
    name, over = MODELS[key]
    m = _model(name, **over).train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.eval()
    b = _batch(name)
    l32, g32 = _step(m, b)
    l16, g16 = _step(m, b, BF)
    assert set(g32) == set(g16)
    rel = abs(float(l16) - float(l32)) / abs(float(l32))
    gmax = max(float(g.norm()) for g in g32.values())
    cos = {k: float(torch.nn.functional.cosine_similarity(g16[k].flatten(), g.flatten(), dim=0, eps=1e-30))
           for k, g in g32.items() if float(g.norm()) > 1e-6 * gmax and not k.endswith("score_func.bias")}
    worst = min(cos, key=cos.get)
    print("AMP %s: loss rel diff %.3g, min grad cosine %.5f (%s)" % (key, rel, cos[worst], worst))
    assert rel <= 2e-2
    assert cos[worst] >= 0.98, (worst, cos[worst])


@pytest.mark.parametrize("key", list(MODELS))
def test_three_adam_steps_under_autocast_are_finite(key):
    """Dropout on (GraftNet's in-kernel fact dropout included)."""
    name, over = MODELS[key]
    m = _model(name, **over).train()
    b = _batch(name)
    opt = torch.optim.Adam([p for p in m.parameters() if p.requires_grad], lr=1e-3)
    for _ in range(3):
        opt.zero_grad()
        with torch.autocast("cuda", dtype=BF):
            loss = m(b, training=True)[0]
        loss.backward()
        torch.nn.utils.clip_grad_norm_([p for p in m.parameters() if p.requires_grad], 1.0)
        opt.step()
        assert torch.isfinite(loss).all()
    assert all(torch.isfinite(p).all() for p in m.parameters())


@pytest.mark.parametrize("name,over", [("ReaRev", dict(entity_dim=264, num_iter=1, num_ins=2, num_gnn=1)),
                                       ("GraftNet", dict(entity_dim=520, num_layer=2))])
def test_torch_fallbacks_run_under_autocast(name, over):
    """ReaRev at D = 264 (the aggregation beyond the kernel) and GraftNet at D = 520 (the fact kernels' limit): the
    per-fact torch ops, scatters accumulated in fp32; the loss agrees with fp32 like the kernel path's."""
    m = _model(name, **over).train()
    b = _batch(name, B=2, N=40, E=120)
    assert not autograd_path._fact_kernels(dev, 520)
    l32, g32 = _step(m, b)
    l16, g16 = _step(m, b, BF)
    assert torch.isfinite(l16) and all(torch.isfinite(g).all() for g in g16.values())
    assert abs(float(l16) - float(l32)) <= 2e-2 * abs(float(l32))


@pytest.mark.parametrize("key", list(MODELS))
def test_fp16_autocast_runs_the_fp32_kernels(key):
    name, over = MODELS[key]
    m = _model(name, **over).train()
    l16, g16 = _step(m, _batch(name), torch.float16)
    assert torch.isfinite(l16) and all(torch.isfinite(g).all() for g in g16.values())


@pytest.mark.parametrize("key", list(MODELS))
def test_inference_ignores_autocast(key):
    name, over = MODELS[key]
    m = _model(name, **over).eval()
    b = _batch(name)
    with torch.no_grad():
        want = [t.clone() for t in m(b)[1:3]]               # pred, pred_dist
        with torch.autocast("cuda", dtype=BF):
            got = m(b)[1:3]
    for a, r in zip(got, want):
        assert a.dtype == r.dtype and torch.equal(a, r)


def test_evaluator_results_ignore_autocast(tmp_path):
    args = S.model_args("ReaRev", entity_dim=32, num_iter=3, num_ins=2, num_gnn=2, word_dim=16, use_cuda=True,
                        checkpoint_dir=str(tmp_path) + "/", experiment_name="t")
    torch.manual_seed(0)
    m = G.ReaRev(dict(args), 500, 30, 60).eval()
    ev = G.Evaluator(args, m, {"m.%04d" % i: i for i in range(500)}, {}, torch.device("cuda"))
    want = ev.evaluate(CG._FakeLoader(B=4, N=64, E=200, num_data=10), test_batch_size=4)
    with torch.autocast("cuda", dtype=BF):
        got = ev.evaluate(CG._FakeLoader(B=4, N=64, E=200, num_data=10), test_batch_size=4)
    assert got == want


# ---- determinism, in child processes --------------------------------------------------------------------------------

CHILD = r'''
import hashlib, json
import torch
torch.use_deterministic_algorithms(True)
import gnn_rag_b200 as G
from gnn_rag_b200 import synthetic as S

CONFIGS = %s

def digest(ts):
    h = hashlib.sha256()
    for t in ts:
        h.update(t.detach().contiguous().view(-1).view(torch.uint8).cpu().numpy().tobytes())
    return h.hexdigest()

def train(key):
    name, over = CONFIGS[key]
    kw = dict(use_cuda=True, lm_dropout=0.0, linear_dropout=0.0)
    kw.update(over)
    torch.manual_seed(0)
    m = getattr(G, name)(S.model_args(name, **kw), 1000, 40, 100).cuda().train()
    if name == "GraftNet":
        b = S.make_graft_batch(5, B=6, N=120, E=600, num_entity=1000, num_relation=40, num_word=100, powerlaw=True,
                               n_real="ragged")
    else:
        b = S.make_batch(5, B=6, N=120, E=600, num_entity=1000, num_relation=40, num_word=100, powerlaw=True,
                         n_real="ragged", with_weights=True)
    params = [p for p in m.parameters() if p.requires_grad]
    opt = torch.optim.Adam(params, lr=1e-3)
    losses = []
    for _ in range(3):
        opt.zero_grad()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = m(b, training=True)[0]
        loss.backward()
        torch.nn.utils.clip_grad_norm_(params, 1.0)
        opt.step()
        losses.append(loss.detach().float().reshape(1))
    return digest(losses + list(m.state_dict().values()))

print("RESULT " + json.dumps({k: [train(k), train(k)] for k in CONFIGS}))
''' % repr(MODELS)


def _child():
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", CHILD]
    res = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stderr[-4000:]
    line = [ln for ln in res.stdout.splitlines() if ln.startswith("RESULT ")][-1]
    return json.loads(line[len("RESULT "):])


def test_deterministic_bf16_autocast_steps_are_bit_identical_across_runs_and_processes():
    """use_deterministic_algorithms(True) with bf16 autocast: three steps of forward, backward, clip_grad_norm_ and
    Adam give bit-identical losses and state_dicts twice in one child process and once more in a second one."""
    a, b = _child(), _child()
    assert set(a) == set(MODELS)
    for k in a:
        assert a[k][0] == a[k][1] == b[k][0] == b[k][1], k
