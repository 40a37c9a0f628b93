"""CPU: the float64 restatements of tests/fp64_ref.py agree with the fp32 oracle (oracle/kgqa_oracle.py, itself
pinned to the unmodified reference by tests/test_oracle.py) on a small synthetic batch, with and without edge
weights.  Bound: 1e-5 of each element's absolute-value scale -- the oracle sums at most a few dozen fp32 terms per
element, so its own error is below 1e-6 of that scale, while a wrong direction, a missing weight factor or a wrong
segment order moves elements by O(1) of it."""
import numpy as np
import pytest
import torch

from gnn_rag_b200 import synthetic as S
from oracle import kgqa_oracle as O

import fp64_ref as R

B, N, E, NE, NR, NW, D, I = 3, 20, 60, 100, 10, 20, 12, 2
TOL = 1e-5


def _batch(weights):
    b = S.make_batch(3, B=B, N=N, E=E, num_entity=NE, num_relation=NR, num_word=NW, multi_seed=True,
                     with_weights=weights)
    heads, rels, tails = (torch.from_numpy(np.asarray(a, dtype=np.int64)) for a in b[2][:3])
    w = torch.tensor(b[2][5], dtype=torch.float32) if weights else None
    wr = torch.tensor(b[2][6], dtype=torch.float32) if weights else None
    return b, (heads, rels, tails), w, wr


def _rand(rs, *shape):
    return torch.from_numpy(rs.randn(*shape).astype(np.float32))


def _close(got32, want64, scale64):
    err = (got32.double() - want64).abs()
    assert (err <= TOL * scale64 + 1e-30).all(), (err - TOL * scale64).max().item()


@pytest.mark.parametrize("weights", [False, True])
@pytest.mark.parametrize("inverse", [False, True])
def test_aggregate_matches_oracle_reason_layer(weights, inverse):
    b, facts, w, _ = _batch(weights)
    rs = np.random.RandomState(1)
    table = _rand(rs, NR + 1, D)
    ins = _rand(rs, B, I, D)
    prior = torch.softmax(_rand(rs, B, N), 1)
    mats = O.FactMats(b[2], B, N, weights)
    direction = "inv" if inverse else "fwd"
    got = R.aggregate(table.double(), ins.double(), prior.double(), *facts, w, direction)
    scale = R.aggregate_abs(table.double(), ins.double(), prior.double(), *facts, w, direction)
    assert scale.max() > 0
    for j in range(I):
        want = O.reason_layer(mats, prior, ins[:, j, :], table, torch.eye(D), None, inverse)
        _close(want, got[:, j * D:(j + 1) * D], scale[:, j * D:(j + 1) * D])


@pytest.mark.parametrize("weights", [False, True])
def test_type_layer_matches_oracle(weights):
    b, facts, _, wr = _batch(weights)
    rs = np.random.RandomState(2)
    rel_f = _rand(rs, NR + 1, D)
    sd = {"x.kb_self_linear.weight": _rand(rs, D, D) * 0.3, "x.kb_self_linear.bias": _rand(rs, D) * 0.1}
    want = O.type_layer(sd, "x.", b[2], rel_f, B, N, weights).reshape(B * N, D)
    table = rel_f.double() @ sd["x.kb_self_linear.weight"].double().t() + sd["x.kb_self_linear.bias"].double()
    got = R.type_layer(table, *facts, wr, B * N)
    scale = R.type_layer_abs(table, *facts, wr, B * N)
    _close(want, got, scale)
    assert (got == 0).any() and (got > 0).any()          # the relu is exercised on both sides


@pytest.mark.parametrize("weights", [False, True])
def test_rearev_layer_matches_oracle_gnn_step(weights):
    b, facts, w, _ = _batch(weights)
    rs = np.random.RandomState(3)
    Kd = (2 * I + 1) * D
    sd = {"reasoning.rel_linear0.weight": _rand(rs, D, D) * 0.3, "reasoning.rel_linear0.bias": _rand(rs, D) * 0.1,
          "reasoning.e2e_linear0.weight": _rand(rs, D, Kd) * 0.2, "reasoning.e2e_linear0.bias": _rand(rs, D) * 0.1,
          "reasoning.score_func.weight": _rand(rs, 1, D), "reasoning.score_func.bias": _rand(rs, 1)}
    rel_f, rel_fi = _rand(rs, NR + 1, D), _rand(rs, NR + 1, D)
    h = _rand(rs, B, N, D)
    ins = _rand(rs, B, I, D)
    prior = torch.from_numpy(np.asarray(b[4], dtype=np.float32))          # the seed distribution (multi-seed)
    prior = 0.5 * prior + 0.5 * torch.softmax(_rand(rs, B, N), 1)         # and mass everywhere else too
    mask = torch.from_numpy((b[0] != NE).astype(np.float32))
    mats = O.FactMats(b[2], B, N, weights)
    dist, h_new, score = O.rearev_gnn_step(sd, mats, h, prior, ins, rel_f, rel_fi, mask, 0)

    Wr, br = sd["reasoning.rel_linear0.weight"].double(), sd["reasoning.rel_linear0.bias"].double()
    tf, ti = rel_f.double() @ Wr.t() + br, rel_fi.double() @ Wr.t() + br
    We, be = sd["reasoning.e2e_linear0.weight"].double(), sd["reasoning.e2e_linear0.bias"].double()
    ws = sd["reasoning.score_func.weight"].double().view(-1)
    args = (h.reshape(B * N, D).double(), prior.double(), tf, ti, ins.double(), We, be)
    y, s = R.rearev_layer(*args, ws, facts, w)
    scale = R.rearev_layer_scale(*args, facts, w)
    _close(h_new.reshape(B * N, D), y, scale)
    assert (y == 0).any() and (y > 0).any()
    live = mask.view(-1) > 0
    s_scale = scale @ ws.abs()
    want_s = s + sd["reasoning.score_func.bias"].double()
    _close(score.view(-1)[live], want_s[live], s_scale[live] + 1)
    logits = torch.where(live, want_s, torch.full_like(want_s, -1e11)).view(B, N)
    assert torch.allclose(dist.double(), torch.softmax(logits, 1), rtol=1e-4, atol=1e-7)


def test_possible_mass_threshold():
    """possible: rows whose prior mass over in-edges (tail direction) exceeds 1e-10, nsm_gnn.py:101-103."""
    heads = torch.tensor([0, 1, 2, 3, 0])
    tails = torch.tensor([1, 2, 3, 3, 4])
    rels = torch.zeros(5, dtype=torch.int64)
    prior = torch.tensor([1.2e-10, 0.9e-10, 0.0, 0.5, 0.0], dtype=torch.float64)
    mask, mass = R.possible(prior, (heads, rels, tails), None, 5)
    assert mask.tolist() == [0.0, 1.0, 0.0, 1.0, 1.0]
    w = torch.tensor([0.5, 1.0, 1.0, 1.0, 2.0])
    mask, mass = R.possible(prior, (heads, rels, tails), w, 5)
    assert mask.tolist() == [0.0, 0.0, 0.0, 1.0, 1.0]      # 0.25 * 1.2e-10 drops below, 4 * 1.2e-10 stays above
