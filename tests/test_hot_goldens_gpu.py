"""GPU parity at the HOT shapes against arrays produced by the unmodified reference (tests/golden/hot/*.npz, generator:
tests/golden/make_golden_hot.py): entity_dim 200 with N >= 64 -- the |v|-accumulating aggregation kernel, the K = 1040
tensor-core GEMM and the sparse-prior / frontier path --, the full-size cfg2 batch bench.py times (B = 64) and the cfg5
stress graph (D = 400).  Weights are rebuilt from synthetic.seeded_state_dict; the files hold reference outputs only."""
import json
import os

import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
import rank_check
from gnn_rag_b200 import batching, evaluate, ops, synthetic as S

pytestmark = pytest.mark.gpu
DEV = "cuda"
HOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hot")
RTOL = 1e-3      # north_star bound on pred_dist (relative, fp32)


class Hot:
    def __init__(self, name):
        z = np.load(os.path.join(HOT, name + ".npz"))
        self.meta = json.loads(str(z["meta_json"]))
        self.out = {k[4:]: z[k] for k in z.files if k.startswith("out/")}
        self.layer = {k[6:]: z[k] for k in z.files if k.startswith("layer/")}
        m = self.meta
        v = m["vocab"]
        self.vocab = v
        self.args = dict(m["args"], use_cuda=True)
        self.batch = S.make_batch(num_entity=v["num_entity"], num_relation=v["num_relation"], num_word=v["num_word"],
                                  test=True, **m["batch"])
        self.sd = {k: torch.from_numpy(a) for k, a in
                   S.seeded_state_dict(m["shapes"], seed=m["wseed"],
                                       sharpen=tuple(m["sharpen"]) if m["sharpen"] else None).items()}

    def model(self):
        v = self.vocab
        m = G.ReaRev(dict(self.args), v["num_entity"], v["num_relation"], v["num_word"])
        m.load_state_dict(self.sd, strict=True)
        return m.to(DEV).eval()

    def ref_lists(self):
        """[(node, entity, prob)] per question from the stored reference candidate lists (entity ids + fp32 probs): the
        node index is recovered through the reference distribution (first unused node with that entity and prob)."""
        le, pd = self.batch[0], self.out["pred_dist"]
        out, o = [], 0
        for b, n in enumerate(self.out["cand_len"].tolist()):
            ids = self.out["cand_ids"][o:o + n]
            pr = self.out["cand_probs"][o:o + n].astype(np.float32)
            o += n
            used, rows = set(), []
            cand = {}
            for node in np.nonzero(np.isin(le[b], ids))[0].tolist():
                cand.setdefault((int(le[b, node]), float(pd[b, node])), []).append(node)
            for e, p in zip(ids.tolist(), pr.tolist()):
                node = next(x for x in cand[(e, p)] if x not in used)
                used.add(node)
                rows.append((node, e, p))
            out.append(rows)
        return out


def _check_dist(got, want, tag, logits=False):
    """``logits=False``: every probability > 1e-12 within RTOL relative.  ``logits=True`` (the sharpened full-size
    cases, whose logits span hundreds of units): the north_star bound is on the LOGITS -- |log p - log p_ref| within
    RTOL of the logit range of the question; the probability-relative error (= absolute logit error) is reported and
    returned so that the ranking comparison can use it as its near-tie margin."""
    got, want = got.double().cpu(), torch.from_numpy(np.asarray(want)).double()
    big = want > 1e-12
    rel = ((got - want).abs()[big] / want[big]).max().item() if big.any() else 0.0
    small = (got - want).abs()[~big].max().item() if (~big).any() else 0.0
    print("%s: max relative error %.2e over %d entries > 1e-12, max abs error %.2e on the rest" % (
        tag, rel, int(big.sum()), small))
    assert small < 1e-12, (tag, small)
    if not logits:
        assert rel < RTOL, (tag, rel)
        return rel
    ok = (want > 1e-30) & (got > 0)
    assert bool((ok == (want > 1e-30)).all())
    lg, lw = got.clamp_min(1e-300).log(), want.clamp_min(1e-300).log()
    span = torch.where(ok, lw, torch.zeros_like(lw)).abs().amax(dim=-1, keepdim=True).clamp_min(1.0)
    lerr = (torch.where(ok, (lg - lw).abs(), torch.zeros_like(lw)) / span).max().item()
    print("%s: max logit error relative to the question's logit range %.2e" % (tag, lerr))
    assert lerr < RTOL, (tag, lerr)
    return rel


@pytest.mark.parametrize("name", ["d200_rand", "d200_sharp", "d200_norm"])
def test_hot_shape_forward_vs_reference(name):
    h = Hot(name)
    m = h.model()
    B, N = h.batch[0].shape
    assert ops.aggregate_dual_abs_supported(N, 200, 208, h.vocab["num_relation"] + 1)   # the hot kernels are on this path
    loss, pred, dist, _ = m(h.batch[:7])
    _check_dist(dist, h.out["pred_dist"], name + " pred_dist")
    hist = torch.stack(m.dist_history[1:])
    _check_dist(hist, h.out["dist_history"], name + " dist_history")
    hf = m.reasoning.h_view.reshape(B, N, -1).cpu()
    want_h = torch.from_numpy(h.out["h_final"])
    assert (hf - want_h).abs().max().item() <= 1e-4 * (want_h.abs().max().item() + 1e-12)
    assert abs(float(loss) - float(h.out["loss"])) < 1e-3 * max(1.0, abs(float(h.out["loss"])))
    got, _ = evaluate.retrieve(dist, m.last_batch, h.vocab["num_entity"], h.args["eps"])
    stats = rank_check.report("hot/" + name, rank_check.compare(got, h.ref_lists(), h.out["pred_dist"]))
    if name != "d200_rand":                                   # peaked: ids strictly identical
        assert stats["swaps"] == 0 and stats["cut_moves"] == 0


@pytest.mark.parametrize("name", ["d200_rand", "d200_sharp", "d200_norm"])
def test_abs_aggregation_kernel_vs_reference_reason_layer(name):
    """gr_aggregate_dual_abs (csrc/aggregate_abs.cu) against reason_layer / reason_layer_inv outputs recorded from the
    reference at D = 200 (reasongnn.py:61-116): every instruction, both directions, dense prior."""
    h = Hot(name)
    L = h.layer
    B, N = h.batch[0].shape
    I, D = L["ins"].shape[1], 200
    R1 = h.vocab["num_relation"] + 1
    normalized = bool(h.args["normalized_gnn"])
    db = batching.stage_batch(h.batch[:7], torch.device(DEV), R1, normalized, False)
    g = db.graph
    wt, wh = (g.w_t, g.w_h) if normalized else (None, None)
    W = h.sd["reasoning.rel_linear1.weight"].to(DEV)
    bias = h.sd["reasoning.rel_linear1.bias"].to(DEV)
    tab = torch.cat([torch.nn.functional.linear(torch.from_numpy(L["rel_features"]).to(DEV), W, bias),
                     torch.nn.functional.linear(torch.from_numpy(L["rel_features_inv"]).to(DEV), W, bias)])
    pn = ops.pad_table256(tab.contiguous())
    prior = torch.from_numpy(L["dist"]).to(DEV)
    ins = torch.from_numpy(L["ins"]).to(DEV)
    Kp = (208 * (2 * I + 1) + 63) // 64 * 64
    for mode in (0, 1, 2, 3):                                 # per-tile / round-1 shape / default shape / gather4
        ops.set_option("agg_abs_ws", mode)
        try:
            planes = [torch.zeros(B * N, Kp, dtype=torch.bfloat16, device=DEV) for _ in range(2)]
            ops.aggregate_dual_abs(g, prior, pn[:R1], pn[R1:], ins, tuple(planes), 208, 208, wt, wh)
        finally:
            ops.set_option("agg_abs_ws", 2)
        y = (planes[0].float() + planes[1].float())[:, 208:208 * (2 * I + 1)].view(B * N, I, 2, 208)
        for j in range(I):
            for d, key in ((0, "neighbor_rep"), (1, "neighbor_rep_inv")):
                want = torch.from_numpy(L[key][j]).to(DEV).reshape(B * N, D)
                got = y[:, j, d, :D]
                err = (got - want).abs().max().item()
                assert err <= 2e-5 * want.abs().max().item() + 1e-30, (name, mode, j, d, err)
                assert ((want == 0) <= (got == 0)).all()      # exact zeros stay exact zeros
                assert (y[:, j, d, D:] == 0).all()


def test_cfg2_full_size_vs_reference():
    """BASELINE configs[1] at full size (B = 64, N = 2000, F = 512 000, D = 200, 3 x 3 layers): the exact batch and
    architecture bench.py times, eager and CUDA-graph paths, against the reference's CPU forward."""
    h = Hot("cfg2_full")
    m = h.model()
    loss, pred, dist, _ = m(h.batch[:7])
    rel = _check_dist(dist, h.out["pred_dist"], "cfg2_full pred_dist", logits=True)
    assert abs(float(loss) - float(h.out["loss"])) < 1e-3 * max(1.0, abs(float(h.out["loss"])))
    keep = h.out["h_final"].shape[1]
    hf = m.reasoning.h_view.reshape(64, 2000, -1)[:, :keep].cpu()
    want_h = torch.from_numpy(h.out["h_final"])
    assert (hf - want_h).abs().max().item() <= 1e-4 * (want_h.abs().max().item() + 1e-12)
    got, _ = evaluate.retrieve(dist, m.last_batch, h.vocab["num_entity"], h.args["eps"])
    # near-tie margin = twice the measured probability error of this forward (fp32 logits of magnitude ~1e2)
    rank_check.report("hot/cfg2_full", rank_check.compare(got, h.ref_lists(), h.out["pred_dist"],
                                                          margin=max(2e-5, 2 * rel)))
    gs = G.GraphedStep(m, h.vocab["num_entity"])
    out = gs(h.batch[:7])
    assert torch.equal(out.pred_dist, dist)                   # graph replay == eager, bit for bit


def test_cfg5_full_size_vs_reference():
    """BASELINE configs[4]: one 100k-node / 1.1M-fact graph, D = 400."""
    h = Hot("cfg5_full")
    m = h.model()
    loss, pred, dist, _ = m(h.batch[:7])
    rel = _check_dist(dist, h.out["pred_dist"], "cfg5_full pred_dist", logits=True)
    got, _ = evaluate.retrieve(dist, m.last_batch, h.vocab["num_entity"], h.args["eps"])
    rank_check.report("hot/cfg5_full", rank_check.compare(got, h.ref_lists(), h.out["pred_dist"],
                                                          margin=max(2e-5, 2 * rel)))
