"""GPU parity tests proper: the CUDA path (through the C ABI) vs the oracle and vs the golden vectors the
unmodified reference produced.  Tolerances: fp32 results within 1e-3 relative of the reference (the
north_star bound; observed error is ~1e-6), index / id work bit-exact."""
import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import batching, evaluate, ops, synthetic as S
import rank_check
from golden_io import Golden, names
from oracle import kgqa_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
RTOL = 1e-3          # north_star: pred_dist within 1e-3 relative fp32
TIGHT = 2e-5         # what the fp32 kernels actually achieve


def rel_err(a, b, floor=1e-30):
    a, b = a.double(), b.double()
    return ((a - b).abs() / b.abs().clamp_min(floor)).max().item()


def max_err(a, b):
    """max-norm relative error (elementwise relative error is meaningless for entries that cancel to ~0)."""
    a, b = a.double(), b.double()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def assert_ranking_equivalent(got, ref, ref_dist, margin=2e-5, name="?"):
    """See tests/rank_check.py: asserts that only reference near-ties (< margin relative) change places, prints and
    records the counts, returns the number of swapped positions."""
    stats = rank_check.compare(got, ref, ref_dist, margin)
    rank_check.report(name, stats)
    return stats["swaps"] + stats["cut_moves"]


def build_model(g, device=DEV):
    cls = G.NSM if g.args["model_name"] == "NSM" else G.ReaRev
    args = dict(g.args)
    args["use_cuda"] = True
    m = cls(args, g.num_entity, g.num_relation, g.num_word)
    m.load_state_dict(g.sd, strict=True)
    m = m.to(device).eval()
    if g.rel_texts is not None:                               # gnn/train_model.py:62-64
        m.encode_rel_texts(g.rel_texts, g.rel_texts_inv)
    return m


def stage(batch, R1, normalized=False, norm_rel=False):
    return batching.stage_batch(batch, torch.device(DEV), R1, normalized, norm_rel)


# ------------------------------------------------------------------ CSR batching ------------------
def np_csr(keys, other, rels, Nt):
    order = np.argsort(keys, kind="stable")
    rowptr = np.zeros(Nt + 1, dtype=np.int64)
    np.add.at(rowptr, keys + 1, 1)
    return np.cumsum(rowptr), other[order], rels[order], order


@pytest.mark.parametrize("kw", [dict(B=3, N=50, E=150), dict(B=2, N=300, E=6000, powerlaw=True),
                                dict(B=4, N=64, E=0), dict(B=1, N=5000, E=60000, powerlaw=True)])
def test_csr_build_stable_and_exact(kw):
    b = S.make_batch(11, num_entity=1000, num_relation=40, num_word=100, with_weights=False, **kw)
    heads, rels, tails = b[2][0], b[2][1], b[2][2]
    B, N = b[0].shape
    db = stage(b, 41)
    db.graph.check_status()
    g = db.graph
    F = len(heads)
    for keys, other, rp, src, rel, fact in ((tails, heads, g.rowptr_t, g.src_t, g.rel_t, g.fact_t),
                                            (heads, tails, g.rowptr_h, g.src_h, g.rel_h, g.fact_h)):
        w_rp, w_src, w_rel, w_order = np_csr(keys, other, rels, B * N)
        assert np.array_equal(rp[: B * N + 1].cpu().numpy(), w_rp)
        assert np.array_equal(src[:F].cpu().numpy(), w_src)
        assert np.array_equal(rel[:F].cpu().numpy(), w_rel)
        assert np.array_equal(fact[:F].cpu().numpy(), w_order)      # stable: original fact order in a row


def test_csr_build_int32_input_and_bad_ids():
    b = S.make_batch(12, B=2, N=40, E=100, num_entity=1000, num_relation=40, num_word=100,
                     with_weights=False)
    h, r, t = (torch.from_numpy(x).to(torch.int32).to(DEV) for x in b[2][:3])
    g32 = ops.csr_build(h, r, t, 2, 40, 41)
    g64 = stage(b, 41).graph
    assert torch.equal(g32.src_t[: g32.F], g64.src_t[: g64.F])
    h[3] = 10_000                                                     # out of range -> status flag
    bad = ops.csr_build(h, r, t, 2, 40, 41)
    with pytest.raises(RuntimeError, match="outside"):
        bad.check_status()


# ------------------------------------------------------------------ dense linear -------------------
@pytest.mark.parametrize("M,N,K", [(300, 200, 1000), (41, 50, 50), (1000, 32, 160), (129, 65, 17)])
def test_linear_vs_torch(M, N, K):
    torch.manual_seed(0)
    A = torch.randn(M, K, device=DEV)
    W = torch.randn(N, K, device=DEV) / K ** 0.5
    b = torch.randn(N, device=DEV)
    want = torch.relu(A.double() @ W.double().T + b.double())
    got = ops.linear(A, W, b, relu=True)
    assert (got.double() - want).abs().max().item() < 1e-4
    add = torch.randn(M, N, device=DEV)
    got2 = ops.linear(A, W, None, addend=add, addend_rows=M // 2)
    want2 = A.double() @ W.double().T
    want2[: M // 2] += add[: M // 2].double()
    assert (got2.double() - want2).abs().max().item() < 1e-4


@pytest.mark.parametrize("M,N,K", [(300, 200, 1000), (1000, 200, 1000), (129, 64, 64), (4000, 50, 250),
                                   (257, 32, 160), (128, 256, 520), (5, 16, 8)])
def test_linear_tc_split_bf16_vs_fp64(M, N, K):
    """wgmma split-bf16 x3 GEMM: fp32-class accuracy (error ~1e-5 of the row scale), TMA OOB tails."""
    torch.manual_seed(1)
    big = torch.empty(M, K + 24, device=DEV).normal_()
    A = big[:, 8:8 + K] if (K % 4 == 0) else big[:, :K]         # strided row view (lda > K)
    W = torch.randn(N, K, device=DEV) / K ** 0.5
    b = torch.randn(N, device=DEV)
    want = torch.relu(A.double() @ W.double().T + b.double())
    out = torch.full((M, N + 8), -7.0, device=DEV)
    got = ops.linear_tc(A, W, b, relu=True, out=out[:, :N])
    scale = (A.double().abs() @ W.double().abs().T).max().item()
    assert (got.double() - want).abs().max().item() < 2e-5 * scale
    assert (out[:, N:] == -7.0).all()                            # nothing written outside the view
    simt = ops.linear(A, W, b, relu=True)
    assert (got - simt).abs().max().item() < 2e-5 * scale


@pytest.mark.parametrize("tma_store", [1, 0])
@pytest.mark.parametrize("bk", [32, 64])
@pytest.mark.parametrize("cluster", [1, 2])
def test_linear_tc_planes_cluster_variants(cluster, bk, tma_store):
    """Planes-in GEMM (persistent, register accumulators) with and without W multicast across a CTA pair;
    odd tile counts, fused score dots and plane outputs."""
    torch.manual_seed(2)
    ops.set_option("tc_cluster", cluster)
    ops.set_option("tc_bk", bk)
    ops.set_option("tc_tma_store", tma_store)
    try:
        for M, N, K in [(128 * 5 + 37, 200, 1000), (128 * 300, 200, 1000), (77, 64, 96), (128 * 9, 32, 160)]:
            A = torch.randn(M, K, device=DEV)
            W = torch.randn(N, K, device=DEV) / K ** 0.5
            b = torch.randn(N, device=DEV)
            ws = torch.randn(N, device=DEV)
            Kp = (K + 63) // 64 * 64
            hi = torch.empty(M, Kp, dtype=torch.bfloat16, device=DEV)
            lo = torch.empty(M, Kp, dtype=torch.bfloat16, device=DEV)
            ops.split_bf16(A, hi, lo)
            out = torch.empty(M, N, device=DEV)
            ohi = torch.zeros(M, (N + 8 + 7) // 8 * 8, dtype=torch.bfloat16, device=DEV)
            olo = torch.zeros_like(ohi)
            dots = torch.empty(2 * M, device=DEV)
            ops.linear_tc_planes(hi, lo, K, W, b, out=out, out_planes=(ohi, olo), w_score=ws, dots=dots)
            want = torch.relu(A.double() @ W.double().T + b.double())
            scale = (A.double().abs() @ W.double().abs().T).max().item()
            assert (out.double() - want).abs().max().item() < 2e-5 * scale
            rec = ohi[:, :N].double() + olo[:, :N].double()
            assert (rec - out.double()).abs().max().item() < 1e-5 * (out.abs().max().item() + 1e-9)
            assert (ohi[:, N:] == 0).all() and (olo[:, N:] == 0).all()
            dsum = dots.view(2, M).double().sum(0)
            assert (dsum - out.double() @ ws.double()).abs().max().item() < 1e-4 * (scale + 1)
    finally:                                      # the documented defaults (linear_tc.cu)
        ops.set_option("tc_cluster", 1)
        ops.set_option("tc_bk", 32)
        ops.set_option("tc_tma_store", 1)


def test_forward_with_tc_linear_matches_golden():
    prev, ops.TC_LINEAR = ops.TC_LINEAR, True
    try:
        for name in ("rearev_sharp_ties", "rearev_small", "rearev_d50_pads", "nsm_reason_kb"):
            g = Golden(name)
            m = build_model(g)
            _, _, dist, _ = m(g.batch)
            ref = torch.from_numpy(g.out["pred_dist"]).to(DEV)
            assert rel_err(dist, ref, 1e-30) < RTOL
            if name == "rearev_sharp_ties":
                assert torch.equal(dist[:, 4], dist[:, 5])       # twins still tie exactly
    finally:
        ops.TC_LINEAR = prev


# ------------------------------------------------------------------ aggregation kernel -------------
@pytest.mark.parametrize("name", names("rearev"))
@pytest.mark.parametrize("tma", [0, 1])
def test_aggregate_vs_reference_reason_layer(name, tma):
    """Isolated reason_layer / reason_layer_inv call recorded from the reference (golden layer/*)."""
    g = Golden(name)
    L = g.layer
    B, N = g.batch[0].shape
    D = L["ins"].shape[1]
    db = stage(g.batch, g.num_relation + 1, g.args["normalized_gnn"])
    lin_w = g.sd["reasoning.rel_linear0.weight"].to(DEV)
    lin_b = g.sd["reasoning.rel_linear0.bias"].to(DEV)
    pe = g.sd["reasoning.pos_emb0.weight"].to(DEV) if g.args.get("pos_emb") else None
    pei = g.sd["reasoning.pos_emb_inv0.weight"].to(DEV) if g.args.get("pos_emb") else None
    nrel = pe.shape[0] if pe is not None else 0
    tf = ops.linear(torch.from_numpy(L["rel_features"]).to(DEV), lin_w, lin_b, addend=pe, addend_rows=nrel)
    ti = ops.linear(torch.from_numpy(L["rel_features_inv"]).to(DEV), lin_w, lin_b, addend=pei,
                    addend_rows=nrel)
    prior = torch.from_numpy(L["dist"]).to(DEV)
    ins = torch.from_numpy(L["ins"]).to(DEV).view(B, 1, D)
    gr = db.graph
    ops.set_option("agg_tma", tma)
    try:
        nb = ops.aggregate(gr, "fwd", prior, tf, ins, w=gr.w_t)
        nbi = ops.aggregate(gr, "inv", prior, ti, ins, w=gr.w_h)
        out = torch.zeros(B * N, 3 * D, device=DEV)
        ops.aggregate_dual(gr, prior, tf, ti, ins, out, D, gr.w_t, gr.w_h)
    finally:
        ops.set_option("agg_tma", 0)
    want = torch.from_numpy(L["neighbor_rep"]).view(B * N, D).to(DEV)
    wanti = torch.from_numpy(L["neighbor_rep_inv"]).view(B * N, D).to(DEV)
    scale = want.abs().max().item() + 1e-12
    assert (nb - want).abs().max().item() <= TIGHT * scale
    assert (nbi - wanti).abs().max().item() <= TIGHT * (wanti.abs().max().item() + 1e-12)
    assert torch.equal(out[:, D:2 * D], nb) and torch.equal(out[:, 2 * D:], nbi)   # dual == 2 singles
    assert (out[:, :D] == 0).all()                                                  # untouched slot


@pytest.mark.parametrize("D,I", [(200, 2), (200, 3), (50, 2), (33, 1), (400, 2), (64, 5)])
def test_aggregate_vs_oracle_shapes(D, I):
    """All vector widths (float4 / float2 / scalar), instruction counts (incl. I>4 -> two launches),
    ragged + multi-seed + hubs, one-hot prior (zero-skip)."""
    rs = np.random.RandomState(5)
    B, N, R = 3, 200, 30
    b = S.make_batch(21, B=B, N=N, E=900, num_entity=1000, num_relation=R, num_word=50,
                     n_real="ragged", powerlaw=True)
    db = stage(b, R + 1, normalized=True)
    gr = db.graph
    table = torch.from_numpy(rs.randn(R + 1, D).astype(np.float32)).to(DEV)
    ins = torch.from_numpy(rs.randn(B, I, D).astype(np.float32)).to(DEV)
    mats = O.FactMats(b[2], B, N, True)
    for prior_kind in ("dense", "onehot"):
        if prior_kind == "dense":
            prior = torch.softmax(torch.from_numpy(rs.randn(B, N).astype(np.float32)), 1)
        else:
            prior = torch.from_numpy(b[4].astype(np.float32))
        out = ops.aggregate(gr, "fwd", prior.to(DEV), table, ins, w=gr.w_t)
        W = torch.eye(D)
        for j in range(I):
            want = O.reason_layer(mats, prior, ins[:, j, :].cpu(), table.cpu(), W, None, False)
            got = out[:, j * D:(j + 1) * D].cpu()
            assert (got - want).abs().max().item() <= TIGHT * (want.abs().max().item() + 1e-12)


def test_aggregate_deterministic_and_tma_identical():
    b = S.make_batch(31, B=8, N=500, E=2500, num_entity=1000, num_relation=60, num_word=50,
                     powerlaw=True, with_weights=False)
    db = stage(b, 61)
    rs = np.random.RandomState(1)
    D, I = 200, 2
    tf = torch.from_numpy(rs.randn(61, D).astype(np.float32)).to(DEV)
    ti = torch.from_numpy(rs.randn(61, D).astype(np.float32)).to(DEV)
    ins = torch.from_numpy(rs.randn(8, I, D).astype(np.float32)).to(DEV)
    prior = torch.softmax(torch.from_numpy(rs.randn(8, 500).astype(np.float32)), 1).to(DEV)
    outs = []
    for tma in (0, 0, 1):
        ops.set_option("agg_tma", tma)
        out = torch.empty(8 * 500, 5 * D, device=DEV)
        ops.aggregate_dual(db.graph, prior, tf, ti, ins, out, D)
        outs.append(out[:, D:].clone())
    ops.set_option("agg_tma", 0)
    assert torch.equal(outs[0], outs[1])          # run-to-run bit identical (atomic-free)
    assert torch.equal(outs[0], outs[2])          # TMA-staged variant bit identical to plain staging


@pytest.mark.parametrize("ws", [2, 1, 0, 3])
@pytest.mark.parametrize("I,normalized", [(2, False), (2, True), (1, False), (3, True), (5, False)])
def test_aggregate_abs_kernel_matches_generic_kernel(I, normalized, ws):
    """|v|-accumulating aggregation (csrc/aggregate_abs.cu) == the generic kernel's planes:
    hubs that overflow the staged edge slice, ragged questions, edge weights, a one-hot prior (zero rows exact),
    I > 4 (two launches), persistent and one-CTA-per-tile builds.  Run-to-run bit identical."""
    B, N, D, R = 5, 700, 200, 60
    b = S.make_batch(41, B=B, N=N, E=5000, num_entity=5000, num_relation=R, num_word=50, n_real="ragged",
                     powerlaw=True)
    db = stage(b, R + 1, normalized=normalized)
    g = db.graph
    wt, wh = (g.w_t, g.w_h) if normalized else (None, None)
    rs = np.random.RandomState(2)
    tab = torch.from_numpy(rs.randn(2 * (R + 1), D).astype(np.float32)).to(DEV)
    tab[3].abs_()                                            # a non-negative table row
    tf, ti = tab[: R + 1], tab[R + 1:]
    ins = torch.from_numpy(rs.randn(B, I, D).astype(np.float32)).to(DEV)
    pn = ops.pad_table256(tab)
    pf, pi = pn[: R + 1], pn[R + 1:]
    assert ops.aggregate_dual_abs_supported(N, D, 208, R + 1)
    Kp = (208 * (2 * I + 1) + 63) // 64 * 64
    ops.set_option("agg_abs_ws", ws)       # persistent warp-specialised kernel / one CTA per tile
    try:
        for kind in ("dense", "onehot"):
            prior = (torch.softmax(torch.from_numpy(rs.randn(B, N).astype(np.float32)), 1) if kind == "dense"
                     else torch.from_numpy(b[4].astype(np.float32))).to(DEV)
            ref = [torch.full((B * N, Kp), 7.0, dtype=torch.bfloat16, device=DEV) for _ in range(2)]
            ops.aggregate_dual(g, prior, tf, ti, ins, None, 208, wt, wh, planes=tuple(ref), seg_pitch=208)
            outs = []
            for _ in range(2):
                got = [torch.full((B * N, Kp), 7.0, dtype=torch.bfloat16, device=DEV) for _ in range(2)]
                ops.aggregate_dual_abs(g, prior, pf, pi, ins, tuple(got), 208, 208, wt, wh)
                outs.append(got)
            assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
            got = outs[0]
            assert (got[0][:, :208] == 7.0).all()            # the h segment is not touched
            a = got[0][:, 208:208 * (2 * I + 1)].float() + got[1][:, 208:208 * (2 * I + 1)].float()
            r = ref[0][:, 208:208 * (2 * I + 1)].float() + ref[1][:, 208:208 * (2 * I + 1)].float()
            assert (a - r).abs().max().item() <= 2e-5 * r.abs().max().item()   # two hi+lo roundings of ~2^-18 each
            assert ((r == 0) <= (a == 0)).all()               # exact zeros stay exact zeros
            seg = a.view(B * N, 2 * I, 208)
            assert (seg[:, :, 200:] == 0).all()               # padding columns written as zeros
    finally:
        ops.set_option("agg_abs_ws", 2)


def test_type_layer_vs_oracle():
    for name in ("rearev_small", "rearev_norm"):
        g = Golden(name)
        B, N = g.batch[0].shape
        D = g.args["entity_dim"]
        db = stage(g.batch, g.num_relation + 1, False, g.args["norm_rel"])
        got = torch.from_numpy(g.out["h0"]).view(B * N, D)
        m = build_model(g)
        rel_f = m.get_rel_feature()
        out = torch.empty(B * N, D, device=DEV)
        m.type_layer(db.graph, rel_f, out)
        assert (out.cpu() - got).abs().max().item() <= TIGHT * (got.abs().max().item() + 1e-12)


# ------------------------------------------------------------------ scoring / seed pick ------------
def test_score_softmax_vs_torch_incl_all_pad_row():
    torch.manual_seed(3)
    B, N, D = 5, 300, 200
    X = torch.randn(B * N, 5 * D, device=DEV)
    w = torch.randn(D, device=DEV)
    bias = torch.randn(1, device=DEV)
    mask = (torch.rand(B, N, device=DEV) > 0.3).float()
    mask[2] = 0                                               # all-padding question -> uniform 1/N
    got = ops.score_softmax(X[:, :D], w, bias, mask.view(-1), B, N)
    score = (X[:, :D] @ w + bias).view(B, N) + (1 - mask) * O.VERY_NEG_NUMBER
    want = torch.softmax(score, 1)
    assert rel_err(got, want, 1e-30) < 1e-4
    assert torch.allclose(got[2], torch.full((N,), 1.0 / N, device=DEV))
    live_rows = mask.sum(1) > 0                               # masked nodes of a question with a live node: exactly 0
    assert (got[live_rows][mask[live_rows] == 0] == 0).all()


def test_seed_retrieve_vs_bmm():
    torch.manual_seed(4)
    B, N, D = 4, 700, 200
    h = torch.randn(B * N, 3 * D, device=DEV)
    seed = torch.zeros(B, N, device=DEV)
    seed[0, 0] = 1.0
    seed[1, [0, 1, 2]] = 1 / 3
    seed[2, [5, 300, 699]] = torch.tensor([0.2, 0.3, 0.5], device=DEV)
    got = ops.seed_retrieve(seed, h[:, :D], B, N, D)
    want = torch.bmm(seed.unsqueeze(1), h[:, :D].reshape(B, N, D)).squeeze(1)
    assert (got - want).abs().max().item() < 1e-5
    assert (got[3] == 0).all()


# ------------------------------------------------------------------ fused question-side kernels -----
@pytest.mark.parametrize("B,Q,D,I", [(5, 12, 200, 2), (3, 7, 50, 3), (2, 40, 64, 1)])
def test_instructions_kernel_vs_torch_chain(B, Q, D, I):
    """gr_instructions == LSTMInstruction.get_instruction applied num_ins times (base_encoder.py:73-114)."""
    from gnn_rag_b200.modules import LSTMInstruction
    torch.manual_seed(11)
    nw = 30
    emb = torch.nn.Embedding(nw + 1, 16, padding_idx=nw)
    ins = LSTMInstruction(dict(num_ins=I, entity_dim=D, word_dim=16), emb, nw).to(DEV).eval()
    text = torch.randint(0, nw, (B, Q), device=DEV)
    text[0, Q // 2:] = nw                                     # padded tail
    text[B - 1, :] = nw                                       # all-pad question
    with torch.no_grad():
        got = ins(text)                                       # fused kernel
        ins.init_reason(text)
        ri, want = ins.relational_ins, []
        for i in range(I):
            ri, _ = ins.get_instruction(ri, step=i)
            want.append(ri)
        want = torch.stack(want, 1)
    assert got.shape == (B, I, D)
    assert max_err(got, want) < 1e-5


@pytest.mark.parametrize("B,Q,D,W", [(64, 12, 200, 300), (5, 7, 50, 16), (9, 30, 256, 64), (3, 4, 33, 8)])
def test_lstm_cluster_kernel_vs_cudnn(B, Q, D, W):
    torch.manual_seed(14)
    lstm = torch.nn.LSTM(input_size=W, hidden_size=D, batch_first=True).to(DEV)
    x = torch.randn(B, Q, W, device=DEV)
    with torch.no_grad():
        z = torch.zeros(1, B, D, device=DEV)
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            want, (hn, _) = lstm(x, (z, z.clone()))
        gx = torch.nn.functional.linear(x, lstm.weight_ih_l0, lstm.bias_ih_l0)
        got = ops.lstm_forward(gx, lstm.weight_hh_l0, lstm.bias_hh_l0)
    assert max_err(got, want) < 3e-5        # cuDNN's cell kernel uses its own sigmoid/tanh formulation
    assert max_err(got[:, -1], hn[0]) < 3e-5


@pytest.mark.parametrize("B,N,D,I", [(4, 700, 200, 2), (3, 1500, 50, 3), (19, 700, 200, 2), (64, 700, 50, 3)])
def test_query_reform_kernel_vs_torch_modules(B, N, D, I):
    from gnn_rag_b200.modules import QueryReform
    torch.manual_seed(12)
    reforms = [QueryReform(D).to(DEV) for _ in range(I)]
    h = torch.randn(B * N, D, device=DEV)
    seed = torch.zeros(B, N, device=DEV)
    seed[0, 0] = 1.0
    seed[1, [0, 1, N - 1]] = 1 / 3
    seed[2, [5, 300, 699]] = torch.tensor([0.2, 0.3, 0.5], device=DEV)   # question 3+ : no seed at all
    x = torch.randn(B, I, D, device=DEV)
    with torch.no_grad():
        got = ops.query_reform(seed, h, x, [r.fusion.r.weight for r in reforms],
                               [r.fusion.g.weight for r in reforms], B, N)
        want = torch.stack([reforms[j](x[:, j], h, seed, B, N) for j in range(I)], 1)
    assert max_err(got, want) < 1e-5


def test_kl_loss_pred_kernel_vs_torch():
    torch.manual_seed(13)
    B, N = 6, 2000
    dist = torch.softmax(torch.randn(B, N, device=DEV) * 3, 1)
    dist[1, 7] = dist[1, 900] = dist[1].max() + 0.1           # tie -> lowest index
    teacher = torch.zeros(B, N, device=DEV)
    teacher[0, [3, 4]] = 1.0
    teacher[1, 10] = 1.0
    teacher[2, torch.arange(0, N, 7)] = 1.0
    teacher[4, 1999] = 1.0                                    # questions 3 and 5: no answer -> case_valid 0
    loss, pred = ops.kl_loss_pred(dist, teacher)
    m = G.ReaRev.__new__(G.ReaRev)
    m.loss_type = "kl"
    valid = (teacher.sum(1, keepdim=True) > 0).float()
    want = G.models.BaseModel.calc_loss_label(m, dist, teacher, valid)
    assert abs(loss.item() - want.item()) <= 1e-5 * abs(want.item())
    assert pred.tolist() == torch.max(dist.cpu(), 1)[1].tolist()
    assert pred[1].item() == 7


# ------------------------------------------------------------------ ranking (bit exact) ------------
@pytest.mark.parametrize("name", names())
def test_rank_candidates_matches_reference_lists(name):
    g = Golden(name)
    db = stage(g.batch, g.num_relation + 1)
    pd = torch.from_numpy(g.out["pred_dist"]).to(DEV)
    got, _ = evaluate.retrieve(pd, db, g.num_entity, g.args["eps"])
    ids, probs = g.cand_lists()
    assert [r.ent.tolist() for r in got] == ids
    assert [r.prob.astype(np.float64).tolist() for r in got] == probs


def test_rank_candidates_large_with_ties():
    rs = np.random.RandomState(9)
    B, N = 3, 6000                                           # > 4096 survivors -> global-memory sort path
    p = rs.rand(B, N).astype(np.float32)
    p[:, ::7] = p[:, 3:4]                                     # many exact ties
    p = p / p.sum(1, keepdims=True)
    le = rs.randint(0, 1000, size=(B, N)).astype(np.int64)
    le[:, -50:] = 1000
    qe = np.zeros((B, N)); qe[:, 0] = 1.0
    want = O.rank_candidates(le, qe, p, 1000, 0.95)
    db = batching.DeviceBatch()
    db.B, db.N = B, N
    db.local_entity = torch.from_numpy(le).to(DEV)
    db.query_entities = torch.from_numpy(qe).float().to(DEV)
    got, _ = evaluate.retrieve(torch.from_numpy(p).to(DEV), db, 1000, 0.95)
    assert [list(zip(r.idx.tolist(), r.ent.tolist())) for r in got] == [[(n, c) for n, c, _ in r] for r in want]


# ------------------------------------------------------------------ end-to-end forward --------------
@pytest.mark.parametrize("name", names(include_lm=True))
def test_forward_matches_reference_golden(name):
    g = Golden(name)
    m = build_model(g)
    loss, pred, dist, tp = m(g.batch)
    ref = torch.from_numpy(g.out["pred_dist"]).to(DEV)
    assert tp is None and dist.shape == ref.shape
    err = rel_err(dist, ref, 1e-30)
    assert err < RTOL, err
    assert abs(float(loss) - float(g.out["loss"])) < 1e-3 * max(1.0, abs(float(g.out["loss"])))
    hist = torch.stack(m.dist_history[1:]).cpu()
    assert rel_err(hist, torch.from_numpy(g.out["dist_history"]), 1e-30) < RTOL
    hf = m.reasoning.h_view.reshape(ref.shape[0], ref.shape[1], -1).cpu()
    want_h = torch.from_numpy(g.out["h_final"])
    assert (hf - want_h).abs().max().item() <= 1e-4 * (want_h.abs().max().item() + 1e-12)
    # retrieved node ids: bit exact against the reference evaluator's lists
    got, _ = evaluate.retrieve(dist, m.last_batch, g.num_entity, g.args["eps"])
    ref_lists = O.rank_candidates(g.batch[0], g.batch[1], g.out["pred_dist"], g.num_entity, g.args["eps"])
    swaps = assert_ranking_equivalent(got, ref_lists, g.out["pred_dist"], name=name)
    if name in ("rearev_sharp_ties", "nsm_reason_kb", "rearev_sbert_reltext"):   # peaked distributions: strictly identical
        assert swaps == 0
        assert [r.ent.tolist() for r in got] == g.cand_lists()[0]
    ref_pred = torch.from_numpy(g.out["pred"]).to(DEV)
    p_at_ref = dist.gather(1, ref_pred.view(-1, 1)).view(-1)
    assert (p_at_ref >= dist.max(1)[0] * (1 - 1e-5)).all()


def test_twin_nodes_tie_exactly_on_gpu():
    g = Golden("rearev_sharp_ties")
    m = build_model(g)
    _, _, dist, _ = m(g.batch)
    assert torch.equal(dist[:, 4], dist[:, 5])      # structurally symmetric nodes -> identical floats


@pytest.mark.parametrize("model,kw", [("ReaRev", dict(num_iter=3, num_ins=2, num_gnn=3)),
                                      ("NSM", dict(num_step=3))])
def test_forward_vs_oracle_webqsp_shape(model, kw):
    """D=200 WebQSP-shape subgraphs (cfg1/cfg2 shape at B=4): CUDA path vs the CPU oracle, same weights."""
    args = S.model_args(model, entity_dim=200, use_cuda=True, **kw)
    torch.manual_seed(0)
    cls = G.NSM if model == "NSM" else G.ReaRev
    m = cls(dict(args), 5000, 300, 400).eval()
    with torch.no_grad():
        m.reasoning.score_func.weight.mul_(20.0)
    sd = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    b = S.make_batch(2, B=4, N=2000, E=6000, num_entity=5000, num_relation=300, num_word=400,
                     with_weights=False, test=True)
    _, _, want = O.forward(sd, args, 5000, 400, b)
    loss, pred, dist, _ = m(b[:7])
    assert rel_err(dist.cpu(), want, 1e-30) < RTOL
    assert torch.allclose(dist.sum(1).cpu(), torch.ones(4), atol=1e-5)
    got, _ = evaluate.retrieve(dist, m.last_batch, 5000, 0.95)
    ref = O.rank_candidates(b[0], b[1], want.numpy(), 5000, 0.95)
    assert_ranking_equivalent(got, ref, want.numpy(), name="oracle_forward")


def test_full_size_properties_cfg2():
    """BASELINE cfg2 (B=64, N=2000, D=200, 3 hops): size-independent properties -- rows are distributions,
    pads/seeds-as-pad get exactly 0, run-to-run bit-identical, questions independent of batch mates."""
    c = S.CONFIGS["cfg2"]
    args = S.model_args("ReaRev", entity_dim=c["D"], num_iter=c["T"], num_ins=c["I"], num_gnn=c["K"],
                        use_cuda=True)
    torch.manual_seed(0)
    m = G.ReaRev(dict(args), S.WEBQSP_NUM_ENTITY, S.WEBQSP_NUM_RELATION, S.WEBQSP_NUM_WORD).eval()
    b = S.make_batch(1, B=c["B"], N=c["N"], E=c["E"], n_real=1500, with_weights=False)
    _, _, d1, _ = m(b)
    _, _, d2, _ = m(b)
    assert torch.equal(d1, d2)
    assert torch.allclose(d1.sum(1), torch.ones(c["B"], device=DEV), atol=1e-4)
    assert (d1[:, 1500:] == 0).all()
    from gnn_rag_b200 import parallel
    half = parallel.shard_batch(b, 1, 2)                      # questions 32..63 alone
    _, _, dh, _ = m(half)
    # block-diagonal independence.  Not bit-exact across batch sizes only because torch's cuDNN/cuBLAS
    # question encoder picks different kernels at B=32 vs B=64; our kernels are row-independent.
    assert rel_err(dh, d1[32:], 1e-30) < 1e-5


# ------------------------------------------------------------------ shortest-path node sets ---------
def test_shortest_path_nodes_vs_oracle():
    b = S.make_batch(41, B=3, N=120, E=300, num_entity=1000, num_relation=20, num_word=50,
                     multi_seed=True, with_weights=False)
    db = stage(b, 21)
    rs = np.random.RandomState(2)
    retrieved = []
    for k in (3, 1, 6):
        ix = rs.choice(np.arange(5, 120), size=k, replace=False).astype(np.int64)
        retrieved.append(evaluate.Retrieved(ix, ix, np.zeros(k, dtype=np.float32)))
    nodes, pair = evaluate.path_node_sets(db, retrieved)
    heads, tails, bids = b[2][0], b[2][2], b[2][3]
    for q in range(3):
        sel = bids == q
        srcs = np.nonzero(b[1][q])[0].tolist()
        tgts = retrieved[q].idx.tolist()
        want, pd = O.shortest_path_nodes((heads[sel] - q * 120).tolist(), (tails[sel] - q * 120).tolist(),
                                         120, srcs, tgts)
        assert nodes[q] == want
        for i, s in enumerate(srcs):
            for j, t in enumerate(tgts):
                assert pair[q, i, j] == pd.get((s, t), -1)
