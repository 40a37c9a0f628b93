"""GraftNet without a GPU: the reference goldens (tests/golden/graft/*.npz, made by tests/golden/make_graft_golden.py from
the UNMODIFIED reference) against the torch-CPU oracle and the training restatement, checkpoint compatibility, the
CLI-shaped args and the synthetic graft tuple."""
import json
import os

import numpy as np
import pytest
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import autograd_path, synthetic as S

GOLDEN_CASE_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "graft")
NUM_ENTITY, NUM_REL, NUM_WORD = 1000, 40, 100
CASES = sorted(os.path.splitext(n)[0] for n in os.listdir(GOLDEN_CASE_DIR) if n.endswith(".npz"))
TRAIN_CASES = [c for c in CASES if "train/loss" in np.load(os.path.join(GOLDEN_CASE_DIR, c + ".npz")).files]


class GraftGolden:
    def __init__(self, name):
        z = np.load(os.path.join(GOLDEN_CASE_DIR, name + ".npz"), allow_pickle=False)
        self.name = name
        self.z = z
        self.args = json.loads(str(z["args_json"]))
        self.sd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd/")}
        b = {k[6:]: z[k] for k in z.files if k.startswith("batch/")}
        kb = (b["heads"], b["rels"], b["tails"], b["batch_ids"], b["fact_ids"], b["weight_list"].tolist(),
              b["weight_rel_list"].tolist())
        ones = np.ones(len(b["e2f_b"]))
        graft = ((b["e2f_b"], b["e2f_f"], b["e2f_e"], ones), (b["f2e_b"], b["f2e_e"], b["f2e_f"], ones.copy()))
        self.batch = (b["local_entity"], b["query_entities"], kb, graft, b["q_input"], b["kb_fact_rel"],
                      b["seed_dist"], None, b["answer_dist"])
        self.rel_texts, self.rel_texts_inv = b.get("rel_texts"), b.get("rel_texts_inv")
        self.out = {k[4:]: z[k] for k in z.files if k.startswith("out/")}
        self.train = {k[6:]: z[k] for k in z.files if k.startswith("train/")}
        self.grads = {k[5:]: z[k] for k in z.files if k.startswith("grad/")}

    def state_dict(self):
        sd = dict(self.sd)
        if self.args.get("lm", "lstm") != "lstm":
            # the LM encoder is not stored: rebuilt as the generator's harness built it
            import transformers
            torch.manual_seed(1234)
            enc = transformers.AutoModel.from_config(transformers.BertConfig(**self.args["lm_config"]))
            sd.update({"instruction.node_encoder." + k: v for k, v in enc.state_dict().items()})
        return sd

    def cand_lists(self):
        ids, o = [], 0
        for n in self.out["cand_len"].tolist():
            ids.append(self.out["cand_ids"][o:o + n].tolist())
            o += n
        return ids


def load_model(name, device="cpu"):
    g = GraftGolden(name)
    m = G.GraftNet(dict(g.args, use_cuda=(device != "cpu")), NUM_ENTITY, NUM_REL, NUM_WORD)
    m.load_state_dict(g.state_dict(), strict=True)
    m.eval()
    if g.rel_texts is not None:
        m.encode_rel_texts(g.rel_texts, g.rel_texts_inv)
    return m, g


@pytest.fixture
def host_check():
    old = autograd_path.HOST_CHECK
    autograd_path.HOST_CHECK = True
    yield
    autograd_path.HOST_CHECK = old


def test_goldens_cover_the_edge_cases():
    assert len(CASES) == 6
    g = GraftGolden("graft_hub_clamp")
    tails = g.batch[3][1][1] + g.batch[3][1][0] * g.batch[0].shape[1]
    assert np.bincount(tails).max() > 2048                              # a hub row
    assert (g.batch[0][1] == NUM_ENTITY).all()                          # an empty question
    assert (g.out["w_tilde"] == 0).any() and (g.out["e2f_softmax"] == np.float32(1e-10)).any()
    p = GraftGolden("graft_dropout_padmax")
    W = p.out["w_tilde"]
    assert (W[1][p.batch[5][1] == NUM_REL] == 1.0).all()               # question 1: the maximum W is the pad relation's


@pytest.mark.parametrize("name", CASES)
def test_reference_state_dict_loads_strict(name):
    m, g = load_model(name)
    assert set(m.state_dict()) == set(g.state_dict())


def test_cli_shaped_args_give_num_layer_instructions():
    args = S.model_args("GraftNet", entity_dim=16, num_layer=4)
    assert "num_ins" not in args and "num_step" not in args
    m = G.GraftNet(args, 50, 10, 20)
    assert m.instruction.num_ins == 4
    assert all(hasattr(m.instruction, "question_linear%d" % i) for i in range(4))
    assert m.num_iter == 4


def test_lstm_with_relation_texts_is_refused():
    m = G.GraftNet(S.model_args("GraftNet", entity_dim=16, num_layer=2), 50, 10, 20)
    m.rel_texts = torch.zeros(11, 3, dtype=torch.long)
    with pytest.raises(NotImplementedError):
        m.get_rel_feature_train()


@pytest.mark.parametrize("inverse", [False, True])
def test_synthetic_tuple_has_the_loader_layout(inverse):
    B, N, R = 4, 30, 11
    b = S.make_graft_batch(3, B, N, 60, num_entity=100, num_relation=R, num_word=20, fact_dropout=0.25,
                           use_inverse_relation=inverse, n_real="ragged", empty_questions=(2,), test=True)
    assert len(b) == 10 and b[7] is None
    le, qe, kb, graft, qi, kfr, sd, _, ad, al = b
    (hb, hf, he, hv), (tb, te, tf, tv) = graft
    T = np.array([((kb[3] == q) & (kb[1] != R - 1)).sum() for q in range(B)])
    assert kfr.shape == (B, 2 * T.max() + N) and kfr.dtype == np.int64
    for q in range(B):
        n = 2 * T[q] if inverse else T[q]
        assert (kfr[q, T[q]:] == R).all()                               # pad slots hold num_kb_relation
        sel = hb == q
        assert sel.sum() == int(np.floor(n * 0.75))                     # floor(n * (1 - fact_dropout)) kept
        assert (hf[sel] < n).all() and len(np.unique(hf[sel])) == sel.sum()
        assert np.array_equal(hf[sel], tf[tb == q])                     # same permutation in both lists
        assert not np.array_equal(hf[sel], np.sort(hf[sel])) or sel.sum() < 3
        if inverse:
            assert (kfr[q, :T[q]] >= (R - 1) // 2).all() or T[q] == 0   # slot i holds the inverse relation of tuple i
    assert (hv == 1.0).all() and (tv == 1.0).all()


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference(name):
    from oracle import graft_oracle
    m, g = load_model(name)
    out = graft_oracle.forward(m, g.batch)
    np.testing.assert_allclose(out["pred_dist"], g.out["pred_dist"], rtol=1e-6, atol=1e-30)
    np.testing.assert_allclose(out["pagerank_history"], g.out["pagerank_history"], rtol=1e-6, atol=1e-30)
    assert abs(out["loss"] - float(g.out["loss"])) <= 1e-6 * abs(float(g.out["loss"]))
    assert graft_oracle.candidate_lists(out["pred_dist"], g.batch, NUM_ENTITY, g.args["eps"]) == g.cand_lists()


@pytest.mark.parametrize("name", TRAIN_CASES)
def test_training_restatement_matches_reference_gradients(name, host_check):
    m, g = load_model(name)
    batch = list(g.batch)
    batch[8] = g.train["answer_dist"]
    loss, pred, pred_dist, tp_list = m(tuple(batch), training=True)
    assert abs(float(loss) - float(g.train["loss"])) <= 2e-5 * abs(float(g.train["loss"]))
    assert tp_list[0] == g.train["h1"].tolist()
    np.testing.assert_allclose(np.array(tp_list[1]), g.train["f1"], rtol=1e-6)
    loss.backward()
    checked = 0
    for k, p in m.named_parameters():
        if k not in g.grads:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, k
            continue
        want = g.grads[k]
        got = p.grad.numpy() if p.grad is not None else np.zeros_like(want)
        assert np.abs(got - want).max() <= 5e-3 * np.abs(want).max() + 1e-9, (k, np.abs(got - want).max())
        checked += 1
    assert checked >= 15
