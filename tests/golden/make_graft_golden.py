"""Generate tests/golden/graft/*.npz by running the UNMODIFIED reference GraftNet (cmavro/GNN-RAG,
gnn/models/GraftNet/graftnet.py) on seeded synthetic graft batches.  Needs the reference checkout that
oracle/ref_harness.py imports:

    python tests/golden/make_graft_golden.py [case ...]

Each file holds the args (json), the reference state_dict, the 9-tuple batch, and the reference's outputs: loss,
pred, pred_dist, the per-layer score and PageRank histories, the evaluator's candidate lists; for the training cases
also ``model(batch, training=True)`` (eval mode: dropout off) -> loss, h1, f1 and every parameter gradient.
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gnn_rag_b200 import synthetic as S  # noqa: E402
from oracle import ref_harness as H  # noqa: E402
from make_golden import NUM_ENTITY, NUM_REL, NUM_WORD, add_twins, bert_tokens, make_rel_texts  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "graft")

SBERT = dict(vocab_size=NUM_WORD + 2, hidden_size=384, num_hidden_layers=1, num_attention_heads=12,
             intermediate_size=32, max_position_embeddings=32, hidden_dropout_prob=0.0,
             attention_probs_dropout_prob=0.0)

CASES = {
    "graft_small": dict(D=16, kw=dict(num_layer=3, norm_rel=True),
                        batch=dict(seed=11, B=3, N=40, E=120, n_real="ragged", multi_seed=True), train=True, hit=True),
    "graft_d50_sharp": dict(D=50, kw=dict(num_layer=2), batch=dict(seed=12, B=3, N=60, E=240, seeds_are_pad=True),
                            sharpen=(3.0, 20.0), twins=True),
    "graft_dropout_padmax": dict(D=24, kw=dict(num_layer=2), batch=dict(seed=13, B=3, N=50, E=200, n_real="ragged"),
                                 fact_dropout=0.3, padmax=1, train=True),
    "graft_hub_clamp": dict(D=16, kw=dict(num_layer=2), batch=dict(seed=14, B=3, N=2400, E=2600, empty_questions=(1,)),
                            hub=2100, clamp=(2, 5), sharpen=(1.0, 0.05)),
    "graft_inverse": dict(D=20, kw=dict(num_layer=3, use_inverse_relation=True),
                          batch=dict(seed=15, B=3, N=40, E=100, n_real="ragged"), inverse=True, train=True),
    "graft_sbert_reltext": dict(D=24, kw=dict(num_layer=2, lm="sbert", relation_word_emb=True, lm_config=SBERT),
                                batch=dict(seed=16, B=3, N=40, E=120, n_real="ragged", multi_seed=True),
                                sharpen=(2.0, 20.0), train=True),
}


def import_graftnet():
    mods = H._import_reference()
    if "GraftNet" not in mods:
        from models.GraftNet.graftnet import GraftNet  # noqa: E402
        mods["GraftNet"] = GraftNet
    return mods


def sharpen(model, e2e, score):
    with torch.no_grad():
        for k, p in model.named_parameters():
            if "e2e_linear" in k and k.endswith("weight"):
                p.mul_(e2e)
            if k.endswith("reasoning.score_func.weight"):
                p.mul_(score)


def query_states(model, q_input):
    with torch.no_grad():
        model.instruction(torch.from_numpy(q_input))
        qh = model.instruction.query_hidden_emb
        mask = model.instruction.query_mask if hasattr(model.instruction, "query_mask") else None
    return qh, mask


def attention_w(qh, mask, rel):
    """compute_attention's W for relation rows ``rel`` [R, D] of every question -> [B, R]."""
    D = rel.shape[1]
    div = float(np.sqrt(D))
    sim = torch.einsum("bqd,rd->bqr", qh, rel) / div + (1 - mask.unsqueeze(2)) * -100000000000
    a = torch.softmax(sim, 1)
    att = torch.einsum("bqr,bqd->brd", a, qh)
    return (att * rel.unsqueeze(0)).sum(2) / div


def set_rel_row(model, r, target):
    """relation_embedding row r such that relation_linear1(row) = target."""
    lin = model.relation_linear1
    with torch.no_grad():
        row = torch.linalg.solve(lin.weight.double(), (target - lin.bias).double()).float()
        model.relation_embedding.weight[r] = row


def rel_features(model):
    with torch.no_grad():
        return model.relation_linear1(model.relation_embedding.weight)


def main():
    import_graftnet()
    os.makedirs(OUT, exist_ok=True)
    for name, c in CASES.items():
        if len(sys.argv) > 1 and name not in sys.argv[1:]:
            continue
        args = S.model_args("GraftNet", entity_dim=c["D"], word_dim=24, **c["kw"])
        lm = args.get("lm", "lstm") != "lstm"
        if lm:
            H.patch_transformers_offline(args["lm_config"])
        model = H.build_reference_model(args, NUM_ENTITY, NUM_REL, NUM_WORD, seed=0)
        if c.get("sharpen"):
            sharpen(model, *c["sharpen"])
        if lm:
            # the LM path never reads word_embedding (bert_encoder.py:83-105): zeros keep the file small; the encoder
            # itself is not stored, tests rebuild it as the harness does (torch.manual_seed(1234) + from_config)
            with torch.no_grad():
                model.word_embedding.weight.zero_()
        bkw = dict(c["batch"])
        N = bkw["N"]
        base = S.make_batch(num_entity=NUM_ENTITY, num_relation=NUM_REL, num_word=NUM_WORD, Q=8, test=True,
                            with_weights=True, **bkw)
        if c.get("twins"):
            base = add_twins(base, N)
        le, qe, kb, qi, sd_, _tb, ad, al = base
        heads, rels, tails, bids = (np.array(x) for x in kb[:4])
        if c.get("hub"):           # question 0: c["hub"] facts into its last node
            sel = np.nonzero((bids == 0) & (rels != NUM_REL - 1))[0][: c["hub"]]
            tails[sel] = N - 1
        if c.get("clamp"):         # question b: every out-fact of node 3 carries relation r (its W is pushed to -inf)
            b, r = c["clamp"]
            rels[(bids == b) & (heads == b * N + 3) & (rels != NUM_REL - 1)] = r
        if c.get("hub") or c.get("clamp"):
            wl, wrl = S._degree_weights(heads, rels)
            kb = (heads, rels, tails, bids, np.arange(len(heads)), wl, wrl)
            base = (le, qe, kb, qi, sd_, None, ad, al)
        if lm:
            base = base[:3] + (bert_tokens(base[3], NUM_WORD),) + base[4:]
        batch = S.graft_from_batch(base, bkw["seed"], NUM_REL, c.get("fact_dropout", 0.0), c.get("inverse", False))
        rel_texts = rel_texts_inv = None
        if lm:
            rel_texts, rel_texts_inv = make_rel_texts(31, NUM_REL + 1), make_rel_texts(32, NUM_REL + 1)
            model.encode_rel_texts(rel_texts, rel_texts_inv)
        if c.get("clamp") or c.get("padmax") is not None:
            qh, mask = query_states(model, batch[4])
            rf = rel_features(model)
            D = c["D"]
            if c.get("clamp"):
                b, r = c["clamp"]
                toks = qh[b][mask[b] > 0]
                u = toks.mean(0)
                u = u / u.norm()
                assert float((toks @ u).min()) > 0
                set_rel_row(model, r, -1000.0 * np.sqrt(D) * u)
                w = attention_w(qh, mask, rel_features(model))
                assert float(w[b].max() - w[b, r]) > 110, (w[b].max(), w[b, r])
            if c.get("padmax") is not None:
                b = c["padmax"]
                toks = qh[b][mask[b] > 0]
                u = toks.mean(0)
                u = u / u.norm()
                fr = batch[5][b]
                real = np.unique(fr[fr != NUM_REL])
                w0 = attention_w(qh, mask, rf)[b, torch.from_numpy(real)].max()
                lo_t, hi_t = 0.0, 400.0
                for _ in range(60):            # W(pad) = max real W + 95: the shift underflows most real facts
                    t = 0.5 * (lo_t + hi_t)
                    wp = attention_w(qh[b:b + 1], mask[b:b + 1], (t * u).unsqueeze(0))[0, 0]
                    lo_t, hi_t = (t, hi_t) if wp < w0 + 95 else (lo_t, t)
                set_rel_row(model, NUM_REL, t * u)
        hist = []
        orig = model.reasoning.forward

        def rec(*a, **k):
            out = orig(*a, **k)
            hist.append(out[2].detach().clone())
            return out
        model.reasoning.forward = rec
        with torch.no_grad():
            loss, pred, pred_dist, _ = model(batch[:9])
        model.reasoning.forward = orig
        wt = model.reasoning.W_tilde.detach()
        e2f = model.reasoning.e2f_softmax.detach()
        retrieved = H.reference_rank(batch, pred_dist.numpy(), NUM_ENTITY, args["eps"])
        blob = {"args_json": np.array(json.dumps(args))}
        for k, v in model.state_dict().items():
            if not (lm and k.startswith("instruction.node_encoder.")):
                blob["sd/" + k] = v.detach().numpy()
        le, qe, kb, graft, qi, kfr, sdist, _, ad = batch[:9]
        blob.update({"batch/local_entity": le, "batch/query_entities": qe, "batch/q_input": qi,
                     "batch/seed_dist": sdist, "batch/answer_dist": ad, "batch/kb_fact_rel": kfr,
                     "batch/heads": kb[0], "batch/rels": kb[1], "batch/tails": kb[2],
                     "batch/batch_ids": kb[3], "batch/fact_ids": kb[4],
                     "batch/weight_list": np.array(kb[5], dtype=np.float64),
                     "batch/weight_rel_list": np.array(kb[6], dtype=np.float64)})
        for i, key in enumerate(("e2f_b", "e2f_f", "e2f_e")):
            blob["batch/" + key] = graft[0][i]
        for i, key in enumerate(("f2e_b", "f2e_e", "f2e_f")):
            blob["batch/" + key] = graft[1][i]
        if lm:
            blob["batch/rel_texts"], blob["batch/rel_texts_inv"] = rel_texts, rel_texts_inv
        blob["out/loss"] = loss.numpy()
        blob["out/pred"] = pred.numpy()
        blob["out/pred_dist"] = pred_dist.numpy()
        blob["out/dist_history"] = np.stack([h.detach().numpy() for h in model.dist_history[1:]])
        blob["out/pagerank_history"] = np.stack([h.numpy() for h in hist])
        blob["out/w_tilde"] = wt.numpy()
        blob["out/e2f_softmax"] = e2f.numpy()
        ids = [[int(c_) for c_, _ in r] for r in retrieved]
        probs = [[float(p_) for _, p_ in r] for r in retrieved]
        blob["out/cand_len"] = np.array([len(r) for r in ids], dtype=np.int64)
        blob["out/cand_ids"] = np.array(sum(ids, []), dtype=np.int64)
        blob["out/cand_probs"] = np.array(sum(probs, []), dtype=np.float64)
        if c.get("train"):
            for k, p in model.named_parameters():
                if "node_encoder" not in k:
                    p.requires_grad_(True)
            tb = list(batch[:9])
            if c.get("hit"):        # the top-1 node (+ node 7) as answers: h1 = 1, f1 > 0
                a2 = np.zeros_like(tb[8])
                for b, t in enumerate(pred_dist.numpy().argmax(1)):
                    a2[b, t] = 1.0
                    a2[b, 7] = 1.0
                tb[8] = a2
            model.zero_grad()
            tl, _tp, tpd, tp_list = model(tuple(tb), training=True)
            tl.backward()
            blob["train/answer_dist"] = tb[8]
            blob["train/loss"] = tl.detach().numpy()
            blob["train/pred_dist"] = tpd.detach().numpy()
            blob["train/h1"] = np.array(tp_list[0], dtype=np.float32)
            blob["train/f1"] = np.array(tp_list[1], dtype=np.float32)
            for k, p in model.named_parameters():
                if p.grad is not None:
                    blob["grad/" + k] = p.grad.numpy()
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **blob)
        nties = sum(len(p) - len(set(p)) for p in probs)
        clamped = int((e2f.numpy() <= 1e-10).sum())
        underflow = int(((wt.numpy() == 0)).sum())
        print("%-22s F=%6d loss=%.5f peak=%.4f cand=%s ties=%d clampedE=%d W~=0:%d  %.0f KB" % (
            name, len(graft[0][0]), float(loss), float(pred_dist.max()), [len(r) for r in ids], nties, clamped,
            underflow, os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main()
