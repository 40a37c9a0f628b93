"""Hot-shape goldens from the UNMODIFIED reference (cmavro/GNN-RAG @ /root/reference): entity_dim 200 with N >= 64 --
the only shapes that reach the |v|-accumulating aggregation kernel, the K = 1040 tensor-core GEMM and the frontier path --
plus the FULL-SIZE cfg2 batch (B = 64, the configuration bench.py times) and the cfg5 stress graph.  Weights are
``synthetic.seeded_state_dict`` (rebuilt by the tests), so the files hold reference OUTPUTS only.  Build container only:

    python tests/golden/make_golden_hot.py [case ...]
"""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from gnn_rag_b200 import synthetic as S  # noqa: E402
from oracle import ref_harness as H  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hot")

SMALL = dict(num_entity=1000, num_relation=40, num_word=100)
WEBQSP = dict(num_entity=S.WEBQSP_NUM_ENTITY, num_relation=S.WEBQSP_NUM_RELATION, num_word=S.WEBQSP_NUM_WORD)

CASES = {
    # random init: near-uniform distributions
    "d200_rand": dict(vocab=SMALL, D=200, kw=dict(num_iter=2, num_ins=2, num_gnn=3), wseed=11,
                      batch=dict(seed=21, B=3, N=96, E=400, n_real="ragged", multi_seed=True), layer_I=2),
    # peaked, hubs (rows longer than the staged slice share), exact structural twins are not needed here
    "d200_sharp": dict(vocab=SMALL, D=200, kw=dict(num_iter=3, num_ins=2, num_gnn=3), wseed=12,
                       sharpen=(4.0, 3.0, 12.0), batch=dict(seed=22, B=3, N=128, E=900, powerlaw=True), layer_I=2),
    "d200_norm": dict(vocab=SMALL, D=200, kw=dict(num_iter=2, num_ins=3, num_gnn=2, normalized_gnn=True), wseed=13,
                      sharpen=(3.0, 3.0, 300.0), batch=dict(seed=23, B=2, N=80, E=300, n_real=70), layer_I=3),
    # BASELINE configs[1] at full size: exactly bench.py's batch (seed 1) and architecture
    "cfg2_full": dict(vocab=WEBQSP, D=200, kw=dict(num_iter=3, num_ins=2, num_gnn=3), wseed=0,
                      sharpen=(4.0, 3.0, 200.0), batch=dict(seed=1, B=64, N=2000, E=6000, with_weights=False), keep_h=16),
    # BASELINE configs[4]: stress graph, D = 400
    "cfg5_full": dict(vocab=WEBQSP, D=400, kw=dict(num_iter=3, num_ins=2, num_gnn=3), wseed=5,
                      sharpen=(4.0, 3.0, 200.0), batch=dict(seed=1, B=1, N=100_000, E=1_000_000, with_weights=False),
                      keep_h=16),
}


def main():
    os.makedirs(OUT, exist_ok=True)
    H._import_reference()
    for name, c in CASES.items():
        if len(sys.argv) > 1 and name not in sys.argv[1:]:
            continue
        t0 = time.time()
        v = c["vocab"]
        args = S.model_args("ReaRev", entity_dim=c["D"], **c["kw"])
        model = H.build_reference_model(args, v["num_entity"], v["num_relation"], v["num_word"], seed=0)
        shapes = {k: tuple(t.shape) for k, t in model.state_dict().items()}
        sd = S.seeded_state_dict(shapes, seed=c["wseed"], sharpen=c.get("sharpen"))
        model.load_state_dict({k: torch.from_numpy(a) for k, a in sd.items()}, strict=True)
        bkw = dict(c["batch"])
        batch = S.make_batch(num_entity=v["num_entity"], num_relation=v["num_relation"], num_word=v["num_word"],
                             test=True, **bkw)
        if batch[2][5] is None:           # the reference's build_matrix wants the weight lists even when unused
            kb = batch[2]
            ones = np.ones(len(kb[0]), dtype=np.float64)
            batch_ref = batch[:2] + ((kb[0], kb[1], kb[2], kb[3], kb[4], ones, ones),) + batch[3:]
        else:
            batch_ref = batch
        loss, pred, pred_dist = H.reference_forward(model, batch_ref)
        retrieved = H.reference_rank(batch_ref, pred_dist.numpy(), v["num_entity"], args["eps"])
        blob = {"meta_json": np.array(json.dumps(dict(args=args, vocab=v, wseed=c["wseed"], sharpen=c.get("sharpen"),
                                                     batch=bkw, shapes={k: list(s) for k, s in shapes.items()}))),
                "out/loss": loss.numpy(), "out/pred": pred.numpy(), "out/pred_dist": pred_dist.numpy(),
                "out/dist_history": np.stack([h.detach().numpy() for h in model.dist_history[1:]])}
        hf = model.reasoning.local_entity_emb.detach().numpy()
        keep = c.get("keep_h")
        blob["out/h_final"] = hf if keep is None else hf[:, :keep]
        ids = [[int(c_) for c_, _ in r] for r in retrieved]
        probs = [[float(p_) for _, p_ in r] for r in retrieved]
        blob["out/cand_len"] = np.array([len(r) for r in ids], dtype=np.int64)
        blob["out/cand_ids"] = np.array(sum(ids, []), dtype=np.int64)
        blob["out/cand_probs"] = np.array(sum(probs, []), dtype=np.float32)      # fp32 values: lossless
        if "layer_I" in c:     # isolated reason_layer / reason_layer_inv calls, all instructions, dense prior
            layer = model.reasoning
            rs = np.random.RandomState(99)
            B, N = batch[0].shape
            dist = torch.softmax(torch.from_numpy(rs.randn(B, N).astype(np.float32)), 1)
            ins = torch.from_numpy(rs.randn(B, c["layer_I"], c["D"]).astype(np.float32))
            nb, nbi = [], []
            with torch.no_grad():
                for j in range(c["layer_I"]):
                    nb.append(layer.reason_layer(dist, ins[:, j], layer.rel_linear1, None).numpy())
                    nbi.append(layer.reason_layer_inv(dist, ins[:, j], layer.rel_linear1, None).numpy())
            blob.update({"layer/dist": dist.numpy(), "layer/ins": ins.numpy(),
                         "layer/rel_features": layer.rel_features.detach().numpy(),
                         "layer/rel_features_inv": layer.rel_features_inv.detach().numpy(),
                         "layer/neighbor_rep": np.stack(nb), "layer/neighbor_rep_inv": np.stack(nbi)})
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **blob)
        print("%-12s F=%8d loss=%.5f peak_p=%.4f cand=%s  %.0f KB  %.0f s" % (
            name, len(batch[2][0]), float(loss), float(pred_dist.max()), [len(r) for r in ids][:8],
            os.path.getsize(path) / 1024, time.time() - t0), flush=True)


if __name__ == "__main__":
    main()
