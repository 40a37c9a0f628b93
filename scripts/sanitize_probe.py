"""Small D=200 ReaRev forward + ranking (every kernel of the hot path incl. the persistent aggregation kernel, the
cluster LSTM, the frontier fix-up and the wgmma GEMM) -- run under compute-sanitizer:
    compute-sanitizer --tool memcheck  python scripts/sanitize_probe.py
    compute-sanitizer --tool racecheck python scripts/sanitize_probe.py"""
import sys

import torch

sys.path.insert(0, ".")
import gnn_rag_b200 as G  # noqa: E402
from gnn_rag_b200 import evaluate, synthetic as S  # noqa: E402

args = S.model_args("ReaRev", entity_dim=200, num_iter=2, num_ins=2, num_gnn=3, word_dim=32, use_cuda=True)
torch.manual_seed(0)
model = G.ReaRev(dict(args), 3000, 40, 100).eval()
batch = S.make_batch(3, B=3, N=200, E=700, num_entity=3000, num_relation=40, num_word=100, powerlaw=True)
for _ in range(2):
    loss, pred, dist, _ = model(batch[:7])
    got, _ = evaluate.retrieve(dist, model.last_batch, 3000, args["eps"])
torch.cuda.synchronize()
assert torch.isfinite(dist).all() and abs(float(dist.sum()) - 3.0) < 1e-3
print("sanitize_probe ok", float(loss), [len(r) for r in got])
