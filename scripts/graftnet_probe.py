"""GraftNet inference throughput on one GPU, per-kernel times, the aggregation's achieved bytes/s, the torch-CPU oracle
on a bounded sample, the GPU outputs against that oracle, and the CUDA-graph serving leg.

    python scripts/graftnet_probe.py [--B 64] [--N 2000] [--E 6000] [--dims 50,200] [--steps 20] [--warmup 5]
                                     [--cpu-questions 2] [--graphed-only] [--out results/graftnet_probe.json]

Device time comes from CUDA events around each forward; a 256 MB buffer is rewritten between steps so every step
starts with a cold L2.  The card name and power limit are read in the same run (nvidia-smi query only).

Graphed leg (``graphed`` per D): device ms per step of eager ``model(batch)`` + ``rank_candidates`` against
``GraphedStep`` (static-buffer fill + replay), both from the same pinned batch, alternating, L2 flushed before each;
end-to-end questions/s of ``submit`` / ``collect`` (two tickets in flight) over pageable-numpy batches whose fact
counts differ (one ``max_fact``, as a loader's); and whether ``pred_dist`` and the candidate lists of the two paths are
bit-identical."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import gnn_rag_b200 as G  # noqa: E402
from gnn_rag_b200 import ops, synthetic as S  # noqa: E402
from oracle import graft_oracle  # noqa: E402

NUM_ENTITY, NUM_REL, NUM_WORD = 100_000, 6106, 5000


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() + " W"
    except Exception as e:  # noqa: BLE001
        power = "unknown (%s)" % e
    return name, power


def agg_bytes(db, D):
    """Algorithmic bytes of one gr_graft_aggregate call: per fact the CSR entry (src, rel, fact: 12 B), slot_of,
    W~, prior[head], E[head] (16 B) and the two gathered fp32 rows (2 * 4D); per row the row pointer, prior, d' (12 B)
    and the split-bf16 writes of sum_v, indeg and q2e (2 planes * 2 B * (2D + 1))."""
    F = int(db.graft.nfacts.item())
    Nt = db.B * db.N
    return F * (12 + 16 + 8 * D) + Nt * (12 + 4 * (2 * D + 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=64)
    ap.add_argument("--N", type=int, default=2000)
    ap.add_argument("--E", type=int, default=6000)
    ap.add_argument("--dims", default="50,200")
    ap.add_argument("--layers", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--cpu-questions", type=int, default=2)
    ap.add_argument("--graphed-only", action="store_true", help="skip the per-kernel and CPU-oracle legs")
    ap.add_argument("--e2e-steps", type=int, default=40)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    name, power = card()
    res = dict(card=name, power_limit=power, B=a.B, N=a.N, E=a.E, layers=a.layers, torch_threads=torch.get_num_threads(),
               dims={})
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device="cuda")
    batch = S.make_graft_batch(0, a.B, a.N, a.E, num_entity=NUM_ENTITY, num_relation=NUM_REL, num_word=NUM_WORD,
                               with_weights=False, test=False)
    for D in [int(x) for x in a.dims.split(",")]:
        args = S.model_args("GraftNet", entity_dim=D, num_layer=a.layers, word_dim=300, use_cuda=True)
        torch.manual_seed(0)
        m = G.GraftNet(dict(args), NUM_ENTITY, NUM_REL, NUM_WORD).cuda().eval()
        if a.graphed_only:
            res["dims"][D] = dict(graphed=graphed_leg(m, args, batch, flush, a))
            print(json.dumps({D: res["dims"][D]}))
            continue
        for _ in range(a.warmup):
            m(batch)
        times = []
        for _ in range(a.steps):
            flush.add_(1.0)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            _l, _p, pd, _ = m(batch)
            e.record()
            torch.cuda.synchronize()
            times.append(s.elapsed_time(e))
        ms = float(np.median(times))
        ops.STATS.reset()
        ops.STATS.time_ops = True
        flush.add_(1.0)
        _l, _p, pd, _ = m(batch)
        torch.cuda.synchronize()
        ops.STATS.time_ops = False
        per = {}
        for s_, e_, cls, _info in ops.STATS.op_events:
            per[cls] = per.get(cls, 0.0) + s_.elapsed_time(e_)
        agg_ms = per.get("aggregation", 0.0) / a.layers
        nbytes = agg_bytes(m.last_batch, D)
        # CPU oracle on the first questions of the same batch (bounded sample)
        k = a.cpu_questions
        sub = _slice(batch, k)
        mc = G.GraftNet(dict(args, use_cuda=False), NUM_ENTITY, NUM_REL, NUM_WORD)
        mc.load_state_dict({kk: v.cpu() for kk, v in m.state_dict().items()})
        mc.eval()
        t0 = time.perf_counter()
        ref = graft_oracle.forward(mc, sub)
        cpu_s = time.perf_counter() - t0
        got = m(sub)[2].cpu().numpy()
        err = float(np.abs(got - ref["pred_dist"]).max() / np.abs(ref["pred_dist"]).max())
        res["dims"][D] = dict(device_ms_per_batch=ms, questions_per_s=a.B / ms * 1e3, per_kernel_ms=per,
                              aggregation_ms_per_layer=agg_ms, aggregation_bytes=nbytes,
                              aggregation_GBps=nbytes / (agg_ms * 1e-3) / 1e9 if agg_ms > 0 else None,
                              cpu_oracle_questions=k, cpu_oracle_s=cpu_s, cpu_oracle_questions_per_s=k / cpu_s,
                              pred_dist_rel_err_vs_oracle=err)
        res["dims"][D]["graphed"] = graphed_leg(m, args, batch, flush, a)
        print(json.dumps({D: res["dims"][D]}))
    print(json.dumps(dict((k, v) for k, v in res.items() if k != "dims")))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


def _pad_max_fact(batch, width):
    """kb_fact_rel padded to ``width`` slots with the pad relation (a loader's max_facts is one dataset constant)."""
    kfr = batch[5]
    wide = np.full((kfr.shape[0], width), NUM_REL, dtype=np.int64)
    wide[:, :kfr.shape[1]] = kfr
    return batch[:5] + (wide,) + batch[6:]


def graphed_leg(m, args, batch, flush, a):
    from gnn_rag_b200 import batching, evaluate
    eps = args["eps"]
    gs = G.GraphedStep(m, NUM_ENTITY)
    pinned = batching.pin_graft_batch(batch)

    def eager():
        _l, _p, pd, _ = m(pinned)
        ops.rank_candidates(pd, m.last_batch.local_entity, m.last_batch.query_entities, NUM_ENTITY, eps)

    def graph():
        gs(pinned)

    for _ in range(a.warmup):
        eager()
        graph()
    t = {"eager": [], "graphed": []}
    for _ in range(a.steps):
        for name, fn in (("eager", eager), ("graphed", graph)):
            flush.add_(1.0)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            torch.cuda.synchronize()
            t[name].append(s.elapsed_time(e))
    out = dict((k + "_ms_per_step", float(np.median(v))) for k, v in t.items())
    out.update((k + "_ms_min", float(np.min(v))) for k, v in t.items())
    out["graphed_speedup"] = out["eager_ms_per_step"] / out["graphed_ms_per_step"]
    # bit-for-bit: pred_dist and the candidate lists of the two paths on the same batch
    _l, _p, pd_e, _ = m(batch)
    ret_e, _ = evaluate.retrieve(pd_e, m.last_batch, NUM_ENTITY, eps)
    pd_e = pd_e.clone()
    o = gs(batch)
    ret_g, _ = gs.retrieve(o)
    out["pred_dist_bit_identical"] = bool(torch.equal(o.pred_dist, pd_e))
    out["candidate_lists_identical"] = [r.ent.tolist() for r in ret_g] == [r.ent.tolist() for r in ret_e] and \
        [r.prob.tolist() for r in ret_g] == [r.prob.tolist() for r in ret_e]
    # end to end: pageable numpy batches with different fact counts, two tickets in flight
    pool = [S.make_graft_batch(100 + i, a.B, a.N, a.E + d, num_entity=NUM_ENTITY, num_relation=NUM_REL,
                               num_word=NUM_WORD, with_weights=False) for i, d in enumerate((0, -150, 120, -60))]
    width = max(b[5].shape[1] for b in pool)
    pool = [_pad_max_fact(b, width) for b in pool]
    for b in pool:                     # capture / warm every bucket outside the timed window
        gs.collect(gs.submit(b))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    prev = None
    for i in range(a.e2e_steps):
        tk = gs.submit(pool[i % len(pool)])
        if prev is not None:
            gs.collect(prev)
        prev = tk
    gs.collect(prev)
    wall = time.perf_counter() - t0
    out.update(e2e_questions_per_s=a.B * a.e2e_steps / wall, e2e_steps=a.e2e_steps, e2e_graphs=len(gs._cache),
               e2e_facts=[int(len(b[2][0])) for b in pool], e2e_graft_facts=[int(len(b[3][0][0])) for b in pool])
    return out


def _slice(batch, k):
    le, qe, kb, graft, qi, kfr, sd, tb, ad = batch[:9]
    heads, rels, tails, bids, fids, wl, wrl = kb
    sel = bids < k
    kb2 = (heads[sel], rels[sel], tails[sel], bids[sel], np.arange(sel.sum()), None, None)
    (hb, hf, he, hv), (tb_, te, tf, tv) = graft
    s0, s1 = hb < k, tb_ < k
    g2 = ((hb[s0], hf[s0], he[s0], hv[s0]), (tb_[s1], te[s1], tf[s1], tv[s1]))
    return (le[:k], qe[:k], kb2, g2, qi[:k], kfr[:k], sd[:k], None, ad[:k])


if __name__ == "__main__":
    main()
