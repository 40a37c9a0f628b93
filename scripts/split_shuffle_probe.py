"""Training rate with fact dropout, the batch sampled and assembled on the host vs on the device
(loader.DeviceSplit(shuffle=True)), and the device time of gr_split_fact_order.

A train_epoch-shaped loop (gnn/train_model.py:219) over a synthetic WebQSP-shape split (scripts/device_split_probe.py:
N = 2000 nodes, E = 6000 stored facts per question, self-loops on): per batch ``get_batch(it, B, 0.1)``, the step,
``loss.item()`` as train_epoch logs it, clip_grad_norm_ and Adam.step().

  host    the loader's get_batch with loader.install(shuffle=True, weights="arrays", index_dtype=np.int32)
          (GraftNet: plus loader.install_graft), so np.random.permutation per question as in the reference
  device  DeviceSplit(loader, weights="arrays", shuffle=True).get_batch
  device_fused  the device batches through a graphed step that also runs clip_grad_norm_ and Adam.step() in its graph
          (``optimizer=``, ``max_norm=``; optim.ClipAdam); graphed shapes only
  device_epoch  the whole epoch as one GraphedTrainStep.train_epoch call (GraftNet: GraphedGraftTrainStep's): the
          batch assembly in the step graphs too, one graph replay per step and one read at the end of the epoch;
          graphed shapes only.  Its number of graphs and the peak device memory after its untimed epoch are reported
          next to device_fused's.

Shapes: ReaRev and NSM at the reference's training shape (B 8, entity_dim 50) through graphed.GraphedTrainStep;
GraftNet (B 8, entity_dim 50) eager (graftnet_d50) and through graphed.GraphedGraftTrainStep (graftnet_d50_graphed);
cfg2 (ReaRev, B 64, entity_dim 200) through GraphedTrainStep; and rearev_d50_varied, ReaRev at B 8 over a split whose
questions hold 500..12 000 stored facts, so that an epoch's batches fall into many fact-capacity buckets (graphs).
``buckets`` counts the distinct fact capacities of an epoch in stored order (GraftNet: also ``graft_buckets``, the
distinct (fact, graft) capacity pairs, one epoch graph each).  A pass runs the whole split; the questions/s of a mode
is the median over ``--runs`` passes, host and device alternating, after one warm-up pass of each (graph captures).
Then gr_split_fact_order alone, between CUDA events over ``--launches`` launches: B = 64 questions of 6 000 facts, and one question of 50 000 facts.  The GPU's
name and power limit are read in the same run.  One JSON line per measurement.

    python scripts/split_shuffle_probe.py [--questions 640] [--runs 3] [--modes host,device,device_fused,device_epoch]
        [--out split_shuffle_probe.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import gnn_rag_b200 as G                                        # noqa: E402
from gnn_rag_b200 import graphed, loader, ops, synthetic as S  # noqa: E402
from device_split_probe import NE, NR, NW, SyntheticSplit, gpu_info  # noqa: E402

SHAPES = {   # name -> model, batch size, model arguments, graphed
    "rearev_d50": ("ReaRev", 8, dict(entity_dim=50, num_ins=3, num_iter=2, num_gnn=3), True),
    "nsm_d50": ("NSM", 8, dict(entity_dim=50), True),
    "graftnet_d50": ("GraftNet", 8, dict(entity_dim=50), False),
    "graftnet_d50_graphed": ("GraftNet", 8, dict(entity_dim=50), True),
    "cfg2": ("ReaRev", 64, dict(entity_dim=200, num_ins=2, num_iter=3, num_gnn=3), True),
    "rearev_d50_varied": ("ReaRev", 8, dict(entity_dim=50, num_ins=3, num_iter=2, num_gnn=3), True),
}
MODES = ("host", "device", "device_fused", "device_epoch")
MAX_GRAPHS = 64      # the graphed modes keep every bucket's graph: the varied split's epoch uses more than the default 8
FACT_DROP = 0.1


def train_pass(data, step_fn, B):
    """One epoch over the split, train_epoch-shaped; -> seconds."""
    nb = (data.num_data + B - 1) // B
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for it in range(nb):
        step_fn(data.get_batch(it, B, FACT_DROP))
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def epoch_pass(data, gts, B):
    """One epoch as GraphedTrainStep.train_epoch (GraftNet: GraphedGraftTrainStep's); -> seconds."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    gts.train_epoch(data, B, FACT_DROP)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def varied_split(num_q):
    """SyntheticSplit with each question cut to 500..12 000 stored facts (seeded)."""
    L = SyntheticSplit(num_q, E=12000)
    rs = np.random.RandomState(1)
    L.kb_adj_mats = [tuple(a[:n] for a in m) for m, n in zip(L.kb_adj_mats, rs.randint(500, 12001, num_q))]
    return L


def make_step(name, m, use_graph, fused=False):
    params = [p for p in m.parameters() if p.requires_grad]
    opt = torch.optim.Adam(params, lr=1e-4)
    cls = graphed.GraphedGraftTrainStep if name == "GraftNet" else graphed.GraphedTrainStep
    if fused:
        fstep = cls(m, optimizer=opt, max_norm=1.0, max_graphs=MAX_GRAPHS)

        def step_fused(batch):
            loss, _pred, _pd, h1, f1 = fstep.step(batch)
            fstep.tp_list(h1, f1)
            loss.item()
        step_fused.gts = fstep
        return step_fused
    gstep = cls(m) if use_graph else None

    def step(batch):
        opt.zero_grad(set_to_none=True)
        if gstep is not None:
            loss, _pred, _pd, h1, f1 = gstep.step(batch)
            gstep.tp_list(h1, f1)
        else:
            loss, _pred, _pd, _tp = m(batch, training=True)
            loss.backward()
        loss.item()
        torch.nn.utils.clip_grad_norm_(params, 1.0)
        opt.step()
    return step


def order_kernel_ms(dev, B, E, launches):
    """Device milliseconds per gr_split_fact_order launch over B questions of E stored facts at FACT_DROP."""
    counts = np.full(B, E, dtype=np.int64)
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(counts)])).to(dev)
    ids = torch.arange(B, dtype=torch.int64, device=dev)
    kept_h = loader.kept_counts(counts, FACT_DROP)
    kept = torch.from_numpy(kept_h).to(dev)
    seed = torch.randint(0, 2 ** 62, (1,), device=dev)
    K, n_total = int(kept_h.sum()), int(counts.sum())
    for _ in range(3):
        ops.split_fact_order(off, ids, kept, seed, 0, n_total, K)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(launches):
        ops.split_fact_order(off, ids, kept, seed, 0, n_total, K)
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--questions", type=int, default=640)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--modes", default=",".join(MODES))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("split_shuffle_probe needs a CUDA device")
    info = gpu_info()
    dev = torch.device("cuda")
    want = a.modes.split(",")
    results = []
    splits = {}
    for shape in a.shapes.split(","):
        name, B, over, use_graph = SHAPES[shape]
        graft = name == "GraftNet"
        varied = shape.endswith("_varied")
        if (graft, varied) not in splits:
            L = varied_split(a.questions) if varied else SyntheticSplit(a.questions, graft=graft)
            loader.install(L, weights="arrays", index_dtype=np.int32, shuffle=True)
            if graft:
                loader.install_graft(L)
            splits[(graft, varied)] = (L, loader.DeviceSplit(L, dev, weights="arrays", index_dtype=torch.int32,
                                                             shuffle=True))
        L, split = splits[(graft, varied)]
        args = S.model_args(name, use_cuda=True, **over)
        torch.manual_seed(0)
        m = {"ReaRev": G.ReaRev, "NSM": G.NSM, "GraftNet": G.GraftNet}[name](dict(args), NE, NR, NW).cuda().train()
        step = make_step(name, m, use_graph)
        modes = {"host": (L, step, train_pass), "device": (split, step, train_pass)}
        if use_graph:
            modes["device_fused"] = (split, make_step(name, m, use_graph, fused=True), train_pass)
            cls = graphed.GraphedGraftTrainStep if graft else graphed.GraphedTrainStep
            ep = cls(m, optimizer=torch.optim.Adam([p for p in m.parameters() if p.requires_grad], lr=1e-4),
                     max_norm=1.0, max_graphs=MAX_GRAPHS)
            modes["device_epoch"] = (split, ep, epoch_pass)
        modes = {k: v for k, v in modes.items() if k in want}
        graphs, peak = {}, {}
        for k, (data, fn, run) in modes.items():      # warm-up: captures, caches
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            run(data, fn, B)
            peak[k] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 3)
            gts = fn if k == "device_epoch" else getattr(fn, "gts", None)
            if gts is not None:
                graphs[k] = len(gts._cache)
        secs = {k: [] for k in modes}
        for _ in range(a.runs):
            for k, (data, fn, run) in modes.items():
                secs[k].append(run(data, fn, B))
        qps = {k: a.questions / float(np.median(v)) for k, v in secs.items()}
        plan = graphed.epoch_plan(np.arange(a.questions), split._stored, split._ents, B, FACT_DROP,
                                  split._graft_count if graft else None)
        res = dict(shape=shape, model=name, B=B, D=over["entity_dim"], graphed=use_graph, fact_drop=FACT_DROP,
                   N=L.max_local_entity, E="500..12000" if varied else 6000, questions=a.questions,
                   buckets=len(set(plan.capacity.tolist())), gpu=info)
        if graft:
            res["graft_buckets"] = len(set(zip(plan.capacity.tolist(), plan.graft_capacity.tolist())))
        for k in modes:
            res[k + "_qps"] = round(qps[k], 1)
            res[k + "_s"] = [round(x, 4) for x in secs[k]]
            res[k + "_peak_gib"] = peak[k]
        for k, v in graphs.items():
            res[k + "_graphs"] = v
        if "host" in qps and "device" in qps:
            res["speedup"] = round(qps["device"] / qps["host"], 2)
        if "device" in qps and "device_fused" in qps:
            res["fused_speedup"] = round(qps["device_fused"] / qps["device"], 2)
        if "device_fused" in qps and "device_epoch" in qps:
            res["epoch_speedup"] = round(qps["device_epoch"] / qps["device_fused"], 3)
        results.append(res)
        print(json.dumps(res), flush=True)
        del step, modes, m
        torch.cuda.empty_cache()
    for B, E in ((64, 6000), (1, 50000)):
        res = dict(kernel="gr_split_fact_order", B=B, E=E, fact_drop=FACT_DROP,
                   ms=round(order_kernel_ms(dev, B, E, a.launches), 4), launches=a.launches, gpu=info)
        results.append(res)
        print(json.dumps(res), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
