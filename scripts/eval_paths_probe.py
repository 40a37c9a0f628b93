"""Evaluation-epoch rate with and without the shortest-path node sets (GraphedStep.start_eval(..., path_targets=T)), and
the device time of the BFS behind them.

A synthetic WebQSP-shape split (scripts/device_split_probe.py: N = 2000 nodes, E = 6000 stored facts per question,
self-loops on) held as a ``loader.DeviceSplit``, evaluated whole:

  plain   ``start_eval(split, B)`` and ``EvalRun.result()``
  paths   ``start_eval(split, B, path_targets=T)``, ``result()`` and ``EvalRun.paths()``

questions/s is the median over ``--runs`` passes, the two modes alternating, after one untimed pass of each (which
captures the graphs).  Shapes: ReaRev, NSM and GraftNet at the reference's WebQSP evaluation (B 20, entity_dim 50) and
cfg2 (ReaRev, B 64, entity_dim 200).  Every shape's node sets are compared with the per-batch
``evaluate.path_node_sets`` on the first ``--profile-steps`` batches.

``bfs``: on those batches, the per-batch call ``ops.shortest_path_nodes`` under ``torch.profiler``: the device time per
batch of each kernel (``bfs_kernel`` and ``mark_kernel``).  With ``--parent-lib`` (a libgnnrag_b200.so built from a
commit that still had the one-CTA-per-question ``paths_kernel``, for instance from a ``git worktree`` of it with
``python -m gnn_rag_b200._build``), the same inputs also go through that library's ``gr_shortest_path_nodes`` (the C
ABI is unchanged): its kernels' time per batch, and whether its outputs are bit-equal.  The GPU's name and power limit
are read in the same run.  One JSON line per shape.

    python scripts/eval_paths_probe.py [--questions 1280] [--runs 3] [--targets 32] [--parent-lib PATH]
"""
import argparse
import collections
import ctypes
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import gnn_rag_b200 as G                                        # noqa: E402
from gnn_rag_b200 import _lib, evaluate, graphed, loader, ops, synthetic as S  # noqa: E402
from device_split_probe import NE, NR, NW, SyntheticSplit, gpu_info  # noqa: E402

SHAPES = {   # name -> model, batch size, model arguments
    "rearev_d50": ("ReaRev", 20, dict(entity_dim=50, num_ins=3, num_iter=2, num_gnn=3)),
    "nsm_d50": ("NSM", 20, dict(entity_dim=50)),
    "graftnet_d50": ("GraftNet", 20, dict(entity_dim=50)),
    "cfg2": ("ReaRev", 64, dict(entity_dim=200, num_ins=2, num_iter=3, num_gnn=3)),
}


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def path_inputs(db, retrieved, T):
    """The sources and targets ``evaluate.path_node_sets`` hands to the kernel, as device tensors."""
    qe = db.query_entities
    S_ = max(int((qe != 0).sum(dim=1).max().item()), 1)
    src = torch.argsort((qe != 0).to(torch.int8), dim=1, descending=True, stable=True)[:, :S_].to(torch.int32)
    scnt = (qe != 0).sum(dim=1).to(torch.int32)
    Tb = max(1, min(T, max(len(r) for r in retrieved)))
    tgt = np.zeros((db.B, Tb), np.int32)
    tcnt = np.zeros(db.B, np.int32)
    for b, r in enumerate(retrieved):
        k = min(len(r), Tb)
        tcnt[b], tgt[b, :k] = k, r.idx[:k]
    dev = qe.device
    return src.contiguous(), scnt.contiguous(), torch.from_numpy(tgt).to(dev), torch.from_numpy(tcnt).to(dev)


def parent_call(lib, g, src, scnt, tgt, tcnt):
    """gr_shortest_path_nodes of the library ``lib`` -> (on_path, pair_dist)."""
    B, N, S_, T = g.B, g.N, src.shape[1], tgt.shape[1]
    dev = src.device
    on = torch.empty(B, N, dtype=torch.uint8, device=dev)
    pair = torch.empty(B, S_, T, dtype=torch.int32, device=dev)
    nbytes = lib.gr_paths_workspace_bytes(B, N, S_, T)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    p = lambda t: ctypes.c_void_p(t.data_ptr())              # noqa: E731
    rc = lib.gr_shortest_path_nodes(p(g.rowptr_t), p(g.src_t), p(g.rowptr_h), p(g.src_h), p(src), p(scnt), S_,
                                    p(tgt), p(tcnt), T, p(on), p(pair), B, N, p(ws), nbytes,
                                    ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, rc
    return on, pair


def kernel_us(prof, steps, keys):
    """Device us per batch of the CUDA kernels whose name holds one of ``keys``."""
    tab = collections.defaultdict(float)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            for k in keys:
                if k in e.name:
                    tab[k] += e.time_range.elapsed_us() / steps
    return {k: round(v, 1) for k, v in tab.items()}


def bfs_section(m, split, B, T, steps, parent):
    """The per-batch node sets of the first ``steps`` batches against the run's, and the BFS kernels' device time."""
    split.reset_batches(is_sequential=True)
    batches = []
    for it in range(steps):
        batch = split.get_batch(it, B, 0.0, test=True)
        with torch.no_grad():
            _l, _p, dist, _tp = m(batch[:-1])
        db = m.last_batch
        ret, _ = evaluate.retrieve(dist, db, NE, m.eps)
        nodes, pair = evaluate.path_node_sets(db, ret, T)
        batches.append((db, path_inputs(db, ret, T), nodes, pair))
    acts = [torch.profiler.ProfilerActivity.CUDA]
    out = {}
    libs = [("new", None)] + ([("parent", parent)] if parent is not None else [])
    for tag, lib in libs:
        outs = []
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=acts) as prof:
            for db, args, _n, _pd in batches:
                outs.append(ops.shortest_path_nodes(db.graph, *args) if lib is None else parent_call(lib, db.graph,
                                                                                                       *args))
            torch.cuda.synchronize()
        out[tag + "_us_per_batch"] = kernel_us(prof, steps, ("bfs_kernel", "mark_kernel", "paths_kernel"))
        out[tag + "_outputs"] = outs
    res = dict(batches=steps, mean_sources=round(float(np.mean([a[1].float().mean().item() for _d, a, _n, _p in
                                                                  batches])), 2),
               new_us_per_batch=out["new_us_per_batch"])
    if parent is not None:
        res["parent_us_per_batch"] = out["parent_us_per_batch"]
        res["parent_bit_equal"] = all(torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
                                      for a, b in zip(out["new_outputs"], out["parent_outputs"]))
    return res, [(n, pd) for _d, _a, n, pd in batches]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--questions", type=int, default=1280)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--targets", type=int, default=32)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--profile-steps", type=int, default=4)
    ap.add_argument("--parent-lib", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_paths_probe needs a CUDA device")
    info = gpu_info()
    dev = torch.device("cuda")
    parent = None
    if a.parent_lib:
        parent = ctypes.CDLL(os.path.abspath(a.parent_lib))
        for name in ("gr_paths_workspace_bytes", "gr_shortest_path_nodes"):
            rest, args = _lib.SIGNATURES[name]
            getattr(parent, name).restype, getattr(parent, name).argtypes = rest, args
    splits = {}
    T = a.targets
    for shape in a.shapes.split(","):
        name, B, over = SHAPES[shape]
        graft = name == "GraftNet"
        if graft not in splits:
            splits[graft] = loader.DeviceSplit(SyntheticSplit(a.questions, graft=graft), dev, weights="arrays",
                                               index_dtype=torch.int32)
        split = splits[graft]
        torch.manual_seed(0)
        m = {"ReaRev": G.ReaRev, "NSM": G.NSM, "GraftNet": G.GraftNet}[name](
            dict(S.model_args(name, use_cuda=True, **over)), NE, NR, NW).cuda().eval()
        step = graphed.GraphedStep(m, NE)

        def plain():
            return step.start_eval(split, B).result()

        def with_paths():
            run = step.start_eval(split, B, path_targets=T)
            return run.result(), run.paths()
        plain()
        _r, (sets, blocks) = with_paths()                        # captures
        secs = {"plain": [], "paths": []}
        for _ in range(a.runs):
            secs["plain"].append(timed(plain)[0])
            secs["paths"].append(timed(with_paths)[0])
        bfs, per_batch = bfs_section(m, split, B, T, a.profile_steps, parent)
        seeds = split.seed_counts()
        for it, (nodes, pair) in enumerate(per_batch):            # the run's node sets are the per-batch ones
            for b in range(len(nodes)):
                q = it * B + b
                assert sets[q] == nodes[b], q
                assert np.array_equal(blocks[q], pair[b, :seeds[q], :blocks[q].shape[1]]), q
        med = {k: float(np.median(v)) for k, v in secs.items()}
        res = dict(shape=shape, model=name, B=B, D=over["entity_dim"], N=split.N, questions=a.questions, T=T,
                   max_seeds=split.max_seeds(), nodes_per_q=round(float(np.mean([len(s) for s in sets])), 1),
                   gpu=info)
        for k, v in med.items():
            res[k + "_qps"] = round(a.questions / v, 1)
            res[k + "_s"] = [round(x, 4) for x in secs[k]]
        res["paths_cost"] = round(med["paths"] / med["plain"], 3)
        res["bfs"] = bfs
        print(json.dumps(res), flush=True)
        del step
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
