"""Milliseconds per training step, eager against graphed (graphed.GraphedTrainStep, GraphedGraftTrainStep), at the
reference's training shape.

    python scripts/train_graph_probe.py [--steps 50] [--warmup 10] [--runs 5] [--out train_graph_probe.json]

Shapes: d50 = ReaRev B 8, entity_dim 50, num_ins 3, num_iter 2, num_gnn 3, lstm (gnn/scripts/rearev_cwq.sh); cfg2 =
ReaRev B 64, entity_dim 200, num_ins 2, num_iter 3, num_gnn 3; graftnet_d50 = GraftNet B 8, entity_dim 50, num_layer 3,
lstm (the reference's GraftNet training shape); graftnet_cfg2 = GraftNet B 64, entity_dim 200, num_layer 3.  All on
WebQSP-shape synthetic subgraphs (N 2000, 6000 facts per question; GraftNet: the same facts as graft tuples), dropout
0.2 / 0.3 as in the reference's defaults.  One step = forward + backward + the train-time hit@1 / F1
as host lists (the tp_list train_epoch keeps), with or without the caller's clip_grad_norm_ + Adam.step(), and
"graphed+fused" with both in the graph (``optimizer=``, ``max_norm=``: optim.ClipAdam).  A run
times ``--steps`` steps between two CUDA events after ``--warmup`` steps; each mode runs ``--runs`` times, alternating
eager and graphed, and the median and the spread are reported.  The GPU's name, SM clock and power limit are read in
the same run and printed beside the numbers.  Last, the two clip + Adam kernels alone (gr_grad_sumsq + gr_clip_adam)
between CUDA events over ``--launches`` launches, with the bytes they move (sumsq reads each gradient; the update
reads and writes gradient, parameter and both moments)."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

import gnn_rag_b200 as G
from gnn_rag_b200 import graphed, synthetic as S

SHAPES = {
    "d50": dict(B=8, D=50, I=3, T=2, K=3),
    "cfg2": dict(B=64, D=200, I=2, T=3, K=3),
    "graftnet_d50": dict(model="GraftNet", B=8, D=50, L=3),
    "graftnet_cfg2": dict(model="GraftNet", B=64, D=200, L=3),
}


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), (s.strip() for s in out.split(","))))
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(), "error": str(e)}


def step_class(c):
    return graphed.GraphedGraftTrainStep if c.get("model") == "GraftNet" else graphed.GraphedTrainStep


def kernel_time(fused, launches):
    """(microseconds per gr_grad_sumsq + gr_clip_adam pair, bytes they move) of ``fused`` (an optim.ClipAdam)."""
    adam = set(fused._adam_rows)
    nbytes = sum(p.numel() * 4 * (1 + (8 if r in adam else 2)) for r, p in enumerate(fused.params))
    for _ in range(3):
        fused.launch()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(launches):
        fused.launch()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) * 1e3 / launches, nbytes


def build(c):
    """-> (model, two batches, the graphed step)."""
    torch.manual_seed(0)
    sizes = (S.WEBQSP_NUM_ENTITY, S.WEBQSP_NUM_RELATION, S.WEBQSP_NUM_WORD)
    if c.get("model") == "GraftNet":
        args = S.model_args("GraftNet", entity_dim=c["D"], num_layer=c["L"], use_cuda=True)
        m = G.GraftNet(dict(args), *sizes).cuda().train()
        batches = [S.make_graft_batch(s, B=c["B"], N=2000, E=6000) for s in (1, 2)]
        return m, batches, step_class(c)(m)
    args = S.model_args("ReaRev", entity_dim=c["D"], num_ins=c["I"], num_iter=c["T"], num_gnn=c["K"], use_cuda=True)
    m = G.ReaRev(dict(args), *sizes).cuda().train()
    batches = [S.make_batch(s, B=c["B"], N=2000, E=6000, with_weights=False)[:7] for s in (1, 2)]
    # the graphed step's buckets: both batches in one capacity bucket, so one graph serves the timed loop
    return m, batches, step_class(c)(m)


def time_mode(step_fn, batches, steps, warmup):
    for i in range(warmup):
        step_fn(batches[i % len(batches)])
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(steps):
        step_fn(batches[i % len(batches)])
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_graph_probe needs a CUDA device")
    res = dict(gpu=gpu_info(), steps=a.steps, warmup=a.warmup, runs=a.runs, results={})
    for name in a.shapes.split(","):
        c = SHAPES[name]
        m, batches, gstep = build(c)
        params = [p for p in m.parameters() if p.requires_grad]
        opt = torch.optim.Adam(params, lr=1e-4)
        fstep = step_class(c)(m, optimizer=opt, max_norm=1.0)

        def eager(b):
            loss, _pred, _pd, tp = m(b, training=True)
            loss.backward()
            return tp

        def graph(b):
            _loss, _pred, _pd, h1, f1 = gstep.step(b)
            return gstep.tp_list(h1, f1)

        def fused(b):
            _loss, _pred, _pd, h1, f1 = fstep.step(b)
            return fstep.tp_list(h1, f1)

        def with_opt(fn):
            def run(b):
                opt.zero_grad(set_to_none=True)
                tp = fn(b)
                torch.nn.utils.clip_grad_norm_(params, 1.0)
                opt.step()
                return tp
            return run

        def plain(fn):
            def run(b):
                opt.zero_grad(set_to_none=True)
                return fn(b)
            return run

        modes = {"eager": plain(eager), "graphed": plain(graph), "eager+clip+adam": with_opt(eager),
                 "graphed+clip+adam": with_opt(graph), "graphed+fused": fused}
        times = {k: [] for k in modes}
        for _ in range(a.runs):
            for k, fn in modes.items():           # alternating, so drift hits every mode alike
                times[k].append(time_mode(fn, batches, a.steps, a.warmup))
        out = {k: dict(median_ms=float(np.median(v)), min_ms=float(np.min(v)), max_ms=float(np.max(v)))
               for k, v in times.items()}
        out["graphs"] = len(gstep._cache)
        out["speedup"] = out["eager"]["median_ms"] / out["graphed"]["median_ms"]
        out["speedup_with_opt"] = out["eager+clip+adam"]["median_ms"] / out["graphed+clip+adam"]["median_ms"]
        out["tail_eager_ms"] = out["graphed+clip+adam"]["median_ms"] - out["graphed"]["median_ms"]
        out["tail_fused_ms"] = out["graphed+fused"]["median_ms"] - out["graphed"]["median_ms"]
        f = next(iter(fstep._cache.values())).fused
        us, nbytes = kernel_time(f, a.launches)
        out["clip_adam_kernels"] = dict(us=us, bytes=nbytes, gb_per_s=nbytes / us * 1e-3, tensors=len(f.params),
                                        elements=sum(p.numel() for p in f.params))
        res["results"][name] = dict(shape=c, **out)
        print(name, json.dumps(res["results"][name]))
        del gstep, fstep, m, opt
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
