"""Evaluation rate over a resident split: the per-batch Evaluator vs the evaluation epoch (GraphedStep.start_eval
through Evaluator(step=...)), and where the device time of an evaluation step goes.

A whole ``Evaluator.evaluate(split, test_batch_size=B)`` over a synthetic WebQSP-shape split
(scripts/device_split_probe.py: N = 2000 nodes, E = 6000 stored facts per question, self-loops on) held as a
``loader.DeviceSplit``, the ``.info`` file written as the reference forces it:

  per_batch         the Evaluator without a step: per batch an eager get_batch, an eager forward, retrieve() and
                    f1_and_hits in Python
  epoch             Evaluator(step=GraphedStep(model, NE)), warm: one graph replay per step, the rows formatted on
                    the device from its records (EvalRun.info) and written with one copy and one write
  epoch_after_step  the same right after an in-place Adam step on every parameter (untimed): what an evaluation
                    between training epochs costs; no graph is captured again
  first_epoch_s     the first evaluation of a new GraphedStep, captures included, timed on its own; ``capture_s`` is
                    it minus the median warm evaluation

Shapes: ReaRev, NSM and GraftNet at the reference's WebQSP evaluation (B 20, entity_dim 50) and cfg2 (ReaRev, B 64,
entity_dim 200).  ``cands_per_q`` is the mean retrieved count: the randomly initialised models' distributions are
flat, so the eps = 0.95 cut keeps most of a question's 1 000..2 000 entities and the ``.info`` rows are large.  The
questions/s of a mode is the median over ``--runs`` passes, the modes alternating, after one
untimed pass of each; both paths' files are compared byte for byte.  ``info`` splits the ``.info`` part of a warm
epoch (median of ``--runs``): gr_info_rows_size and gr_info_rows_write (CUDA events), the device-to-host copy of the
bytes into pinned memory and the file write (host clock); ``info_bytes`` is the file's size.  The one-time build of the
evaluator's host tables (``evaluate.InfoTables``: question prefixes and entity names) is timed on its own and printed
on a line of its own before the shape's.  Then one ``torch.profiler`` run per shape over ``--profile-steps`` steps of each path (a split
of that many batches): per step, the launches and device time of every kernel, and the kernels the evaluation graph
launches more often than the per-batch forward (the weight formatting the graphs redo on every replay,
``ops.graph_private_weights``).  The GPU's name and power limit are read in the same run.  One JSON line per shape.

    python scripts/eval_split_probe.py [--questions 1280] [--runs 3] [--shapes ...] [--out eval_split_probe.json]
"""
import argparse
import collections
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import gnn_rag_b200 as G                                        # noqa: E402
from gnn_rag_b200 import evaluate, graphed, loader, synthetic as S  # noqa: E402
from device_split_probe import NE, NR, NW, SyntheticSplit, gpu_info  # noqa: E402

SHAPES = {   # name -> model, batch size, model arguments
    "rearev_d50": ("ReaRev", 20, dict(entity_dim=50, num_ins=3, num_iter=2, num_gnn=3)),
    "nsm_d50": ("NSM", 20, dict(entity_dim=50)),
    "graftnet_d50": ("GraftNet", 20, dict(entity_dim=50)),
    "cfg2": ("ReaRev", 64, dict(entity_dim=200, num_ins=2, num_iter=3, num_gnn=3)),
}
ENT = None           # entity2id of the synthetic vocabulary (NE entries: the pad id is NE)


class EvalSplit(SyntheticSplit):
    """SyntheticSplit + the ``get_quest`` the evaluator's ``.info`` rows read."""

    def get_quest(self, training=False):
        return ["question %d" % s for s in self.sample_ids]


def evaluator(name, m, tmp, step=None):
    args = dict(S.model_args(name), checkpoint_dir=tmp, experiment_name=name)
    return evaluate.Evaluator(args, m, ENT, {"r%d" % i: i for i in range(NR)}, torch.device("cuda"), step=step)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def optimizer_step(m, opt, g):
    """One in-place Adam step on every parameter, from small random gradients."""
    for p in opt.param_groups[0]["params"]:
        p.grad = torch.randn(p.shape, device=p.device, generator=g) * 1e-3
    opt.step()
    opt.zero_grad(set_to_none=True)


def kernel_table(prof, steps):
    """name -> [launches per step, device us per step] of the CUDA kernels of a profile."""
    tab = collections.defaultdict(lambda: [0.0, 0.0])
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name and "Memset" not in e.name:
            tab[e.name][0] += 1.0 / steps
            tab[e.name][1] += e.time_range.elapsed_us() / steps
    return tab


def profile(name, m, B, steps, tmp):
    """torch.profiler of ``steps`` batches through each path -> per-step kernel tables and the difference."""
    L = EvalSplit(steps * B, graft=name == "GraftNet", seed=1)
    split = loader.DeviceSplit(L, torch.device("cuda"), weights="arrays", index_dtype=torch.int32)
    step = graphed.GraphedStep(m, NE)
    ev_b, ev_e = evaluator(name, m, tmp), evaluator(name, m, tmp, step=step)
    ev_b.evaluate(split, B)
    ev_e.evaluate(split, B)                       # captures
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    tabs = {}
    for k, ev in (("per_batch", ev_b), ("epoch", ev_e)):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=acts) as prof:
            ev.evaluate(split, B)
            torch.cuda.synchronize()
        tabs[k] = kernel_table(prof, steps)
    extra = {}
    for kname, (n, us) in tabs["epoch"].items():
        nb = tabs["per_batch"].get(kname, [0.0, 0.0])[0]
        if n > nb + 1e-9:
            extra[kname[:90]] = dict(launches=round(n - nb, 2), us_per_launch=round(us / n, 2))
    summary = {}
    for k, tab in tabs.items():
        summary[k] = dict(launches_per_step=round(sum(v[0] for v in tab.values()), 1),
                          kernel_us_per_step=round(sum(v[1] for v in tab.values()), 1),
                          top=[(n[:60], round(v[0], 2), round(v[1], 1))
                               for n, v in sorted(tab.items(), key=lambda kv: -kv[1][1])[:8]])
    summary["extra_in_epoch"] = extra
    summary["extra_us_per_step"] = round(sum(v["launches"] * v["us_per_launch"] for v in extra.values()), 1)
    return summary


def info_parts(ev, step, split, B, runs, path):
    """Median seconds of each part of ``EvalRun.info`` + the file write over ``runs`` warm evaluations."""
    from gnn_rag_b200 import ops
    tables = ev.info_tables(split)
    parts = collections.defaultdict(list)
    for _ in range(runs):
        run = step.start_eval(split, B)
        run.check()
        n = run.num_data
        v = graphed._EvalBuffers.views(run.blob, n)
        recs = (v["metrics"], v["cases"], v["counts"], v["cand_off"], v["cand_total"])
        row_off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
        summary = torch.empty(2, dtype=torch.int64, device="cuda")
        ev0, ev1, ev2, ev3 = (torch.cuda.Event(enable_timing=True) for _ in range(4))
        ev0.record()
        ops.info_rows_size(*recs, v["status"], run.cand, run.order, tables, row_off, summary)
        ev1.record()
        total = int(summary[0])
        out = torch.empty(max(total, 1), dtype=torch.uint8, device="cuda")
        ev2.record()
        ops.info_rows_write(*recs, run.cand, run.order, tables, row_off, summary, out)
        ev3.record()
        host = torch.empty(total, dtype=torch.uint8, pin_memory=True)
        t_copy, _ = timed(lambda: host.copy_(out[:total]))
        t0 = time.perf_counter()
        with open(path, "wb") as f:
            f.write(host.numpy())
        parts["write_s"].append(time.perf_counter() - t0)
        parts["size_kernels_ms"].append(ev0.elapsed_time(ev1))
        parts["write_kernel_ms"].append(ev2.elapsed_time(ev3))
        parts["d2h_ms"].append(t_copy * 1e3)
        parts["bytes"] = [total]
    return {k: round(float(np.median(x)), 4) for k, x in parts.items()}


def main():
    global ENT
    ap = argparse.ArgumentParser()
    ap.add_argument("--questions", type=int, default=1280)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--profile-steps", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_split_probe needs a CUDA device")
    info = gpu_info()
    dev = torch.device("cuda")
    ENT = {"e%d" % i: i for i in range(NE)}
    tmp = tempfile.mkdtemp(prefix="eval_split_probe")
    splits = {}
    results = []
    for shape in a.shapes.split(","):
        name, B, over = SHAPES[shape]
        graft = name == "GraftNet"
        if graft not in splits:
            L = EvalSplit(a.questions, graft=graft)
            splits[graft] = loader.DeviceSplit(L, dev, weights="arrays", index_dtype=torch.int32)
        split = splits[graft]
        torch.manual_seed(0)
        m = {"ReaRev": G.ReaRev, "NSM": G.NSM, "GraftNet": G.GraftNet}[name](
            dict(S.model_args(name, use_cuda=True, **over)), NE, NR, NW).cuda().eval()
        opt = torch.optim.Adam([p for p in m.parameters() if p.requires_grad], lr=1e-4)
        gen = torch.Generator(device=dev).manual_seed(0)
        ev_b = evaluator(name, m, tmp)
        step = graphed.GraphedStep(m, NE)
        ev_e = evaluator(name, m, tmp, step=step)
        t_tables, _ = timed(lambda: ev_e.info_tables(split))
        print(json.dumps(dict(shape=shape, info_tables_s=round(t_tables, 3), questions=a.questions, gpu=info)),
              flush=True)
        first, want = timed(lambda: ev_e.evaluate(split, B))
        path = os.path.join(tmp, name + "_test.info")
        with open(path, "rb") as f:
            want_file = f.read()
        graphs = len(step._cache)
        cands = float(np.mean([len(r) for r in step.evaluate_split(split, B)[6]]))
        got = ev_b.evaluate(split, B)                 # untimed pass of the per-batch path
        assert got == want, (got, want)
        with open(path, "rb") as f:
            assert f.read() == want_file

        def after_step():
            optimizer_step(m, opt, gen)
            return timed(lambda: ev_e.evaluate(split, B))[0]
        secs = {"per_batch": [], "epoch": [], "epoch_after_step": []}
        for _ in range(a.runs):
            secs["per_batch"].append(timed(lambda: ev_b.evaluate(split, B))[0])
            secs["epoch"].append(timed(lambda: ev_e.evaluate(split, B))[0])
            secs["epoch_after_step"].append(after_step())
        assert len(step._cache) == graphs
        # after the optimizer steps both paths still agree
        assert ev_b.evaluate(split, B) == ev_e.evaluate(split, B)
        med = {k: float(np.median(v)) for k, v in secs.items()}
        plan = graphed.epoch_plan(np.arange(a.questions), split._stored, split._ents, B, 0.0,
                                  split._graft_count if graft else None)
        res = dict(shape=shape, model=name, B=B, D=over["entity_dim"], N=split.N, E=6000, questions=a.questions,
                   steps=plan.steps, graphs=graphs, cands_per_q=round(cands, 1), gpu=info)
        for k, v in med.items():
            res[k + "_qps"] = round(a.questions / v, 1)
            res[k + "_s"] = [round(x, 4) for x in secs[k]]
        res["first_epoch_s"] = round(first, 3)         # the tables were built before it
        res["capture_s"] = round(first - med["epoch"], 3)
        res["speedup"] = round(med["per_batch"] / med["epoch"], 2)
        res["info"] = info_parts(ev_e, step, split, B, a.runs, os.path.join(tmp, "parts.info"))
        res["profile"] = profile(name, m, B, a.profile_steps, tmp)
        results.append(res)
        print(json.dumps(res), flush=True)
        del step, ev_e
        torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as f:
            for r in results:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
