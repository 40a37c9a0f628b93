"""Aggregate training rate of K runs side by side on one GPU (graphed.Sweep) against the same K runs one after another.

K independent ReaRev / NSM / GraftNet runs (each its own model, Adam and generator; all over one synthetic WebQSP-shape
split, as seeds of one dataset are) train one epoch each:

  solo   K ``start_epoch`` calls one after another, then one device synchronisation
  sweep  one ``Sweep.start_epochs`` over the K members, then one device synchronisation

for K = 1, 2, 4, 8, the two alternating within the run after one warm-up epoch of each (graph capture).  The rate is
training questions per second over all K runs (K x questions / seconds, median over ``--runs``).  One more sweep mixes
evaluation members in: two members train, then two evaluation-only members of the same family and shape evaluate the
split (``start_epochs`` and then ``start_evals``, one synchronisation), against the same work done solo, one run after
another.  Each call overlaps its own members only, so the two trainings overlap each other, then the two
evaluations do; training and evaluation do not overlap.

Shapes: the reference's training shape (``--batch_size 8 --entity_dim 50``) for ReaRev, NSM and GraftNet, and ReaRev at
cfg2 (B 64, entity_dim 200).  The card's name and power limit are read in the same run (an nvidia-smi query only).
One JSON line per (shape, K); a configuration that runs out of device memory is reported as such.

    python scripts/sweep_probe.py [--questions 1280] [--runs 3] [--shapes rearev_d50,nsm_d50,graftnet_d50,cfg2]
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

import gnn_rag_b200 as G                                          # noqa: E402
from gnn_rag_b200 import graphed, loader, synthetic as S          # noqa: E402
from device_split_probe import NE, NR, NW, SyntheticSplit, gpu_info  # noqa: E402

SHAPES = {   # name -> model, batch size, model arguments, member counts, questions (None: --questions)
    "rearev_d50": ("ReaRev", 8, dict(entity_dim=50, num_ins=3, num_iter=2, num_gnn=3), (1, 2, 4, 8), None),
    "nsm_d50": ("NSM", 8, dict(entity_dim=50), (1, 2, 4, 8), None),
    "graftnet_d50": ("GraftNet", 8, dict(entity_dim=50), (1, 2, 4, 8), None),
    "cfg2": ("ReaRev", 64, dict(entity_dim=200, num_ins=2, num_iter=3, num_gnn=3), (1, 2, 4, 8), 256),
}


def build(name, over, seed):
    torch.manual_seed(seed)
    args = S.model_args(name, use_cuda=True, **over)
    cls = {"ReaRev": G.ReaRev, "NSM": G.NSM, "GraftNet": G.GraftNet}[name]
    return cls(dict(args), NE, NR, NW).cuda()


def train_step(name, m):
    opt = torch.optim.Adam([p for p in m.parameters() if p.requires_grad], lr=5e-4)
    cls = graphed.GraphedGraftTrainStep if name == "GraftNet" else graphed.GraphedTrainStep
    return cls(m, optimizer=opt, max_norm=1.0)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def probe(shape, questions, runs):
    name, B, over, ks, nq = SHAPES[shape]
    nq = nq or questions
    L = SyntheticSplit(nq, graft=name == "GraftNet", seed=1)
    split = loader.DeviceSplit(L, torch.device("cuda"), shuffle=True, weights="none", index_dtype=torch.int32)
    K = max(ks)
    steps = [train_step(name, build(name, over, k)) for k in range(K)]
    sweep = graphed.Sweep(steps)
    job = (split, B, 0.0)

    def solo(k):
        for s in steps[:k]:
            s.start_epoch(*job)

    def swept(k):
        sweep.start_epochs([job] * k + [None] * (K - k))

    out = []
    for k in ks:
        row = dict(shape=shape, model=name, B=B, entity_dim=over["entity_dim"], questions=nq, K=k)
        try:
            solo(k)                                                 # warm-up: captures
            swept(k)
            t = {"solo": [], "sweep": []}
            for _ in range(runs):
                t["solo"].append(timed(lambda: solo(k)))
                t["sweep"].append(timed(lambda: swept(k)))
            med = {m: float(np.median(v)) for m, v in t.items()}
            row.update({m + "_q_per_s": round(k * nq / med[m], 1) for m in med})
            row.update({m + "_s": [round(x, 4) for x in t[m]] for m in t})
            row["sweep_over_solo"] = round(med["solo"] / med["sweep"], 3)
        except torch.cuda.OutOfMemoryError as e:
            row["error"] = "out of device memory: %s" % str(e).splitlines()[0][:120]
            torch.cuda.empty_cache()
        print(json.dumps(row), flush=True)
        out.append(row)
    if shape != "cfg2":
        out.append(mixed(name, B, over, split, steps, sweep, nq, runs))
    return out


def mixed(name, B, over, split, steps, sweep, nq, runs):
    """Members 0, 1 train, then two evaluation-only members evaluate the split, in one sweep; solo: the same work one
    run after another."""
    evals = [graphed.GraphedStep(build(name, over, 100 + k).eval(), NE) for k in range(2)]
    mix = graphed.Sweep(steps[:2] + evals)
    train_jobs = [(split, B, 0.0)] * 2 + [None, None]
    eval_jobs = [None, None] + [(split, B)] * 2

    def solo():
        for s in steps[:2]:
            s.start_epoch(split, B, 0.0)
        for e in evals:
            e.start_eval(split, B)

    def swept():
        mix.start_epochs(train_jobs)
        mix.start_evals(eval_jobs)
    row = dict(shape="mixed_" + name, model=name, B=B, entity_dim=over["entity_dim"], questions=nq, K=4,
               training=2, evaluating=2)
    try:
        solo()
        swept()
        t = {"solo": [], "sweep": []}
        for _ in range(runs):
            t["solo"].append(timed(solo))
            t["sweep"].append(timed(swept))
        med = {m: float(np.median(v)) for m, v in t.items()}
        row.update({m + "_q_per_s": round(4 * nq / med[m], 1) for m in med})
        row.update({m + "_s": [round(x, 4) for x in t[m]] for m in t})
        row["sweep_over_solo"] = round(med["solo"] / med["sweep"], 3)
    except torch.cuda.OutOfMemoryError as e:
        row["error"] = "out of device memory: %s" % str(e).splitlines()[0][:120]
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--questions", type=int, default=1280)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out", default=None, help="also write the rows as JSON to this file")
    a = ap.parse_args()
    shapes = [s for s in a.shapes.split(",") if s]
    unknown = [s for s in shapes if s not in SHAPES]
    if unknown:
        ap.error("unknown shapes %s (known: %s)" % (unknown, ", ".join(SHAPES)))
    if not torch.cuda.is_available():
        sys.exit("sweep_probe: no CUDA device; the rates are measured on the GPU")
    card = gpu_info()
    print(json.dumps(dict(card=card)), flush=True)
    rows = []
    for s in shapes:
        rows += probe(s, a.questions, a.runs)
        torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(card=card, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
