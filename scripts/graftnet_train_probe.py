"""GraftNet training step on one GPU: the kernel path of ``model(batch, training=True)`` (fact attention, fact messages
and TypeLayer in csrc/graft.cu / csrc/aggregate_bwd.cu) against the per-fact torch path (``autograd_path.USE_KERNELS =
False``), alternating in one run.

    python scripts/graftnet_train_probe.py [--B 64] [--N 2000] [--E 6000] [--dims 50,200] [--steps 10] [--warmup 2]
                                           [--dropout 0.2] [--out results/graftnet_train_probe.json]

One step = forward + backward + Adam step from the loader's numpy tuple, as ``Trainer_KBQA.train_epoch`` runs it
(gnn/train_model.py:219-231).  Step time: host clock between device synchronisations (the step reads metrics back to
the host itself), median over ``--steps`` per path.  Peak memory: ``torch.cuda.max_memory_allocated`` over each path's
steps, reset before them, and the same less what was allocated before the step (parameters, Adam state).  The card name
and power limit are read in the same run (nvidia-smi query only)."""
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
from gnn_rag_b200 import autograd_path, synthetic as S  # noqa: E402

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


def step(m, opt, batch):
    opt.zero_grad(set_to_none=True)
    loss = m(batch, training=True)[0]
    loss.backward()
    opt.step()
    return float(loss.detach())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=64)
    ap.add_argument("--N", type=int, default=2000)
    ap.add_argument("--E", type=int, default=6000)
    ap.add_argument("--dims", default="50,200")
    ap.add_argument("--layers", type=int, default=3)
    ap.add_argument("--dropout", type=float, default=0.2)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("graftnet_train_probe measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    name, power = card()
    res = dict(card=name, power_limit=power, B=a.B, N=a.N, E=a.E, layers=a.layers, linear_dropout=a.dropout, dims={})
    batch = S.make_graft_batch(0, a.B, a.N, a.E, num_entity=NUM_ENTITY, num_relation=NUM_REL, num_word=NUM_WORD,
                               with_weights=False, test=False)
    res["graft_facts"] = int(len(batch[3][0][0]))
    res["kb_facts"] = int(len(batch[2][0]))
    res["max_fact"] = int(batch[5].shape[1])
    paths = {"kernels": True, "torch": False}
    for D in [int(x) for x in a.dims.split(",")]:
        args = S.model_args("GraftNet", entity_dim=D, num_layer=a.layers, word_dim=300, use_cuda=True,
                            linear_dropout=a.dropout)
        torch.manual_seed(0)
        m = G.GraftNet(dict(args), NUM_ENTITY, NUM_REL, NUM_WORD).cuda().train()
        opt = torch.optim.Adam([p for p in m.parameters() if p.requires_grad], lr=1e-4)
        times = {k: [] for k in paths}
        peak = {k: 0 for k in paths}
        peak_step = {k: 0 for k in paths}
        losses = {k: [] for k in paths}
        try:
            for k, mode in paths.items():          # warm-up (module loads, cuBLAS heuristics, Adam state)
                autograd_path.USE_KERNELS = mode
                for _ in range(a.warmup):
                    step(m, opt, batch)
            for _ in range(a.steps):
                for k, mode in paths.items():      # alternate the two paths
                    autograd_path.USE_KERNELS = mode
                    torch.cuda.synchronize()
                    base = torch.cuda.memory_allocated()
                    torch.cuda.reset_peak_memory_stats()
                    t0 = time.perf_counter()
                    losses[k].append(step(m, opt, batch))
                    torch.cuda.synchronize()
                    times[k].append(1e3 * (time.perf_counter() - t0))
                    mx = torch.cuda.max_memory_allocated()
                    peak[k] = max(peak[k], mx)
                    peak_step[k] = max(peak_step[k], mx - base)
        finally:
            autograd_path.USE_KERNELS = True
        r = {}
        for k in paths:
            r[k] = dict(step_ms_median=float(np.median(times[k])), step_ms_min=float(np.min(times[k])),
                        step_ms_max=float(np.max(times[k])), peak_mem_gb=peak[k] / 1e9,
                        peak_step_mem_gb=peak_step[k] / 1e9, loss_first=losses[k][0], loss_last=losses[k][-1])
        r["speedup_median"] = r["torch"]["step_ms_median"] / r["kernels"]["step_ms_median"]
        r["peak_step_mem_ratio_torch_over_kernels"] = peak_step["torch"] / max(peak_step["kernels"], 1)
        res["dims"][D] = r
        print(json.dumps({D: r}))
        del m, opt
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
