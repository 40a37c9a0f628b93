"""Training step on one GPU, two paths alternating in one run.

    python scripts/graftnet_train_probe.py [--model graftnet|rearev|nsm] [--compare torch|det|amp] [--B 64]
                                           [--N 2000] [--E 6000] [--dims 50,200] [--num_ins 2] [--num_iter 3]
                                           [--steps 10] [--warmup 2] [--dropout 0.2] [--out results/train_probe.json]

``--compare torch`` (GraftNet only): the kernel path of ``model(batch, training=True)`` (fact attention, fact messages
and TypeLayer in csrc/graft.cu / csrc/aggregate_bwd.cu) against the per-fact torch path (``autograd_path.USE_KERNELS =
False``).  ``--compare det``: the default backward kernels against the deterministic ones
(``torch.use_deterministic_algorithms(True)``; CUBLAS_WORKSPACE_CONFIG is set before torch is imported), with the
device time of every backward kernel class from CUDA events in one extra step per mode.  ``--compare amp``: fp32
against ``torch.autocast("cuda", dtype=torch.bfloat16)`` around the forward (bf16 node-tensor I/O in the training
kernels); with ``--model rearev`` it also times, at B x N x E, D = 200, I = 2, the aggregation forward and backward
with bf16 I/O against the alternative of casting at the Function boundary (fp32 kernel, then ``.to(bf16)``; backward:
``grad_out.float()``, then the fp32 kernel).

One step = forward + backward + clip_grad_norm_ + Adam step from the loader's numpy tuple, as
``Trainer_KBQA.train_epoch`` runs it (gnn/train_model.py:219-231).  Step time: host clock between device synchronisations (the step reads metrics back to
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

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")      # before cuBLAS starts: the deterministic mode needs it
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import gnn_rag_b200 as G  # noqa: E402
from gnn_rag_b200 import autograd_path, ops, synthetic as S  # noqa: E402

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


AMP = False      # --compare amp: the forward runs under bf16 autocast


def step(m, opt, batch):
    opt.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=AMP):
        loss = m(batch, training=True)[0]
    loss.backward()
    torch.nn.utils.clip_grad_norm_([p for p in m.parameters() if p.requires_grad], 1.0)
    opt.step()
    return float(loss.detach())


def set_mode(compare, mode):
    global AMP
    if compare == "torch":
        autograd_path.USE_KERNELS = mode
    elif compare == "amp":
        AMP = mode
    else:
        torch.use_deterministic_algorithms(mode)


def aggregation_io(batch, D=200, I=2, reps=50):
    """Median device ms of one aggregation direction, forward and backward, with bf16 output / bf16 grad_out in the
    kernels against casting at the Function boundary around the fp32 kernels."""
    from gnn_rag_b200 import batching
    g = batching.stage_batch(batch, torch.device("cuda"), NUM_REL + 1).graph
    gen = torch.Generator(device="cuda").manual_seed(0)
    table = torch.randn(NUM_REL + 1, D, device="cuda", generator=gen)
    ins = torch.randn(g.B, I, D, device="cuda", generator=gen)
    prior = torch.softmax(torch.randn(g.B, g.N, device="cuda", generator=gen), 1)
    G16 = torch.randn(g.B * g.N, I * D, device="cuda", generator=gen).to(torch.bfloat16)
    bufs = [torch.zeros_like(t) for t in (table, ins, prior)]
    variants = {
        "fwd_bf16_io": lambda: ops.aggregate(g, "fwd", prior, table, ins, dtype=torch.bfloat16),
        "fwd_fp32_then_cast": lambda: ops.aggregate(g, "fwd", prior, table, ins).to(torch.bfloat16),
        "bwd_bf16_io": lambda: ops.aggregate_backward(g, "fwd", prior, table, ins, G16, *bufs),
        "bwd_cast_then_fp32": lambda: ops.aggregate_backward(g, "fwd", prior, table, ins, G16.float(), *bufs),
    }
    ms = {k: [] for k in variants}
    for fn in variants.values():
        fn()
    for _ in range(reps):
        for k, fn in variants.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            e.synchronize()
            ms[k].append(s.elapsed_time(e))
    return dict(B=g.B, N=g.N, F=g.F, D=D, I=I, reps=reps, **{k + "_ms_median": float(np.median(v)) for k, v in ms.items()})


def backward_kernel_ms(m, opt, batch):
    """Device time (ms) per backward kernel class in one step, from the CUDA events ops records around each call."""
    ops.STATS.reset()
    ops.STATS.time_ops = True
    try:
        step(m, opt, batch)
        torch.cuda.synchronize()
    finally:
        ops.STATS.time_ops = False
    out = {}
    for s, e, cls, _info in ops.STATS.op_events:
        if "bwd" in cls:
            out[cls] = out.get(cls, 0.0) + s.elapsed_time(e)
    ops.STATS.reset()
    return out


def make_model(model, D, layers, dropout, num_ins=2, num_iter=3):
    if model == "graftnet":
        args = S.model_args("GraftNet", entity_dim=D, num_layer=layers, word_dim=300, use_cuda=True,
                            linear_dropout=dropout)
        return G.GraftNet(dict(args), NUM_ENTITY, NUM_REL, NUM_WORD)
    if model == "rearev":
        args = S.model_args("ReaRev", entity_dim=D, num_iter=num_iter, num_ins=num_ins, num_gnn=3, word_dim=300,
                            use_cuda=True, linear_dropout=dropout)
        return G.ReaRev(dict(args), NUM_ENTITY, NUM_REL, NUM_WORD)
    args = S.model_args("NSM", entity_dim=D, num_step=3, word_dim=300, use_cuda=True, linear_dropout=dropout)
    return G.NSM(dict(args), NUM_ENTITY, NUM_REL, NUM_WORD)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=["graftnet", "rearev", "nsm"], default="graftnet")
    ap.add_argument("--compare", choices=["torch", "det", "amp"], default="torch")
    ap.add_argument("--B", type=int, default=64)
    ap.add_argument("--N", type=int, default=2000)
    ap.add_argument("--E", type=int, default=6000)
    ap.add_argument("--dims", default="50,200")
    ap.add_argument("--layers", type=int, default=3)
    ap.add_argument("--num_ins", type=int, default=2)       # ReaRev
    ap.add_argument("--num_iter", type=int, default=3)      # ReaRev
    ap.add_argument("--dropout", type=float, default=0.2)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("graftnet_train_probe measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    name, power = card()
    if a.compare == "torch" and a.model != "graftnet":
        raise SystemExit("--compare torch is a GraftNet comparison")
    res = dict(card=name, power_limit=power, model=a.model, compare=a.compare, B=a.B, N=a.N, E=a.E, layers=a.layers,
               linear_dropout=a.dropout, dims={})
    if a.model == "rearev":
        res.update(num_ins=a.num_ins, num_iter=a.num_iter, num_gnn=3)
    if a.model == "graftnet":
        batch = S.make_graft_batch(0, a.B, a.N, a.E, num_entity=NUM_ENTITY, num_relation=NUM_REL, num_word=NUM_WORD,
                                   with_weights=False, test=False)
        res["graft_facts"] = int(len(batch[3][0][0]))
        res["max_fact"] = int(batch[5].shape[1])
    else:
        batch = S.make_batch(0, a.B, a.N, a.E, num_entity=NUM_ENTITY, num_relation=NUM_REL, num_word=NUM_WORD,
                             test=False)
    res["kb_facts"] = int(len(batch[2][0]))
    paths = {"torch": {"kernels": True, "torch": False}, "det": {"default": False, "deterministic": True},
             "amp": {"fp32": False, "bf16_autocast": True}}[a.compare]
    if a.compare == "amp" and a.model == "rearev":
        res["aggregation_io"] = aggregation_io(batch)
        print(json.dumps(res["aggregation_io"]))
    for D in [int(x) for x in a.dims.split(",")]:
        torch.manual_seed(0)
        m = make_model(a.model, D, a.layers, a.dropout, a.num_ins, a.num_iter).cuda().train()
        opt = torch.optim.Adam([p for p in m.parameters() if p.requires_grad], lr=1e-4)
        times = {k: [] for k in paths}
        peak = {k: 0 for k in paths}
        peak_step = {k: 0 for k in paths}
        losses = {k: [] for k in paths}
        try:
            for k, mode in paths.items():          # warm-up (module loads, cuBLAS heuristics, Adam state)
                set_mode(a.compare, mode)
                for _ in range(a.warmup):
                    step(m, opt, batch)
            for _ in range(a.steps):
                for k, mode in paths.items():      # alternate the two paths
                    set_mode(a.compare, mode)
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
            kernel_ms = {}
            for k, mode in paths.items():
                set_mode(a.compare, mode)
                kernel_ms[k] = backward_kernel_ms(m, opt, batch)
        finally:
            autograd_path.USE_KERNELS = True
            torch.use_deterministic_algorithms(False)
            set_mode("amp", False)
        r = {}
        for k in paths:
            r[k] = dict(step_ms_median=float(np.median(times[k])), step_ms_min=float(np.min(times[k])),
                        step_ms_max=float(np.max(times[k])), peak_mem_gb=peak[k] / 1e9,
                        peak_step_mem_gb=peak_step[k] / 1e9, loss_first=losses[k][0], loss_last=losses[k][-1],
                        backward_kernel_ms=kernel_ms[k])
        slow, fast = list(paths)[1], list(paths)[0]
        r["step_time_ratio_%s_over_%s" % (slow, fast)] = r[slow]["step_ms_median"] / r[fast]["step_ms_median"]
        r["peak_step_mem_ratio_%s_over_%s" % (slow, fast)] = peak_step[slow] / max(peak_step[fast], 1)
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
