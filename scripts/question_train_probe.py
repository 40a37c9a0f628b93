"""Training step with the question side on the kernels against the torch question side, alternating in one run.

    python scripts/question_train_probe.py [--steps 10] [--warmup 2] [--dropout 0.2] [--out DIR/question_train.json]

Kernel path: the instruction steps in gr_instructions_train / gr_instructions_backward and ReaRev's query reform in
gr_query_reform_ex / gr_query_reform_backward (autograd_path._InstructionsFn, _QueryReformFn).  Torch path: the same
model with those two Functions switched off (the torch restatement of autograd_path._instructions and the reform
loop); everything else is the same in both.  Workloads: ReaRev at the shipped shapes (B = 8, D = 50, I = 2, T = 3 and
I = 3, T = 2), NSM at B = 8, D = 50 (3 steps), and ReaRev at cfg2 (B = 64, N = 2000, D = 200, I = 2, T = 3).

One step = forward + backward + clip_grad_norm_ + Adam step, as Trainer_KBQA.train_epoch runs it.  Step time: host
clock between device synchronisations, median over ``--steps`` per path, the paths alternating step by step.  Device
time of the question-side kernels: CUDA events around each of their calls (ops' "question_train" class) in one extra
step of the kernel path.  The card name and power limit are read in the same run (nvidia-smi query only)."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import gnn_rag_b200 as G  # noqa: E402
from gnn_rag_b200 import autograd_path, ops, synthetic as S  # noqa: E402
from graftnet_train_probe import card  # noqa: E402

NUM_ENTITY, NUM_REL, NUM_WORD = 100_000, 6106, 5000
WORKLOADS = {
    "rearev_webqsp_b8_d50_i2_t3": ("ReaRev", dict(B=8, N=2000, E=8000), dict(entity_dim=50, num_ins=2, num_iter=3)),
    "rearev_cwq_b8_d50_i3_t2": ("ReaRev", dict(B=8, N=2000, E=8000), dict(entity_dim=50, num_ins=3, num_iter=2)),
    "nsm_b8_d50": ("NSM", dict(B=8, N=2000, E=8000), dict(entity_dim=50, num_step=3)),
    "rearev_cfg2_b64_d200_i2_t3": ("ReaRev", dict(B=64, N=2000, E=8000), dict(entity_dim=200, num_ins=2, num_iter=3)),
}

_REAL = (autograd_path._instruction_kernels, autograd_path._reform_kernels)


def set_kernels(on):
    autograd_path._instruction_kernels = _REAL[0] if on else (lambda *a: False)
    autograd_path._reform_kernels = _REAL[1] if on else (lambda *a: False)


def step(m, opt, batch):
    opt.zero_grad(set_to_none=True)
    loss = m(batch, training=True)[0]
    loss.backward()
    torch.nn.utils.clip_grad_norm_([p for p in m.parameters() if p.requires_grad], 1.0)
    opt.step()
    return float(loss.detach())


def question_kernel_ms(m, opt, batch):
    ops.STATS.reset()
    ops.STATS.time_ops = True
    try:
        step(m, opt, batch)
        torch.cuda.synchronize()
    finally:
        ops.STATS.time_ops = False
    ms = sum(s.elapsed_time(e) for s, e, cls, _i in ops.STATS.op_events if cls == "question_train")
    ops.STATS.reset()
    return ms


def run(name, a):
    model, bshape, over = WORKLOADS[name]
    kw = dict(use_cuda=True, linear_dropout=a.dropout, word_dim=300)
    if model == "ReaRev":
        kw["num_gnn"] = 3
    kw.update(over)
    torch.manual_seed(0)
    m = getattr(G, model)(dict(S.model_args(model, **kw)), NUM_ENTITY, NUM_REL, NUM_WORD).cuda().train()
    batch = S.make_batch(0, bshape["B"], bshape["N"], bshape["E"], num_entity=NUM_ENTITY, num_relation=NUM_REL,
                         num_word=NUM_WORD, powerlaw=True, with_weights=True)
    opt = torch.optim.Adam([p for p in m.parameters() if p.requires_grad], lr=1e-4)
    times = {True: [], False: []}
    for i in range(a.warmup + a.steps):
        for on in (True, False):
            set_kernels(on)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            step(m, opt, batch)
            torch.cuda.synchronize()
            if i >= a.warmup:
                times[on].append((time.perf_counter() - t0) * 1e3)
    set_kernels(True)
    qk = question_kernel_ms(m, opt, batch)
    res = dict(model=model, **bshape, **over, dropout=a.dropout, steps=a.steps,
               step_ms_kernels=float(np.median(times[True])), step_ms_torch=float(np.median(times[False])),
               question_kernels_ms_per_step=qk)
    res["speedup"] = res["step_ms_torch"] / res["step_ms_kernels"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--dropout", type=float, default=0.2)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("question_train_probe needs a CUDA device")
    gpu, power = card()
    results = []
    for name in a.workloads.split(","):
        r = run(name, a)
        r["workload"] = name
        print(json.dumps(r), flush=True)
        results.append(r)
    out = dict(gpu=gpu, power_limit=power, results=results)
    print(json.dumps(dict(gpu=gpu, power_limit=power)))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
