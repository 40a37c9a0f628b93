"""Device time of the cfg2 dense-layer GEMM (grouped K order, M = 64 x 2000, N = 200, K = 5 x 208) in the three forms a
ReaRev forward launches it in the last layer of an iteration:

  full            fp32 h of every row + the next layer's hi/lo planes + the score dots (every last layer, before the
                  seed-row output; still every layer that is not the last of an iteration, without the fp32 h)
  seed_rows       fp32 h of the seed rows only (out_rows = query_entities) + planes + dots: iterations t < T - 1
  full_no_planes  fp32 h of every row + dots, no planes: the last layer of the last iteration

CUDA events around each launch, a 256 MiB write between launches (L2 flushed, as between bench.py steps), the forms
interleaved, the median over --reps launches each.  Prints one JSON line with the card and its power limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gnn_rag_b200 import ops  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        out = ""
    return dict(zip(q.split(","), (v.strip() for v in out.split(",")))) if out else {"name": torch.cuda.get_device_name()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=64)
    ap.add_argument("--N", type=int, default=2000)
    ap.add_argument("--seeds", type=int, default=2, help="seed rows per question")
    ap.add_argument("--reps", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("seed_rows_probe.py needs a CUDA device")
    dev = "cuda"
    D, P, I = 200, 208, 2
    M, K = a.B * a.N, (2 * I + 1) * P
    kp = (ops.k_order_nb0(P) + 2 * I * P + 63) // 64 * 64
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(M, kp, device=dev, generator=g)
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    del x
    W = torch.randn(D, (2 * I + 1) * D, device=dev, generator=g) / D ** 0.5
    bias, wsc = torch.randn(D, device=dev, generator=g), torch.randn(D, device=dev, generator=g)
    rs = np.random.RandomState(0)
    sel = np.zeros((a.B, a.N), np.float32)
    for b in range(a.B):
        sel[b, rs.choice(a.N, a.seeds, replace=False)] = 1.0
    rows = torch.from_numpy(sel.reshape(-1)).to(dev)
    h32 = torch.empty(M, D, device=dev)
    planes = tuple(torch.zeros(M, kp, dtype=torch.bfloat16, device=dev) for _ in range(2))
    dots = torch.empty(2 * M, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    kw = dict(w_score=wsc, dots=dots, relu=True, k_seg=D, k_seg_pitch=P, k_grouped=True, k_order=True)
    forms = {
        "full": lambda: ops.linear_tc_planes(hi, lo, K, W, bias, out=h32, out_planes=planes, **kw),
        "seed_rows": lambda: ops.linear_tc_planes(hi, lo, K, W, bias, out=h32, out_planes=planes, out_rows=rows, **kw),
        "full_no_planes": lambda: ops.linear_tc_planes(hi, lo, K, W, bias, out=h32, **kw),
    }
    for f in forms.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    ms = {k: [] for k in forms}
    for _ in range(a.reps):
        for k, f in forms.items():
            flush.fill_(1)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            f()
            e.record()
            ms[k].append((s, e))
    torch.cuda.synchronize()
    res = {}
    for k, evs in ms.items():
        t = sorted(s.elapsed_time(e) for s, e in evs)
        res[k] = {"median_ms": t[len(t) // 2], "min_ms": t[0], "max_ms": t[-1]}
    # HBM bytes each form writes (A planes read and W re-streaming are the same in all three)
    wr = {"full": M * D * 4 + 2 * M * P * 2 + 2 * M * 4,
          "seed_rows": int(sel.astype(bool).sum()) * D * 4 + 2 * M * P * 2 + 2 * M * 4,
          "full_no_planes": M * D * 4 + 2 * M * 4}
    for k in res:
        res[k]["written_bytes"] = wr[k]
    print(json.dumps({"shape": {"M": M, "N": D, "K": K, "seed_rows": int(sel.astype(bool).sum())}, "reps": a.reps,
                      "card": card(), "forms": res}))


if __name__ == "__main__":
    main()
