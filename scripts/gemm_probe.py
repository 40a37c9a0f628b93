"""Micro-benchmark of gr_linear_tc_planes: where does the time go? (L2-resident vs HBM-streamed A, K, N, BK, cluster)"""
import sys, os, json, itertools
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from gnn_rag_b200 import ops
dev = "cuda"
def run(M, N, K, bk, cs, outputs="all", reps=10):
    ops.set_option("tc_bk", bk); ops.set_option("tc_cluster", cs)
    Kp = (K + 63) // 64 * 64
    hi = torch.randn(M, Kp, device=dev).to(torch.bfloat16); lo = (torch.randn(M, Kp, device=dev) * 0.01).to(torch.bfloat16)
    W = torch.randn(N, K, device=dev) / K ** 0.5; b = torch.randn(N, device=dev); ws = torch.randn(N, device=dev)
    out = torch.empty(M, N, device=dev) if outputs in ("all", "f32") else None
    oh = torch.empty(M, Kp, dtype=torch.bfloat16, device=dev); ol = torch.empty(M, Kp, dtype=torch.bfloat16, device=dev)
    planes = (oh, ol) if outputs in ("all", "planes") else None
    dots = torch.empty(2 * M, device=dev)
    f = lambda: ops.linear_tc_planes(hi, lo, K, W, b, out=out, out_planes=planes, w_score=ws if outputs != "none" else None,
                                     dots=dots if outputs != "none" else None)
    if outputs == "none":
        out = torch.empty(M, N, device=dev)   # still need one output: tiny trick -> fp32 only
        f = lambda: ops.linear_tc_planes(hi, lo, K, W, b, out=out)
    for _ in range(3): f()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); f(); e.record(); torch.cuda.synchronize(); ts.append(s.elapsed_time(e) * 1e3)
    ts.sort(); us = ts[len(ts) // 2]
    tiles = (M + 127) // 128; nkb = (K + bk - 1) // bk
    nsm, hz = torch.cuda.get_device_properties(0).multi_processor_count, torch.cuda.get_device_properties(0).clock_rate * 1e3
    clk_per_kb = us * 1e-6 * hz / (tiles / nsm * nkb) if tiles >= nsm else us * 1e-6 * hz / nkb
    print("M=%7d N=%3d K=%4d bk=%2d cs=%d out=%-6s  %8.1f us  %6.0f clk/kblock  %.1f TFLOP/s(x3)" % (
        M, N, K, bk, cs, outputs, us, clk_per_kb, 3 * 2 * M * N * K / us / 1e6))
for st in (1, 0):
    ops.set_option("tc_tma_store", st); print("tma_store", st)
    for bk, cs in [(64, 2), (32, 2), (64, 1)]:
        run(128000, 200, 1000, bk, cs, "all")
ops.set_option("tc_tma_store", 1)
run(128000, 200, 1000, 64, 2, "f32")
run(128000, 200, 1000, 64, 2, "planes")
run(16896, 200, 1000, 64, 2, "all")      # 132 tiles: A planes 68 MB total
run(18944, 200, 1000, 32, 2, "all")
run(18944, 200, 1000, 64, 2, "f32")
run(128000, 64, 1000, 64, 2, "all")      # small N: little MMA work, W tiny
run(128000, 200, 256, 64, 2, "all")
run(128000, 200, 4096, 64, 2, "f32")
