"""Per-layer time of the four ways to run one dense-prior ReaRev layer, alternated in one process:
     fused          gr_fused_layer (aggregation inside the GEMM kernel), and its mainloop alone: the same launch with
                    the aggregation warps' work switched off (gr_set_option("fused_debug", 1); results are wrong)
     pair k-order   gr_aggregate_dual_abs_ex (GR_AGG_K_ORDER) + gr_linear_tc_planes in grouped K order over the K-order
                    layout (GR_LINEAR_K_ORDER_PLANES): the fused kernel's bits, what ops.dense_layer runs
     pair grouped   gr_aggregate_dual_abs + gr_linear_tc_planes in grouped K order over the segment layout (same bits)
     pair segment   gr_aggregate_dual_abs + gr_linear_tc_planes in segment order (other fp32 rounding)
   at the cfg2 layer shape (B = 64) and at the per-GPU shape of cfg4 (B = 128), with tc_cluster 1 and 2 for the GEMMs,
   and the grouped-order against the segment-order GEMM alone at the d50 width.  CUDA events around every launch, a
   256 MiB write between launches to flush L2, 3 warm-up and 30 timed rounds: median and min..max.
       python scripts/dense_layer_probe.py
   Needs a GPU.  Prints the card, its power limit and max SM clock first: the times belong to that card at that limit."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from gnn_rag_b200 import batching, ops
from gnn_rag_b200 import synthetic as S

if not torch.cuda.is_available():
    sys.exit("dense_layer_probe: no GPU")
dev = torch.device("cuda")
print("card:", subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                               "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip())
PEAK_FLOPS, PEAK_HBM = 989e12, 3.35e12          # H100 SXM data sheet (700 W): dense bf16, HBM3
ROUNDS, WARM = 30, 3
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def timed(fn):
    flush.fill_(1)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record(); fn(); e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e3


def alternate(variants):
    """{name: [us per round]}: every round runs each variant once, in turn."""
    ts = {k: [] for k in variants}
    for r in range(WARM + ROUNDS):
        for k, fn in variants.items():
            t = timed(fn)
            if r >= WARM:
                ts[k].append(t)
    return ts


def report(name, us, flop, hbm_bytes):
    med = float(np.median(us))
    print("  %-34s median %7.1f us (min %7.1f, max %7.1f)   %.0f TFLOP/s = %.2f of the data-sheet 989   "
          "%.2f TB/s = %.2f of the data-sheet 3.35" % (name, med, min(us), max(us), flop / med / 1e6,
                                                       flop / (med * 1e-6) / PEAK_FLOPS, hbm_bytes / med / 1e6,
                                                       hbm_bytes / (med * 1e-6) / PEAK_HBM))


def layer_shape(cfg):
    c = bench.per_gpu_config(cfg)
    B, N, D, I = c["B"], c["N"], c["D"], c["I"]
    P, T, M = 208, 2 * I + 1, B * N
    R1 = S.WEBQSP_NUM_RELATION + 1
    g = batching.stage_batch(bench.make_cfg_batch(c, 1), dev, R1, False, False).graph
    rs = np.random.RandomState(0)
    pn = ops.pad_table256(torch.from_numpy(rs.randn(2 * R1, D).astype(np.float32)).to(dev))
    pf, pi = pn[:R1], pn[R1:]
    ins = torch.from_numpy(rs.randn(B, I, D).astype(np.float32)).to(dev)
    Kp = (T * P + 63) // 64 * 64
    Pl = [[torch.zeros(M, Kp, dtype=torch.bfloat16, device=dev) for _ in range(2)] for _ in range(2)]
    ops.split_bf16(torch.from_numpy(rs.randn(M, D).astype(np.float32)).to(dev), Pl[0][0], Pl[0][1])
    W = torch.from_numpy((rs.randn(D, T * D) / 14).astype(np.float32)).to(dev)
    bias = torch.zeros(D, device=dev)
    wsc = torch.from_numpy(rs.randn(D).astype(np.float32)).to(dev)
    dots = torch.empty(2 * M, device=dev)
    prior = torch.softmax(torch.from_numpy(rs.randn(B, N).astype(np.float32)), 1).to(dev)
    cur, nxt = tuple(Pl[0]), tuple(Pl[1])

    def fused():
        ops.fused_layer(g, prior, pf, pi, ins, cur, P, W, bias, out_planes=nxt, w_score=wsc, dots=dots, relu=True)

    def fused_no_agg():                                        # the mainloop alone: aggregation warps skip their work
        ops.set_option("fused_debug", 1)
        fused()
        ops.set_option("fused_debug", 0)

    def agg(k_order=False):
        ops.aggregate_dual_abs(g, prior, pf, pi, ins, cur, ops.k_order_nb0(P) if k_order else P, P, k_order=k_order)

    def gemm(grouped, k_order=False):
        ops.linear_tc_planes(cur[0], cur[1], T * P, W, bias, out_planes=nxt, w_score=wsc, dots=dots, relu=True,
                             k_seg=D, k_seg_pitch=P, k_grouped=grouped, k_order=k_order)

    flop = 3 * 2.0 * M * P * T * P
    edges = 2 * g.F
    plane_bytes = 2 * 2 * M * P                                # hi + lo of one 208-column segment
    csr = edges * 8 + 2 * M * 4 + M * 4                        # src + rel per in-edge, row pointers, prior
    # fused: CSRs, tables, the h segment in, h planes out.  pair: + the 2I neighbour segments written and read back
    hbm_fused = csr + 2 * R1 * 1024 + 2 * plane_bytes
    hbm_pair = hbm_fused + 2 * (T - 1) * plane_bytes
    print("%s layer shape: M = %d rows, D = %d, I = %d, %d in-edges (both directions)" % (cfg, M, D, I, edges))
    for cs in (1, 2):
        ops.set_option("tc_cluster", cs)
        ts = alternate({"fused": fused, "fused no agg": fused_no_agg, "agg": agg, "agg k-order": lambda: agg(True),
                        "gemm grouped": lambda: gemm(True), "gemm segment": lambda: gemm(False),
                        "gemm k-order": lambda: gemm(True, True)})
        print(" tc_cluster = %d (the GEMMs; the fused kernel always pairs CTAs)" % cs)
        report("fused (gr_fused_layer)", ts["fused"], flop, hbm_fused)
        report("  fused, aggregation off (fused_debug 1)", ts["fused no agg"], flop, hbm_fused)
        report("pair, K-order layout", [a + b for a, b in zip(ts["agg k-order"], ts["gemm k-order"])], flop, hbm_pair)
        report("pair, grouped K order", [a + b for a, b in zip(ts["agg"], ts["gemm grouped"])], flop, hbm_pair)
        report("pair, segment K order", [a + b for a, b in zip(ts["agg"], ts["gemm segment"])], flop, hbm_pair)
        agg_bytes = csr + 2 * R1 * 1024 + (T - 1) * plane_bytes
        report("  gr_aggregate_dual_abs alone", ts["agg"], 0.0, agg_bytes)
        report("  gr_aggregate_dual_abs K-order", ts["agg k-order"], 0.0, agg_bytes)
        report("  GEMM grouped alone", ts["gemm grouped"], flop, (T + 1) * plane_bytes)
        report("  GEMM segment alone", ts["gemm segment"], flop, (T + 1) * plane_bytes)
        report("  GEMM K-order alone", ts["gemm k-order"], flop, (T + 1) * plane_bytes)
    ops.set_option("tc_cluster", 1)


def gemm_shape(M, D, I):
    """The two K orders of the GEMM alone at a width the aggregation kernel does not specialise (d50)."""
    P, T = (D + 15) // 16 * 16, 2 * I + 1
    rs = np.random.RandomState(1)
    Kp = (T * P + 63) // 64 * 64
    A = np.zeros((M, T, P), np.float32)
    A[:, :, :D] = rs.randn(M, T, D)
    hi, lo = (torch.zeros(M, Kp, dtype=torch.bfloat16, device=dev) for _ in range(2))
    ops.split_bf16(torch.from_numpy(A.reshape(M, T * P)).to(dev), hi, lo)
    nxt = tuple(torch.zeros(M, Kp, dtype=torch.bfloat16, device=dev) for _ in range(2))
    W = torch.from_numpy((rs.randn(D, T * D) / 14).astype(np.float32)).to(dev)
    bias = torch.zeros(D, device=dev)

    def gemm(grouped):
        ops.linear_tc_planes(hi, lo, T * P, W, bias, out_planes=nxt, relu=True, k_seg=D, k_seg_pitch=P,
                             k_grouped=grouped)

    print("GEMM alone: M = %d, D = %d, I = %d (pitch %d)" % (M, D, I, P))
    ts = alternate({"grouped": lambda: gemm(True), "segment": lambda: gemm(False)})
    for k in ts:
        report("GEMM %s" % k, ts[k], 3 * 2.0 * M * P * T * P, (T + 1) * 2 * 2 * M * P)


layer_shape("cfg2")
layer_shape("cfg4")
c = bench.per_gpu_config("d50")
gemm_shape(c["B"] * c["N"], c["D"], c["I"])
