"""Timing decomposition of the fused layer kernel at the cfg2 hot shape (CUDA events, L2 flushed between launches):
   python scripts/fused_probe.py            -> full kernel, then with roles switched off (gr_set_option("fused_debug"))"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import bench
from gnn_rag_b200 import batching, ops
from gnn_rag_b200 import synthetic as S

dev = torch.device("cuda")
c = bench.per_gpu_config("cfg2")
B, N, D, I = c["B"], c["N"], c["D"], c["I"]
b = bench.make_cfg_batch(c, 1)
R1 = S.WEBQSP_NUM_RELATION + 1
g = batching.stage_batch(b, dev, R1, False, False).graph
rs = np.random.RandomState(0)
M = B * N
pn = ops.pad_table256(torch.from_numpy(rs.randn(2 * R1, D).astype(np.float32)).to(dev))
pf, pi = pn[:R1], pn[R1:]
ins = torch.from_numpy(rs.randn(B, I, D).astype(np.float32)).to(dev)
h = torch.from_numpy(rs.randn(M, D).astype(np.float32)).to(dev)
Kp = 1088
P = [[torch.zeros(M, Kp, dtype=torch.bfloat16, device=dev) for _ in range(2)] for _ in range(2)]
ops.split_bf16(h, P[0][0], P[0][1])
W = torch.from_numpy((rs.randn(D, 5 * D) / 14).astype(np.float32)).to(dev)
bias = torch.zeros(D, device=dev)
wsc = torch.from_numpy(rs.randn(D).astype(np.float32)).to(dev)
dots = torch.empty(2 * M, device=dev)
prior = torch.softmax(torch.from_numpy(rs.randn(B, N).astype(np.float32)), 1).to(dev)
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
h32 = torch.empty(M, D, device=dev)


def run(out32):
    ops.fused_layer(g, prior, pf, pi, ins, tuple(P[0]), 208, W, bias, out=h32 if out32 else None,
                    out_planes=tuple(P[1]), w_score=wsc, dots=dots, relu=True)


def timeit(out32=False, n=10):
    ts = []
    for _ in range(n + 2):
        flush.fill_(1)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); run(out32); e.record(); torch.cuda.synchronize()
        ts.append(s.elapsed_time(e) * 1e3)
    return np.mean(ts[2:]), np.min(ts[2:])


for name, bits in (("full", 0), ("no aggregation work", 1), ("no edge staging", 2), ("no agg + no staging", 3),
                   ("no epilogue stores", 4), ("nothing but TMA/MMA/epilogue math", 7), ("... and no W loads", 15),
                   ("... and 1 epilogue chunk of 13", 23), ("... neither W nor epilogue", 31)):
    ops.set_option("fused_debug", bits)
    m, mn = timeit()
    print("%-36s %7.1f us (min %.1f)" % (name, m, mn))
ops.set_option("fused_debug", 0)
m, mn = timeit(True)
print("%-36s %7.1f us (min %.1f)" % ("full + fp32 h output", m, mn))


# wait-cycle profile of every role (debug bit 32), averaged over the CTAs
import ctypes
from gnn_rag_b200 import _lib
names = ["MMA loop total", "MMA wait W", "MMA wait aggregated operand", "MMA wait h operand", "MMA wait accumulator",
         "producer wait W slot", "producer wait h slot", "agg warp0 total", "agg wait operand slots", "agg wait descriptor",
         "agg work", "stager wait buffer", "stager work", "epilogue wait accumulator", "epilogue total"]
for label, bits in (("full", 32), ("no agg work", 33), ("no staging", 34), ("no agg, no staging", 35), ("bare (31)", 63)):
    ops.set_option("fused_debug", bits)
    flush.fill_(1); run(False); torch.cuda.synchronize()
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    mhz = torch.cuda.get_device_properties(0).clock_rate / 1e3
    buf = (ctypes.c_ulonglong * (nsm * 16))()
    _lib.check(_lib.load().gr_fused_profile_read(ctypes.cast(buf, ctypes.c_void_p), nsm * 16))
    a = np.array(list(buf), dtype=np.float64).reshape(nsm, 16) / mhz      # -> us at the SM clock
    print("--", label)
    print("   " + " | ".join("%s %.0f" % (n, a[:, i].mean()) for i, n in enumerate(names)))
ops.set_option("fused_debug", 0)
