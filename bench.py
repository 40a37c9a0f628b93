#!/usr/bin/env python
"""bench.py -- questions/sec of the GNN retrieval hot path (ReaRev forward + score + candidate ranking) on
WebQSP-shape synthetic subgraphs, with the aggregation kernel's achieved HBM bandwidth (roofline) and the
CPU oracle port timed beside it.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--config cfg2] [--impl ours|reference] [--dump-outputs DIR]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...

One "step" = one pass of the hot path over one batch: CSR batching of the fact list -> TypeLayer ->
num_iter x num_gnn GNN layers (aggregation + e2e linear + score/softmax) -> instruction updates -> loss ->
candidate ranking.  `value` times steps whose inputs (raw fact arrays etc.) are already in HBM, with CUDA
events on the launching stream (L2 flushed between steps); `e2e` times model.forward(host batch) + retrieve:
pinned-host -> device copies, CSR batching, forward, ranking and the device -> host read of the retrieved
candidate lists, by wall clock between synchronizes.  Multi-GPU: one process per GPU, every rank runs its
own B questions (weak scaling), no communication during the forward, one NCCL all-gather of the answer
scores at the end of each step; time = max over ranks.

--dump-outputs DIR writes what the timed path returned in its last timed step (pred_dist, loss, pred and the ranked
candidate lists) as DIR/<name>.npy in float32 / float64.  Inputs and weights are seeded, so two builds run with the
same arguments can be compared output for output.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from gnn_rag_b200 import synthetic as S  # noqa: E402

METRIC = "questions/sec (GNN forward+score) on WebQSP-shape subgraphs; agg-kernel HBM GB/s"
UNIT = "questions/s"
WORKLOADS = {
    "cfg1": "single WebQSP question, ~2k-node/~6k-edge subgraph, 3-hop ReaRev fp32",
    "cfg2": "batch=64 WebQSP-shape synthetic subgraphs (~2k nodes, 200-dim feat, 3 hops) on 1xH100",
    "cfg3": "batch=256 CWQ-shape synthetic subgraphs (~10k nodes, ~40k edges, 4 hops)",
    "cfg4": "batch=1024 WebQSP-shape subgraphs sharded across 8xH100 = 128 questions per GPU (weak scaling)",
    "cfg5": "stress: 100k-node / 1M-edge synthetic subgraph, 400-dim feat, 3 hops",
    "d50": "batch=64 WebQSP-shape subgraphs at the PUBLISHED model shape (gnn/README.md:19: entity_dim 50, num_iter 3, "
           "num_ins 2, num_gnn 3)",
}


def per_gpu_config(name):
    """Per-GPU shape of a named workload: cfg4 is the 1024-question batch split over 8 GPUs, i.e. 128 per GPU
    whatever --gpus is (weak scaling); every other config is per GPU as written."""
    c = dict(S.CONFIGS[name])
    if name == "cfg4":
        c["B"] = c["B"] // 8
    if _BATCH_OVERRIDE:
        c["B"] = _BATCH_OVERRIDE
    return c


_BATCH_OVERRIDE = None


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--config", default="cfg2", choices=sorted(WORKLOADS))
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--batch", type=int, default=None, help="override the questions per GPU of the config")
    ap.add_argument("--cpu-sample", type=int, default=None,
                    help="questions per CPU step (default: 8 for the cpu_baseline leg, the whole batch -- at most 64 -- "
                         "for --impl reference)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--agg-tma", type=int, default=None)
    ap.add_argument("--agg-abs", type=int, default=None, help="0: generic aggregation kernel instead of the |v|-accumulating one")
    ap.add_argument("--agg-abs-ws", type=int, default=None, help="0: one CTA per tile instead of the persistent kernel")
    ap.add_argument("--tc-bk", type=int, default=None)
    ap.add_argument("--tc-cluster", type=int, default=None)
    ap.add_argument("--act-bf16", type=int, default=None,
                    help="1: bf16 activation storage (hi plane only, one-product GEMM); default: on for cfg3 "
                         "(BASELINE configs[2] names bf16), off elsewhere")
    ap.add_argument("--fused", type=int, default=1,
                    help="0: dense-prior layers as aggregation kernel + GEMM instead of the fused layer kernel")
    ap.add_argument("--cuda-graph", type=int, default=1,
                    help="1: run the step through gnn_rag_b200.GraphedStep (CUDA-graph replay over static buffers)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the outputs of the last timed step to DIR/<name>.npy (float32 / float64)")
    return ap.parse_args()


DUMP_BUDGET = 64 << 20     # bytes of all dumped arrays together


def dump_outputs(path, outs):
    """Write {name: tensor} as float32 (floating outputs) / float64 (integer outputs: exact below 2^53) .npy files.
    An array whose share of the budget is too small is reduced to a fixed, seeded sample of its rows (the row indices
    go to <name>_rows.npy)."""
    os.makedirs(path, exist_ok=True)
    share = DUMP_BUDGET // max(len(outs), 1) // 2       # room for the row-index files too
    for name, t in outs.items():
        a = t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
        a = a.astype(np.float32 if a.dtype.kind == "f" else np.float64)
        if a.nbytes > share and a.ndim >= 1:
            keep = max(1, share // max(a.nbytes // a.shape[0], 1))
            rows = np.sort(np.random.RandomState(0).choice(a.shape[0], keep, replace=False))
            np.save(os.path.join(path, name + "_rows.npy"), rows.astype(np.float64))
            a = a[rows]
        np.save(os.path.join(path, name + ".npy"), a)


def model_args_for(c, use_cuda):
    return S.model_args("ReaRev", entity_dim=c["D"], num_iter=c["T"], num_ins=c["I"], num_gnn=c["K"],
                        use_cuda=use_cuda)


def make_cfg_batch(c, seed, B=None):
    B = c["B"] if B is None else B
    return S.make_batch(seed, B=B, N=c["N"], E=c["E"], with_weights=False)


def config_dict(name, c, extra=None, world=1):
    wl = "%s: %s" % (name, WORKLOADS[name])
    if world > 1 or name == "cfg4":
        wl += " -- weak scaling at %d questions per GPU" % c["B"]
    d = {"workload": wl, "questions_per_gpu": c["B"], "nodes": c["N"],
         "kg_edges": c["E"], "facts_incl_self_loops": c["E"] + c["N"], "feat_dim": c["D"],
         "num_iter": c["T"], "num_gnn": c["K"], "num_ins": c["I"],
         "relations": S.WEBQSP_NUM_RELATION, "seeds": {"data": 1, "weights": 0}}
    if extra:
        d.update(extra)
    return d


# ---------------------------------------------------------------------------------------------------
# CPU oracle port (cpu_baseline / --impl reference)
# ---------------------------------------------------------------------------------------------------
def cpu_oracle_run(c, sd_cpu, nq, steps, warmup, with_loader=True):
    """Time the oracle port (oracle/kgqa_oracle.py: the reference's op sequence on torch-CPU) on `nq`
    questions of the workload with all host threads.  Returns (questions/s, ms/step, cores)."""
    from oracle import kgqa_oracle as O
    args = model_args_for(c, False)
    # pick the fastest thread count for the reference's op mix (many small ops: more threads is not
    # always faster on big hosts) with a 2-question probe, so the baseline is the CPU path at its best
    ncpu = os.cpu_count() or 1
    probe = make_cfg_batch(c, 2, B=min(2, nq))
    best = (None, float("inf"))
    for th in sorted({ncpu, min(ncpu, 32), min(ncpu, 16), min(ncpu, 8)}, reverse=True):
        torch.set_num_threads(th)
        with torch.no_grad():
            O.forward(sd_cpu, args, S.WEBQSP_NUM_ENTITY, S.WEBQSP_NUM_WORD, probe)
            t0 = time.perf_counter()
            O.forward(sd_cpu, args, S.WEBQSP_NUM_ENTITY, S.WEBQSP_NUM_WORD, probe)
            dt = time.perf_counter() - t0
        if dt < best[1]:
            best = (th, dt)
    cores = best[0]
    torch.set_num_threads(cores)
    batch = make_cfg_batch(c, 1, B=nq)
    times, loader_s = [], None
    with torch.no_grad():
        for i in range(warmup + steps):
            t0 = time.perf_counter()
            _, _, dist = O.forward(sd_cpu, args, S.WEBQSP_NUM_ENTITY, S.WEBQSP_NUM_WORD, batch)
            O.rank_candidates(batch[0], batch[1], dist.numpy(), S.WEBQSP_NUM_ENTITY, args["eps"])
            dt = time.perf_counter() - t0
            if i >= warmup:
                times.append(dt)
    if with_loader:
        # the reference's get_batch cost for the same questions (oracle/loader_oracle.py: _build_fact_mat in the
        # reference's own form), SURVEY 8d (ii): forward + get_batch + ranking
        from oracle import loader_oracle
        st = loader_oracle.state_from_batch(batch, S.WEBQSP_NUM_RELATION)
        np.random.seed(0)
        t0 = time.perf_counter()
        loader_oracle.build_fact_mat(st, list(range(nq)), 0.0)
        loader_s = time.perf_counter() - t0
    tot = sum(times)
    qps = nq * len(times) / tot
    qps_with_loader = nq / (tot / len(times) + loader_s) if loader_s is not None else None
    return qps, 1e3 * tot / len(times), cores, qps_with_loader


def init_state_dict_cpu(c):
    """Random-init weights of the ReaRev architecture (torch.manual_seed(0)), CPU fp32."""
    import gnn_rag_b200 as G
    torch.manual_seed(0)
    m = G.ReaRev(model_args_for(c, False), S.WEBQSP_NUM_ENTITY, S.WEBQSP_NUM_RELATION, S.WEBQSP_NUM_WORD)
    return {k: v.detach().clone() for k, v in m.state_dict().items()}


def run_reference(a):
    """The reference's own CPU implementation of the path (the oracle port oracle/kgqa_oracle.py: the reference is pure
    Python, so there is no compiled reference binary), all host threads, on this arm's config.
    One step = forward + ranking of `sample` questions of the workload (the whole batch for cfg1 / cfg2 / cfg4)."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    c = per_gpu_config(a.config)
    sd = init_state_dict_cpu(c)
    default_nq = {"cfg3": 2, "cfg5": 1}.get(a.config, min(c["B"], 64))
    nq = min(a.cpu_sample if a.cpu_sample else default_nq, c["B"])
    heavy = a.config in ("cfg3", "cfg5")
    steps = max(1, min(a.steps, 1 if heavy else 2))
    warmup = 0 if heavy else max(1, min(a.warmup, 1))
    qps, ms, cores, qps_l = cpu_oracle_run(c, sd, nq, steps, warmup)
    sample = "%d of %d questions per step, %d timed step(s), %d warm-up" % (nq, c["B"], steps, warmup)
    line = {"impl": "reference", "metric": METRIC, "value": qps, "unit": UNIT, "n_gpus": a.gpus,
            "steps": steps, "warmup": warmup, "ms_per_step": ms, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": config_dict(a.config, c, {"sample": sample, "questions_per_step": nq}),
            "cpu_baseline": {"value": qps, "unit": UNIT, "cores": cores, "kind": "port", "sample": sample,
                             "with_get_batch": qps_l},
            "e2e": {"value": qps, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0}
    print(json.dumps(line))


# ---------------------------------------------------------------------------------------------------
# clocks sampler
# ---------------------------------------------------------------------------------------------------
class ClockSampler:
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.Q, "--format=csv,noheader,nounits",
                 "-lms", "25"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:  # noqa: BLE001
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([x.strip() for x in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        sm, mx, reasons = [], None, set()
        for r in self.rows:
            try:
                sm.append(float(r[1]))
                mx = float(r[2])
                for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"),
                                   r[5:9]):
                    if v.lower().startswith("active"):
                        reasons.add(name)
            except Exception:  # noqa: BLE001
                pass
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": mx,
                "reasons": sorted(reasons), "samples": len(sm)}


# ---------------------------------------------------------------------------------------------------
# our arm
# ---------------------------------------------------------------------------------------------------
def agg_algorithmic_bytes(B, N, F, D, I, R1, out_elem_bytes=4):
    """Minimal HBM bytes of ONE fused aggregation launch (both directions, I instructions), fp32/int32:
    two CSRs (src+rel per edge, row pointers), prior, two relation tables, instructions, 2*I output rows
    (4 bytes per element as split-bf16 hi+lo, 2 with bf16 activation storage).
    (= 2*I units of SURVEY.md 8d minus the reads the fused launch shares.)"""
    Nt = B * N
    return (2 * F * 8 + 2 * (Nt + 1) * 4 + Nt * 4 + 2 * R1 * D * 4 + B * I * D * 4
            + 2 * I * Nt * D * out_elem_bytes)


def run_ours(a):
    import torch.distributed as dist

    import gnn_rag_b200 as G
    from gnn_rag_b200 import batching, evaluate, ops, parallel

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py --impl ours needs a CUDA device (there is no CPU fallback)")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    if a.agg_tma is not None:
        ops.set_option("agg_tma", a.agg_tma)
    if a.agg_abs is not None:
        ops.AGG_ABS = bool(a.agg_abs)
    if a.agg_abs_ws is not None:
        ops.set_option("agg_abs_ws", a.agg_abs_ws)
    if a.tc_bk is not None:
        ops.set_option("tc_bk", a.tc_bk)
    if a.tc_cluster is not None:
        ops.set_option("tc_cluster", a.tc_cluster)
    act_bf16 = bool(a.act_bf16) if a.act_bf16 is not None else (a.config == "cfg3")
    ops.ACT_BF16 = act_bf16
    ops.FUSED_LAYER = bool(a.fused)
    c = per_gpu_config(a.config)
    B, N, D, I = c["B"], c["N"], c["D"], c["I"]
    args = model_args_for(c, True)
    torch.manual_seed(0)
    model = G.ReaRev(dict(args), S.WEBQSP_NUM_ENTITY, S.WEBQSP_NUM_RELATION, S.WEBQSP_NUM_WORD).eval()
    R1 = S.WEBQSP_NUM_RELATION + 1
    host_batch = make_cfg_batch(c, 1 + rank)
    F = len(host_batch[2][0])
    pinned = batching.pin_batch(host_batch)
    # device-resident raw inputs for the `value` leg (fact arrays stay int64 exactly as the loader emits)
    dev_batch = tuple(
        (tuple(x.to(dev) if isinstance(x, torch.Tensor) else x for x in t) if isinstance(t, tuple)
         else (t.to(dev) if isinstance(t, torch.Tensor) else t)) for t in pinned)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2
    eps = args["eps"]

    gs = G.GraphedStep(model, S.WEBQSP_NUM_ENTITY) if a.cuda_graph else None

    def step_eager(batch):
        loss, pred, pred_dist, _ = model(batch)
        cand = ops.rank_candidates(pred_dist, model.last_batch.local_entity,
                                   model.last_batch.query_entities, S.WEBQSP_NUM_ENTITY, eps)
        if world > 1:
            parallel.all_gather_scores(pred_dist, B * world)
        return (loss, pred, pred_dist) + tuple(cand)

    def step(batch):
        """-> (loss, pred, pred_dist, cand_idx, cand_count, cand_total): what a caller of the step receives"""
        if gs is None:
            return step_eager(batch)
        out = gs(batch)                     # copies the inputs into the static buffers, replays the graph
        if world > 1:
            parallel.all_gather_scores(out.pred_dist, B * world)
        return out.loss, out.pred, out.pred_dist, out.cand_idx, out.cand_count, out.cand_total

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    # ---- warm-up -------------------------------------------------------------------------------
    for _ in range(max(a.warmup, 3)):
        step(dev_batch)
    barrier()
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    # ---- eager replica of the timed region: per-launch CUDA events around every aggregation launch (the
    # live roofline measurement) and the launch count; with --cuda-graph the same kernels are replayed from the
    # graph in the timed region below, where per-launch events cannot be recorded
    def replica(nsteps):
        ops.STATS.reset()
        ops.STATS.time_agg = True
        ops.STATS.time_ops = True
        evs_ = []
        for _ in range(nsteps):
            flush.fill_(1)
            s0, e0 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s0.record()
            step_eager(dev_batch)
            e0.record()
            evs_.append((s0, e0))
        barrier()
        ops.STATS.time_agg = False
        ops.STATS.time_ops = False
        agg_ = [(s.elapsed_time(e), tag) for s, e, tag in ops.STATS.agg_events]
        # per-kernel-class device time of the eager replica (events around every wrapper, on the launching stream)
        op_ms_, gemm_, fused_ = {}, {}, []
        for s_, e_, cls, info in ops.STATS.op_events:
            ms = s_.elapsed_time(e_)
            op_ms_[cls] = op_ms_.get(cls, 0.0) + ms
            if cls == "gemm_tc":
                gemm_.setdefault(info, []).append(ms)
            if cls == "fused_layer":
                fused_.append(ms)
        return (ops.STATS.launches, agg_, op_ms_, gemm_, fused_,
                sum(s_.elapsed_time(e_) for s_, e_ in evs_), nsteps)

    launches, agg, op_ms, gemm, fused_ms, rep_ms, agg_steps = replica(a.steps)
    if fused_ms:
        # the unfused pair stays the roofline unit of the aggregation kernel and of the K = (2I+1)D GEMM: a second
        # replica with the fused layer kernel switched off supplies `roofline` / `roofline_gemm`
        ops.FUSED_LAYER = False
        _l, agg, _o, gemm, _f, _r, agg_steps = replica(min(a.steps, 10))
        ops.FUSED_LAYER = True
    for _ in range(3):
        step(dev_batch)
    barrier()
    # ---- timed region: K steps, device-resident inputs, CUDA events, L2 flushed between steps -------
    evs = []
    barrier()
    wall0 = time.perf_counter()
    last = None
    for _ in range(a.steps):
        flush.fill_(1)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        last = step(dev_batch)
        e.record()
        evs.append((s, e))
    barrier()
    wall = time.perf_counter() - wall0
    if a.dump_outputs and rank == 0:
        # before the e2e legs below: with --cuda-graph the outputs live in the graph's static buffers
        loss, pred, pred_dist, cand_idx, cand_count, cand_total = last
        ranked = cand_idx.long()
        valid = torch.arange(ranked.shape[1], device=dev)[None, :] < cand_count.view(-1, 1).long()
        ranked = torch.where(valid, ranked, torch.full_like(ranked, -1))     # slots past a question's count: -1
        dump_outputs(a.dump_outputs, {"pred_dist": pred_dist, "loss": loss, "pred": pred, "cand_idx": ranked,
                                      "cand_count": cand_count, "cand_total": cand_total})
    dev_ms = sum(s.elapsed_time(e) for s, e in evs)
    # clocks are sampled over the device-timed region only: nvidia-smi polling takes a driver lock and
    # perturbs the wall-clock e2e loop below (measured: 5.5 ms/step alone vs 8-19 ms with the sampler on)
    clocks = sampler.stop() if rank == 0 else None
    # ---- e2e: host (pinned) batch in, retrieved candidate lists out -------------------------------
    def e2e_step():
        if gs is None:
            _loss, _pred, pred_dist, _ = model(pinned)
            retrieved, nb = evaluate.retrieve(pred_dist, model.last_batch, S.WEBQSP_NUM_ENTITY, eps)
        else:
            out = gs(pinned)
            pred_dist = out.pred_dist
            retrieved, nb = gs.retrieve(out)
        if world > 1:
            parallel.all_gather_scores(pred_dist, B * world)
        return nb

    for _ in range(2):      # warm the host-batch path (allocator, pinned staging)
        e2e_step()
    barrier()
    h2d = d2h = 0
    if gs is not None:
        # serving loop: two batches in flight -- submit(i) enqueues the H2D of batch i's inputs (pinned host
        # memory -> copy stream), the graph and the D2H of its results; collect(i-1) reads batch i-1's candidate
        # lists on the host.  Every step's H2D and D2H happen inside the timed region; pipeline fill and drain
        # are inside it too.
        for _ in range(2):
            gs.collect(gs.submit(pinned))
        barrier()
        t0 = time.perf_counter()
        prev = None
        for _ in range(a.steps):
            tk = gs.submit(pinned)
            if world > 1:
                parallel.all_gather_scores(tk.ent.outs[3], B * world)
            if prev is not None:
                _ret, d2h, _l, _p = gs.collect(prev)
            prev = tk
        _ret, d2h, _l, _p = gs.collect(prev)
        h2d = model.last_batch.h2d_bytes
        barrier()
        e2e_s = time.perf_counter() - t0
        e2e_mode = "pipelined submit/collect, 2 batches in flight"
    else:
        t0 = time.perf_counter()
        for _ in range(a.steps):
            nb = e2e_step()
            h2d, d2h = model.last_batch.h2d_bytes, nb
        barrier()
        e2e_s = time.perf_counter() - t0
        e2e_mode = "synchronous"
    # ---- e2e from what the loader returns: pageable numpy tuples (int64 facts, float64 distributions), a different
    # batch every step, conversion + pinning-free H2D inside the timed region --------------------------------
    e2e_pg_s, h2d_pg = float("nan"), 0
    if gs is not None:
        pool = [make_cfg_batch(c, 100 + rank * 16 + i) for i in range(4)]
        for hb in pool[:2]:
            gs.collect(gs.submit(hb))
        barrier()
        t0 = time.perf_counter()
        prev = None
        for i in range(a.steps):
            tk = gs.submit(pool[i % len(pool)])
            if world > 1:
                parallel.all_gather_scores(tk.ent.outs[3], B * world)
            if prev is not None:
                gs.collect(prev)
            prev = tk
        gs.collect(prev)
        h2d_pg = model.last_batch.h2d_bytes
        barrier()
        e2e_pg_s = time.perf_counter() - t0
    # ---- max over ranks ------------------------------------------------------------------------
    t = torch.tensor([dev_ms, e2e_s * 1e3, e2e_pg_s * 1e3], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    dev_ms, e2e_ms, e2e_pg_ms = t.tolist()
    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    value = world * B * a.steps / (dev_ms / 1e3)
    e2e_value = world * B * a.steps / (e2e_ms / 1e3)
    # ---- roofline of the dominant kernel (aggregation) ------------------------------------------------
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:  # noqa: BLE001
        pass
    peak = float(peaks.get("hbm_gbs", 3350.0))
    peak_src = ("MEASURED_PEAKS.json hbm_gbs (of measured)" if "hbm_gbs" in peaks
                else "3350 GB/s (H100 SXM data sheet, not reached)")
    per_step = len(agg) // max(agg_steps, 1)
    # layer 0 of every iteration sees the one-hot seed prior.  With the sparse-prior fast path (default) that layer
    # never reaches the aggregation kernel (K = D GEMM + frontier fix-up), so every timed launch is a dense-prior
    # launch; without it those launches are pure output writes and are reported separately.
    K = c["K"]
    if ops.SPARSE_PRIOR_FASTPATH and ops.TC_LINEAR:
        dense, seedl = [ms for ms, _ in agg], []
    else:
        dense = [ms for i, (ms, _) in enumerate(agg) if (i % per_step) % K != 0] if per_step else []
        seedl = [ms for i, (ms, _) in enumerate(agg) if (i % per_step) % K == 0] if per_step else []
    abytes = agg_algorithmic_bytes(B, N, F, D, I, R1, 2 if act_bf16 else 4)
    traffic = None     # measured DRAM bytes of the dense-prior launch: not measured
    dense_ms = float(np.mean(dense)) if dense else float("nan")
    achieved = abytes / (dense_ms * 1e-3) / 1e9
    agg_name = ("agg_abs_wsg_kernel (gr_aggregate_dual_abs)" if ops.AGG_ABS and D == 200 and ops.TC_LINEAR
                else "agg_kernel (gr_aggregate_dual)")
    roofline = {"bound": "hbm", "kernel": agg_name, "achieved": achieved, "peak": peak,
                "unit": "GB/s", "frac": achieved / peak, "traffic": traffic, "peak_source": peak_src,
                "algorithmic_bytes_per_launch": abytes, "avg_launch_ms": dense_ms,
                "launches_per_step": per_step,
                "measured_in": "eager replica of the timed region (same process, same inputs, L2 flushed)",
                "seed_prior_launch_ms": float(np.mean(seedl)) if seedl else None,
                "agg_share_of_step": ((sum(ms for ms, _ in agg) / max(agg_steps, 1)) / (dev_ms / a.steps))
                if (dev_ms and not fused_ms) else None}
    # ---- tensor-core GEMM roofline (the largest e2e GEMM of the step) and the share table ---------------------
    roofline_gemm = None
    if gemm:
        (gM, gN, gK), ts = max(gemm.items(), key=lambda kv: kv[0][0] * kv[0][2] * len(kv[1]))
        g_ms = float(np.mean(ts))
        nprod = 1 if act_bf16 else 3                         # bf16 products per output (3 = fp32-class split)
        flops = nprod * 2.0 * gM * gN * gK
        tf_peak = float(peaks.get("bf16_tflops", 989.0))
        roofline_gemm = {"bound": "tensor", "kernel": "linear_tc_kernel (gr_linear_tc_planes, %d bf16 product%s)" % (
                             nprod, "s" if nprod > 1 else ""),
                         "shape": {"M": gM, "N": gN, "K": gK}, "achieved": flops / (g_ms * 1e-3) / 1e12,
                         "peak": tf_peak, "unit": "TFLOP/s", "frac": flops / (g_ms * 1e-3) / 1e12 / tf_peak,
                         "peak_source": "MEASURED_PEAKS.json bf16_tflops (burst, of measured)" if "bf16_tflops" in peaks
                         else "989 TFLOP/s (H100 SXM data sheet, dense bf16, not reached)",
                         "avg_launch_ms": g_ms, "launches_per_step": len(ts) // max(agg_steps, 1),
                         "fp32_equivalent_tflops": 2.0 * gM * gN * gK / (g_ms * 1e-3) / 1e12}
    roofline_fused = None
    if fused_ms:
        f_ms = float(np.mean(fused_ms))
        Kd = (2 * I + 1) * D
        flops = 3 * 2.0 * B * N * D * Kd
        tf_peak = float(peaks.get("bf16_tflops", 989.0))
        # what the fused kernel has to move: both CSRs + prior, the relation tables, h planes in, h planes out
        fbytes = 2 * F * 8 + 2 * (B * N + 1) * 4 + B * N * 4 + 2 * R1 * D * 4 + B * I * D * 4 + 2 * B * N * D * 4
        roofline_fused = {"bound": "tensor", "kernel": "fused_layer_kernel (gr_fused_layer: aggregation -> wgmma GEMM)",
                          "achieved": flops / (f_ms * 1e-3) / 1e12, "peak": tf_peak, "unit": "TFLOP/s",
                          "frac": flops / (f_ms * 1e-3) / 1e12 / tf_peak, "avg_launch_ms": f_ms,
                          "launches_per_step": len(fused_ms) // max(a.steps, 1),
                          "replaces_ms": (dense_ms + roofline_gemm["avg_launch_ms"]) if roofline_gemm else None,
                          "algorithmic_hbm_bytes_per_launch": int(fbytes),
                          "hbm_gbs": fbytes / (f_ms * 1e-3) / 1e9}
        roofline["measured_in"] = ("second eager replica with the fused layer kernel switched off (the timed step runs "
                                   "the fused kernel; the unfused pair is the roofline unit of the aggregation)")
    shares = {k: v / rep_ms for k, v in sorted(op_ms.items(), key=lambda kv: -kv[1])} if rep_ms else {}
    shares["_note"] = ("device time per kernel class / eager step time, from CUDA events around every wrapper in the "
                       "eager replica (the question side runs on a second stream and overlaps: shares can sum past 1)")
    line = {"metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": a.steps,
            "warmup": max(a.warmup, 3), "ms_per_step": dev_ms / a.steps, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None,
            "dtype": "bf16 activation storage, f32 tables / accumulate / scores" if act_bf16 else "f32",
            "data": "synthetic",
            "config": config_dict(a.config, c, world=world, extra={
                "global_questions": world * B, "l2": "256 MiB flush write between timed steps",
                "timing": "CUDA events per step on the launch stream, max over ranks",
                "cuda_graph": bool(a.cuda_graph), "fused_layer_kernel": bool(fused_ms),
                "wall_s_timed_region_incl_flush": wall}),
            "e2e": {"value": e2e_value, "unit": UNIT, "h2d_bytes_per_step": int(h2d),
                    "d2h_bytes_per_step": int(d2h), "ms_per_step": e2e_ms / a.steps, "mode": e2e_mode,
                    "from_pageable_numpy": {
                        "value": world * B * a.steps / (e2e_pg_ms / 1e3) if e2e_pg_ms == e2e_pg_ms else None,
                        "ms_per_step": e2e_pg_ms / a.steps if e2e_pg_ms == e2e_pg_ms else None,
                        "h2d_bytes_per_step": int(h2d_pg),
                        "what": "a different get_batch-layout tuple every step (pageable numpy, int64 facts, float64 "
                                "distributions): host casts + H2D + graph + D2H inside the timed region"}},
            "gpu_launches": int(launches), "gpu_launches_per_step": int(launches // max(a.steps, 1)), "clocks": clocks,
            "roofline": roofline,
            "roofline_gemm": roofline_gemm, "roofline_fused": roofline_fused, "shares": shares}
    if not a.no_cpu_baseline and world == 1:
        sd_cpu = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
        nq = min(a.cpu_sample if a.cpu_sample else {"cfg3": 1, "cfg5": 1}.get(a.config, 8), B)
        qps, ms, cores, qps_l = cpu_oracle_run(c, sd_cpu, nq, 3 if a.config not in ("cfg3", "cfg5") else 1, 1
                                               if a.config not in ("cfg3", "cfg5") else 0)
        line["cpu_baseline"] = {"value": qps, "unit": UNIT, "cores": cores, "kind": "port",
                                "with_get_batch": qps_l,
                                "sample": "%d of %d questions per forward, timed forwards + ranking (oracle port of "
                                          "the reference op sequence, torch-CPU, all host threads); with_get_batch "
                                          "adds the reference-form batch assembly" % (nq, B)}
    print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


def main():
    global _BATCH_OVERRIDE
    a = parse()
    _BATCH_OVERRIDE = a.batch
    if a.impl == "reference":
        run_reference(a)
    else:
        run_ours(a)


if __name__ == "__main__":
    main()
