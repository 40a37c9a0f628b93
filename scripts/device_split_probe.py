"""End-to-end serving rate with the batch assembled on the host vs on the device (loader.DeviceSplit).

An evaluator-shaped loop over a synthetic WebQSP-shape split (N = 2000 nodes, E = 6000 stored facts per question, 4 to
N entities each with their self-loops, WebQSP's relation and entity vocabularies): for every batch ``get_batch(it, B,
0.0, test=True)`` and ``GraphedStep.submit``, collecting the previous ticket (two in flight).

  host    the loader's get_batch with loader.install(shuffle=False, weights="none", index_dtype=np.int32)
          (GraftNet: plus loader.install_graft), then submit of the numpy tuple
  device  DeviceSplit(loader, weights="none").get_batch, then submit of the CUDA tuple

A pass runs the whole split; the questions/s of a mode is the median over ``--runs`` passes, host and device
alternating, after one warm-up pass of each (graph capture).  Also printed: the split's build time (upload) and
resident bytes, and the GPU's name and power limit, read in the same run.  One JSON line per configuration.

    python scripts/device_split_probe.py [--questions 640] [--runs 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import gnn_rag_b200 as G                                     # noqa: E402
from gnn_rag_b200 import graphed, loader, synthetic as S    # noqa: E402

NE, NR, NW = S.WEBQSP_NUM_ENTITY, S.WEBQSP_NUM_RELATION, S.WEBQSP_NUM_WORD


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), (s.strip() for s in out.split(","))))
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(), "error": str(e)}


class SyntheticSplit:
    """The fields SingleDataLoader.get_batch / GraftSingleDataLoader.get_batch read, for num_q synthetic questions."""
    q_type = "seq"
    data_eff = False
    use_self_loop = True

    def __init__(self, num_q, N=2000, E=6000, Q=12, seed=0, graft=False):
        rs = np.random.RandomState(seed)
        self.num_data, self.max_local_entity = num_q, N
        self.num_kb_relation = NR
        self.batches = np.arange(num_q)
        self.kb_adj_mats, self.global2local_entity_maps = [], []
        self.candidate_entities = np.full((num_q, N), NE, dtype=np.int64)
        self.query_entities = np.zeros((num_q, N))
        self.seed_distribution = np.zeros((num_q, N))
        self.answer_dists = np.zeros((num_q, N))
        self.query_texts = np.full((num_q, Q), NW, dtype=np.int64)
        self.answer_lists = np.empty(num_q, dtype=object)
        for q in range(num_q):
            n = int(rs.randint(N // 2, N + 1))
            self.kb_adj_mats.append((rs.randint(0, n, E), rs.randint(0, NR - 1, E), rs.randint(0, n, E)))
            self.global2local_entity_maps.append(range(n))
            self.candidate_entities[q, :n] = rs.randint(0, NE, n)
            self.query_entities[q, 0] = self.seed_distribution[q, 0] = 1.0
            self.answer_dists[q, 1:3] = 1.0
            self.answer_lists[q] = self.candidate_entities[q, 1:3].tolist()
            self.query_texts[q, :Q // 2] = rs.randint(0, NW, Q // 2)
        if graft:
            self.max_facts = 2 * E + N
            self.kb_fact_rels = np.full((num_q, self.max_facts), NR, dtype=np.int64)
            for q in range(num_q):
                self.kb_fact_rels[q, :E] = self.kb_adj_mats[q][1]
            self.create_kb_adj_mats_facts = self._graft_facts

    def _build_fact_mat(self, sample_ids, fact_dropout):
        raise NotImplementedError("replaced by loader.install")

    def _build_fact_mat_maxfacts(self, sample_ids, fact_dropout):
        raise NotImplementedError("replaced by loader.install_graft")

    def _graft_facts(self, q):
        h, r, t = self.kb_adj_mats[q]
        f = np.arange(len(h))
        ones = np.ones(len(h))
        return ((f, h, ones), (t, f.copy(), ones.copy())), self.kb_fact_rels[q]

    def reset_batches(self, is_sequential=True):
        self.batches = np.arange(self.num_data) if is_sequential else np.random.permutation(self.num_data)

    def get_batch(self, iteration, batch_size, fact_dropout, q_type=None, test=False):
        ids = self.batches[batch_size * iteration:min(batch_size * (iteration + 1), self.num_data)]
        self.sample_ids = ids
        kb = self._build_fact_mat(ids, fact_dropout)
        head = (self.candidate_entities[ids], self.query_entities[ids], kb)
        tail = (self.seed_distribution[ids], None, self.answer_dists[ids])
        if hasattr(self, "kb_fact_rels"):
            graft, _ = self._build_fact_mat_maxfacts(ids, fact_dropout)
            out = head + (graft, self.query_texts[ids], self.kb_fact_rels[ids]) + tail
        else:
            out = head + (self.query_texts[ids],) + tail
        return out + ((self.answer_lists[ids],) if test else ())


def serve_pass(data, step, B):
    """One pass over the split, evaluator-shaped; -> seconds."""
    nb = (data.num_data + B - 1) // B
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    pending = None
    for it in range(nb):
        batch = data.get_batch(it, B, 0.0, test=True)
        t = step.submit(batch[:-1])
        if pending is not None:
            step.collect(pending)
        pending = t
    step.collect(pending)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--questions", type=int, default=640)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--models", default="ReaRev,GraftNet")
    ap.add_argument("--batch", default="20,64")
    ap.add_argument("--dims", default="50,200")
    a = ap.parse_args()
    info = gpu_info()
    dev = torch.device("cuda")
    for name in a.models.split(","):
        graft = name == "GraftNet"
        L = SyntheticSplit(a.questions, graft=graft)
        loader.install(L, weights="none", index_dtype=np.int32, shuffle=False)
        if graft:
            loader.install_graft(L)
        split = loader.DeviceSplit(L, dev, weights="none", index_dtype=torch.int32)
        for D in (int(x) for x in a.dims.split(",")):
            args = S.model_args(name, entity_dim=D, use_cuda=True)
            torch.manual_seed(0)
            m = {"ReaRev": G.ReaRev, "GraftNet": G.GraftNet}[name](dict(args), NE, NR, NW).cuda().eval()
            for B in (int(x) for x in a.batch.split(",")):
                step = graphed.GraphedStep(m, NE, max_graphs=16)
                modes = {"host": L, "device": split}
                for data in modes.values():                   # warm-up: captures, pipeline buffers, caches
                    serve_pass(data, step, B)
                secs = {k: [] for k in modes}
                for _ in range(a.runs):
                    for k, data in modes.items():
                        secs[k].append(serve_pass(data, step, B))
                qps = {k: a.questions / float(np.median(v)) for k, v in secs.items()}
                print(json.dumps(dict(
                    model=name, D=D, B=B, N=L.max_local_entity, E=6000, questions=a.questions,
                    host_qps=round(qps["host"], 1), device_qps=round(qps["device"], 1),
                    speedup=round(qps["device"] / qps["host"], 2),
                    host_s=[round(x, 4) for x in secs["host"]], device_s=[round(x, 4) for x in secs["device"]],
                    split_build_s=round(split.build_seconds, 3), resident_mb=round(split.resident_bytes / 2 ** 20, 1),
                    gpu=info)), flush=True)
                del step
                torch.cuda.empty_cache()
        del split


if __name__ == "__main__":
    main()
