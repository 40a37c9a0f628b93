"""Exact restatement of gr_eval_step_paths (csrc/paths.cu), the shortest-path node sets of one evaluation step, on
the shortest-path restatement of tests/retrieval_ref.py.  tests/test_eval_paths_gpu.py holds the entry point to it."""
import numpy as np

from retrieval_ref import path_nodes


def eval_step_paths(graphs, N, query_entities, cand_idx, cand_count, S, T):
    """gr_eval_step_paths on one step: per question (its (heads, tails) local node lists in ``graphs``), the sources
    are its local indices with an fp32 ``query_entities`` entry != 0, ascending, the first S of them, and the targets
    the first min(cand_count, T) entries of its ``cand_idx`` row -> [(sorted node list, int32 [S, T] pair distances
    with -1 past the counts)]."""
    out = []
    for b, (h, t) in enumerate(graphs):
        src = np.nonzero(np.asarray(query_entities[b], dtype=np.float32) != 0)[0][:S].tolist()
        tgt = np.asarray(cand_idx[b])[:min(max(int(cand_count[b]), 0), T)].tolist()
        _ds, _dt, pair, nodes = path_nodes(h, t, N, src, tgt)
        block = np.full((S, T), -1, dtype=np.int32)
        block[:len(src), :len(tgt)] = pair
        out.append((nodes, block))
    return out
