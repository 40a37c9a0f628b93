"""Question-sharded multi-GPU execution (SURVEY.md 8e).

The batched graph is block diagonal by construction (gnn/dataset_load.py:483,492-493): question ``b`` owns
node rows ``[b*N,(b+1)*N)`` and its facts never leave the block; softmax and instructions are per question.
So rank ``g`` of ``G`` takes a contiguous question range, weights are replicated, there is NO communication
during the forward, and one all-gather of the ``[B/G, N]`` answer scores at the end.  The partition is
pure index arithmetic and is tested on CPU with gloo, world_size 2 (tests/test_host_logic.py).
"""
import numpy as np
import torch
import torch.distributed as dist


def question_range(B, rank, world):
    """Contiguous, balanced split of B questions: the first B % world ranks get one extra."""
    base, extra = divmod(B, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def shard_batch(batch, rank, world):
    """Slice a ``get_batch`` tuple down to this rank's questions (facts re-based to local rows)."""
    local_entity, query_entities, kb, q_input, seed_dist, tb, answer_dist = batch[:7]
    B, N = local_entity.shape
    lo, hi = question_range(B, rank, world)
    heads, rels, tails, bids, fids, wl, wrl = kb
    bids = np.asarray(bids)
    sel = np.nonzero((bids >= lo) & (bids < hi))[0]
    off = lo * N
    h, r, t = np.asarray(heads)[sel] - off, np.asarray(rels)[sel], np.asarray(tails)[sel] - off
    wl2 = None if wl is None else np.asarray(wl, dtype=np.float64)[sel].tolist()
    wrl2 = None if wrl is None else np.asarray(wrl, dtype=np.float64)[sel].tolist()
    kb2 = (h, r, t, bids[sel] - lo, np.arange(len(sel), dtype=np.int64), wl2, wrl2)
    out = (local_entity[lo:hi], query_entities[lo:hi], kb2, q_input[lo:hi], seed_dist[lo:hi], tb,
           answer_dist[lo:hi])
    if len(batch) > 7:
        out = out + (batch[7][lo:hi],)
    return out


def shard_graft_batch(batch, rank, world):
    """Slice a ``GraftSingleDataLoader.get_batch`` 9/10-tuple down to this rank's questions: the kb part as
    :func:`shard_batch`; of both graft lists the entries of these questions, in their original order, with the
    question id re-based (the fact slot f and the local node ids are per question already); ``kb_fact_rel``,
    ``q_input``, the [B, N] arrays and ``answer_lists`` by rows."""
    (local_entity, query_entities, kb, graft, q_input, kb_fact_rel, seed_dist, tb, answer_dist) = batch[:9]
    B = local_entity.shape[0]
    lo, hi = question_range(B, rank, world)
    kb_part = shard_batch((local_entity, query_entities, kb, q_input, seed_dist, tb, answer_dist), rank, world)

    def lists(lst, bcol):
        b = np.asarray(lst[bcol])
        sel = np.nonzero((b >= lo) & (b < hi))[0]
        out = [np.asarray(a)[sel] for a in lst]
        out[bcol] = out[bcol] - lo
        return tuple(out)
    graft2 = (lists(graft[0], 0), lists(graft[1], 0))
    out = (kb_part[0], kb_part[1], kb_part[2], graft2, kb_part[3], kb_fact_rel[lo:hi], kb_part[4], tb, kb_part[6])
    if len(batch) > 9:
        out = out + (batch[9][lo:hi],)
    return out


def all_gather_scores(local_scores, B, group=None):
    """Gather per-rank ``[B_g, N]`` score blocks into the full ``[B, N]`` matrix on every rank (NCCL
    over NVLink on GPUs, gloo on CPU).  Ragged splits are padded to the largest block."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    N = local_scores.shape[1]
    sizes = [question_range(B, r, world)[1] - question_range(B, r, world)[0] for r in range(world)]
    mx = max(sizes)
    pad = local_scores
    if local_scores.shape[0] < mx:
        pad = torch.zeros(mx, N, dtype=local_scores.dtype, device=local_scores.device)
        pad[: local_scores.shape[0]] = local_scores
    full = torch.empty(world * mx, N, dtype=local_scores.dtype, device=local_scores.device)
    dist.all_gather_into_tensor(full, pad.contiguous(), group=group)
    if all(s == mx for s in sizes):
        return full
    return torch.cat([full[r * mx: r * mx + sizes[r]] for r in range(world)], dim=0)
