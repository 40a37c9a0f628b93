"""Host batch tuple -> device-resident batch (the ``dataset_load batching into CSR`` subsystem).

The reference hands ``model.forward`` a tuple of host numpy arrays (gnn/dataset_load.py:623-629) and then
(a) converts every array to a torch tensor and copies it (gnn/models/ReaRev/rearev.py:169-177) and (b)
re-builds seven COO sparse tensors from python lists inside ``build_matrix``
(gnn/modules/kg_reasoning/base_gnn.py:19-51).  Here the raw int64 fact arrays are copied once and the two
destination-CSRs are built on the GPU (csrc/csr_build.cu).  A :class:`DeviceBatch` can also be built
ahead of time and passed to ``forward`` in place of the tuple (pre-staged inputs).
"""
import numpy as np
import torch

from . import ops


class DeviceBatch:
    """Everything ``forward`` needs, resident in HBM."""

    def __init__(self):
        self.B = self.N = self.F = 0
        self.local_entity = None     # int64 [B,N]
        self.query_entities = None   # fp32  [B,N]
        self.seed_dist = None        # fp32  [B,N]
        self.answer_dist = None      # fp32  [B,N]
        self.q_input = None          # int64 [B,Q]
        self.graph = None            # ops.CsrGraph
        self.h2d_bytes = 0


def _to_dev(x, device, dtype=None):
    """numpy array / host tensor (pinned or pageable) / device tensor -> device tensor of ``dtype``."""
    if isinstance(x, torch.Tensor):
        t = x
    else:
        t = torch.from_numpy(np.ascontiguousarray(x))
    if t.device != device:
        t = t.to(device, non_blocking=True)
    if dtype is not None and t.dtype != dtype:
        t = t.to(dtype)                      # cast on the device (tiny [B,N] arrays)
    return t


def pin_batch(batch):
    """Copy the numpy arrays of a ``get_batch`` tuple into pinned host tensors (bench.py's e2e leg)."""
    def pin(a):
        return torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
    le, qe, kb, qi, sd, tb, ad = batch[:7]
    kb2 = (pin(kb[0]), pin(kb[1]), pin(kb[2]), None, None, kb[5], kb[6])
    return (pin(le), pin(qe.astype(np.float32)), kb2, pin(qi), pin(sd.astype(np.float32)), tb,
            pin(ad.astype(np.float32)))


def pin_graft_batch(batch):
    """:func:`pin_batch` for a ``GraftSingleDataLoader.get_batch`` tuple: the kb part as there, the two graft lists and
    ``kb_fact_rel`` as pinned int64 tensors."""
    def pin(a, dtype=np.int64):
        return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=dtype))).pin_memory()
    le, qe, kb, qi, sd, tb, ad = pin_batch((batch[0], batch[1], batch[2], batch[4], batch[6], batch[7], batch[8]))
    (hb, hf, he, hv), (tb_, te, tf, tv) = batch[3]
    graft = ((pin(hb), pin(hf), pin(he), hv), (pin(tb_), pin(te), pin(tf), tv))
    return (le, qe, kb, graft, qi, pin(batch[5]), sd, tb, ad) + tuple(batch[9:])


def stage_batch(batch, device, num_rel_rows, normalized_gnn=False, norm_rel=False, nfacts=None):
    """Copy one ``get_batch`` tuple to the device and build its CSRs.  Returns DeviceBatch.
    ``nfacts``: optional int32[1] device tensor with the number of live facts when the fact arrays are fixed-capacity
    buffers (GraphedStep); the weight lists, if used, must then have the same capacity."""
    if isinstance(batch, DeviceBatch):
        return batch
    local_entity, query_entities, kb_adj_mat, q_input, seed_dist, _true_batch_id, answer_dist = batch[:7]
    db = DeviceBatch()
    B, N = local_entity.shape
    db.B, db.N = B, N
    db.local_entity = _to_dev(local_entity, device, torch.int64)
    db.query_entities = _to_dev(query_entities, device, torch.float32)
    db.seed_dist = _to_dev(seed_dist, device, torch.float32)
    db.answer_dist = _to_dev(answer_dist, device, torch.float32)
    db.q_input = _to_dev(q_input, device, torch.int64)
    heads, rels, tails, _bids, _fids, weight_list, weight_rel_list = kb_adj_mat
    if not isinstance(heads, torch.Tensor):
        heads = np.asarray(heads)
        if heads.dtype not in (np.int64, np.int32):
            heads = heads.astype(np.int64)
        rels = np.asarray(rels).astype(heads.dtype, copy=False)
        tails = np.asarray(tails).astype(heads.dtype, copy=False)
    F = int(heads.shape[0])
    db.F = F
    dh, dr, dt = _to_dev(heads, device), _to_dev(rels, device), _to_dev(tails, device)
    db.graph = ops.csr_build(dh, dr, dt, B, N, num_rel_rows, nfacts)
    nbytes = (db.local_entity.numel() * 8 + db.q_input.numel() * 8 + 3 * B * N * 4
              + 3 * F * dh.element_size())
    if (normalized_gnn and weight_list is None) or (norm_rel and weight_rel_list is None):
        raise ValueError("normalized_gnn / norm_rel need kb_adj_mat's weight_list / weight_rel_list "
                         "(the loader was built with weights='none'?)")

    def wdev(w):
        return w.to(device=device, dtype=torch.float32) if isinstance(w, torch.Tensor) \
            else _to_dev(np.asarray(w, dtype=np.float32), device)
    if normalized_gnn and F > 0:      # COO values of build_matrix, base_gnn.py:38-41
        w = wdev(weight_list)
        db.graph.w_t = ops.gather_f32(w, db.graph.fact_t)
        db.graph.w_h = ops.gather_f32(w, db.graph.fact_h)
        nbytes += 4 * F
    if norm_rel and F > 0:            # TypeLayer values, layer_init.py:39-42
        wr = wdev(weight_rel_list)
        db.graph.wr_t = ops.gather_f32(wr, db.graph.fact_t)
        db.graph.wr_h = ops.gather_f32(wr, db.graph.fact_h)
        nbytes += 4 * F
    db.h2d_bytes = int(nbytes)
    return db


def stage_graft_batch(batch, device, num_rel_rows, normalized_gnn=False, norm_rel=False, nfacts=None, graft_live=None):
    """Copy one ``GraftSingleDataLoader.get_batch`` tuple (gnn/dataset_load_graft.py:113-149) to the device: the regular
    CSRs of ``kb_adj_mat`` (the TypeLayer input) as :func:`stage_batch` builds them, plus the graft facts of
    ``kb_adj_mat_graft`` paired by slot and ordered by (b, f) with their CSRs (``db.graft``, ops.GraftGraph).
    Fixed-capacity buffers (GraphedStep): ``nfacts`` int32[1] = live kb facts (see :func:`stage_batch`),
    ``graft_live`` int32[2] = live entries of the graft head and tail lists (``ops.graft_stage(live=...)``)."""
    if isinstance(batch, DeviceBatch):
        return batch
    (local_entity, query_entities, kb_adj_mat, kb_adj_mat_graft, q_input, kb_fact_rel, seed_dist, true_batch_id,
     answer_dist) = batch[:9]
    db = stage_batch((local_entity, query_entities, kb_adj_mat, q_input, seed_dist, true_batch_id, answer_dist),
                     device, num_rel_rows, normalized_gnn, norm_rel, nfacts=nfacts)
    (e2f_b, e2f_f, e2f_e, _v0), (f2e_b, f2e_e, f2e_f, _v1) = kb_adj_mat_graft

    def idx(a):
        if isinstance(a, torch.Tensor):
            return a.to(device=device, dtype=torch.int64)
        return _to_dev(np.asarray(a).astype(np.int64, copy=False), device)
    rel = idx(kb_fact_rel)
    if rel.dim() != 2:
        rel = rel.view(db.B, -1)
    db.graft = ops.graft_stage([idx(e2f_b), idx(e2f_f), idx(e2f_e)], [idx(f2e_b), idx(f2e_e), idx(f2e_f)], rel,
                               db.B, db.N, num_rel_rows, live=graft_live)
    db.h2d_bytes += 8 * (rel.numel() + 3 * len(e2f_b) + 3 * len(f2e_b))
    return db
