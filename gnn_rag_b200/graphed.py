"""CUDA-graph execution of the whole hot-path step for fixed batch shapes.

One step = CSR batching of the fact list -> model.forward -> candidate ranking.  It launches ~70 kernels, most of
them small, so at WebQSP batch sizes the GPU idles between launches.  :class:`GraphedStep` captures the step into a
CUDA graph over static device buffers and replays it: per call it only copies the host batch into the static buffers
(H2D from pinned or pageable memory), replays, and returns views of the static outputs.  The numerics are those of
the eager path (same kernels, same order).

Shapes.  A graph is fixed in ``(B, N, Q)`` and in the CAPACITY of its fact buffers.  ``get_batch`` returns a different
fact count F for almost every batch (gnn/dataset_load.py:473-527), so capacities are bucketed (8 buckets per octave,
<= 12.5 % padding): the batch's facts occupy the front of the buffers, a device-side counter tells the CSR build how
many slots are live (``gr_csr_build(..., nfacts)``) and everything downstream sees live facts only, through the row
pointers.  Captured graphs are kept in an LRU cache (``max_graphs``); the graph, its static buffers, landing buffers
and pinned host buffers of an evicted entry are released.

Serving loop: :meth:`GraphedStep.submit` / :meth:`GraphedStep.collect` pipeline two batches -- the H2D copy of
batch i+1 (copy stream, into a landing buffer set) and the D2H read of batch i's results overlap the graph of
batch i, so the end-to-end rate is bounded by the device time of the step, not by device + PCIe time.

Models.  The input side is a per-model layout chosen from the model class: :class:`_KbLayout` for the 7-tuple of
``SingleDataLoader.get_batch`` (ReaRev, NSM) and :class:`_GraftLayout` for the 9/10-tuple of
``GraftSingleDataLoader.get_batch`` (GraftNet: two more fact lists at their own bucketed capacity with live counts for
``gr_graft_stage``, and ``kb_fact_rel``).  The LRU, the pipeline and the streams are shared.  The status words of the
step (one per CSR build / staging) travel back with the results and are checked on the host after the step.
"""
import collections

import numpy as np
import torch

from . import batching, ops
from .modules import live_plane_buffers


class StepOutput:
    __slots__ = ("loss", "pred", "pred_dist", "cand_idx", "cand_count", "cand_total", "db")


class _Captured:
    pass


class Ticket:
    """One in-flight step of the submit/collect pipeline."""
    __slots__ = ("slot", "done", "ent", "local_entity_host", "B", "N")


def fact_capacity(F):
    """Bucketed capacity for a batch of F facts: next multiple of 2^(floor(log2 F) - 3), at least 1024."""
    F = max(int(F), 1)
    g = max(1 << max(F.bit_length() - 4, 0), 1024)
    return (F + g - 1) // g * g


def _host(src, dtype):
    t = src if isinstance(src, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(np.asarray(src)))
    if t.dtype != dtype and not t.is_cuda:
        t = t.to(dtype)
    return t


def _put(dst, src):
    dst.copy_(_host(src, dst.dtype), non_blocking=True)


def _put_front(dst, src, F):
    dst[:F].copy_(_host(src, dst.dtype), non_blocking=True)


def _stage_copy(dst, src, n=None):
    """pageable ``src`` -> pinned ``dst`` (or its first ``n`` entries) by host memcpy with a cast."""
    d = dst.numpy() if n is None else dst.numpy()[:n]
    np.copyto(d, src.numpy() if isinstance(src, torch.Tensor) else np.asarray(src), casting="unsafe")
    return dst if n is None else dst[:n]


class _KbLayout:
    """Input side of the 7-tuple of ``SingleDataLoader.get_batch`` (ReaRev, NSM)."""

    def __init__(self, step):
        self.step = step
        m = step.model
        self.weights = bool(m.normalized_gnn), bool(m.norm_rel)

    @staticmethod
    def kb_view(batch):
        """(local_entity, query_entities, kb_adj_mat, q_input, seed_dist, true_batch_id, answer_dist)."""
        return batch[:7]

    def key(self, batch):
        le, _qe, kb, qi = self.kb_view(batch)[:4]
        B, N = le.shape
        cap = fact_capacity(int(kb[0].shape[0]))
        Q = int(qi.shape[1])
        idx_dtype = torch.int32 if str(kb[0].dtype).endswith("int32") else torch.int64
        return (B, N, cap, Q, idx_dtype)

    def static_inputs(self, key):
        B, N, cap, Q, idx_dtype = key[:5]
        dev = self.step.device
        st = _Captured()
        st.local_entity = torch.zeros(B, N, dtype=torch.int64, device=dev)
        st.query_entities = torch.zeros(B, N, dtype=torch.float32, device=dev)
        st.seed_dist = torch.zeros(B, N, dtype=torch.float32, device=dev)
        st.answer_dist = torch.zeros(B, N, dtype=torch.float32, device=dev)
        st.q_input = torch.zeros(B, Q, dtype=torch.int64, device=dev)
        st.heads = torch.zeros(cap, dtype=idx_dtype, device=dev)
        st.rels = torch.zeros(cap, dtype=idx_dtype, device=dev)
        st.tails = torch.zeros(cap, dtype=idx_dtype, device=dev)
        st.nfacts = torch.zeros(1, dtype=torch.int32, device=dev)
        st.weight_list = torch.ones(cap, dtype=torch.float32, device=dev) if self.weights[0] else None
        st.weight_rel_list = torch.ones(cap, dtype=torch.float32, device=dev) if self.weights[1] else None
        return st

    def names(self):
        names = ["local_entity", "query_entities", "seed_dist", "answer_dist", "q_input", "heads", "rels", "tails",
                 "nfacts"]
        if self.weights[0]:
            names.append("weight_list")
        if self.weights[1]:
            names.append("weight_rel_list")
        return names

    def fill(self, st, batch):
        """Host batch -> the buffers of ``st`` (facts to the front of the capacity, live count to ``nfacts``);
        returns the bytes copied."""
        le, qe, kb, qi, sd, _, ad = self.kb_view(batch)
        F = int(kb[0].shape[0])
        _put(st.local_entity, le); _put(st.query_entities, qe); _put(st.seed_dist, sd); _put(st.answer_dist, ad)
        _put(st.q_input, qi)
        _put_front(st.heads, kb[0], F); _put_front(st.rels, kb[1], F); _put_front(st.tails, kb[2], F)
        if st.weight_list is not None:
            if kb[5] is None:
                raise ValueError("normalized_gnn needs kb_adj_mat's weight_list")
            _put_front(st.weight_list,
                       np.asarray(kb[5], dtype=np.float32) if not isinstance(kb[5], torch.Tensor) else kb[5], F)
        if st.weight_rel_list is not None:
            if kb[6] is None:
                raise ValueError("norm_rel needs kb_adj_mat's weight_rel_list")
            _put_front(st.weight_rel_list,
                       np.asarray(kb[6], dtype=np.float32) if not isinstance(kb[6], torch.Tensor) else kb[6], F)
        st.nfacts.copy_(torch.tensor([F], dtype=torch.int32), non_blocking=True)
        idx_b = st.heads.element_size()
        return (st.local_entity.numel() * 8 + st.q_input.numel() * 8 + 3 * st.seed_dist.numel() * 4
                + 3 * F * idx_b + 4 + 4 * F * (int(st.weight_list is not None) + int(st.weight_rel_list is not None)))

    @staticmethod
    def needs_staging(batch):
        """True when the batch lives in pageable host memory (numpy arrays / unpinned CPU tensors)."""
        x = batch[2][0]
        if isinstance(x, torch.Tensor):
            return (not x.is_cuda) and (not x.is_pinned())
        return True

    def stage_host(self, stage, batch):
        """Cast + copy a pageable ``get_batch`` tuple into the pinned staging set (host memcpy); returns a tuple over the
        staged tensors that ``fill`` can DMA asynchronously."""
        le, qe, kb, qi, sd, _, ad = self.kb_view(batch)
        F = int(kb[0].shape[0])
        put = _stage_copy
        wl = put(stage.weight_list, np.asarray(kb[5], dtype=np.float32), F) if stage.weight_list is not None else None
        wr = put(stage.weight_rel_list, np.asarray(kb[6], dtype=np.float32), F) if stage.weight_rel_list is not None \
            else None
        kb2 = (put(stage.heads, kb[0], F), put(stage.rels, kb[1], F), put(stage.tails, kb[2], F), None, None, wl, wr)
        return (put(stage.local_entity, le), put(stage.query_entities, qe), kb2, put(stage.q_input, qi),
                put(stage.seed_dist, sd), None, put(stage.answer_dist, ad))

    def run(self, st):
        """The model part of the captured step -> (db, loss, pred, pred_dist)."""
        m = self.step.model
        tup = (st.local_entity, st.query_entities,
               (st.heads, st.rels, st.tails, None, None, st.weight_list, st.weight_rel_list),
               st.q_input, st.seed_dist, None, st.answer_dist)
        db = batching.stage_batch(tup, self.step.device, m.num_relation + 1, m.normalized_gnn, m.norm_rel,
                                  nfacts=st.nfacts)
        loss, pred, pred_dist, _ = m(db)
        return db, loss, pred, pred_dist

    @staticmethod
    def status_words(db):
        """Device int32[1] status words of the step, in the order :meth:`raise_for` reads them."""
        return [db.graph.status]

    @staticmethod
    def raise_for(words):
        """ids outside the batch are clamped by the CSR build and flagged (a malformed / mis-sharded fact list)."""
        if int(words[0]) != 0:
            raise RuntimeError("fact list contains node/relation ids outside the batch (clamped)")

    def check(self, db):
        self.raise_for(torch.cat(self.status_words(db)).tolist())


class _GraftLayout(_KbLayout):
    """Input side of the 9/10-tuple of ``GraftSingleDataLoader.get_batch`` (GraftNet): the kb part as
    :class:`_KbLayout`, plus both graft lists -- (b, f, head) and (b, tail, f), int64 at ``fact_capacity`` of the
    longer list, live counts in ``graft_live`` -- and ``kb_fact_rel`` [B, max_fact]."""

    LIST_NAMES = ["e2f_b", "e2f_f", "e2f_e", "f2e_b", "f2e_e", "f2e_f"]

    @staticmethod
    def kb_view(batch):
        return batch[0], batch[1], batch[2], batch[4], batch[6], batch[7], batch[8]

    def key(self, batch):
        (hb, _hf, _he, _hv), (tb, _te, _tf, _tv) = batch[3]
        gcap = fact_capacity(max(len(hb), len(tb)))
        kfr = batch[5]
        max_fact = int(kfr.shape[-1]) if len(kfr.shape) == 2 else int(kfr.shape[0]) // len(batch[0])
        return super().key(batch) + (gcap, max_fact)

    def static_inputs(self, key):
        st = super().static_inputs(key)
        B, gcap, max_fact = key[0], key[5], key[6]
        dev = self.step.device
        for name in self.LIST_NAMES:
            setattr(st, name, torch.zeros(gcap, dtype=torch.int64, device=dev))
        st.graft_live = torch.zeros(2, dtype=torch.int32, device=dev)
        st.kb_fact_rel = torch.zeros(B, max_fact, dtype=torch.int64, device=dev)
        return st

    def names(self):
        return super().names() + self.LIST_NAMES + ["graft_live", "kb_fact_rel"]

    def fill(self, st, batch):
        nbytes = super().fill(st, batch)
        (hb, hf, he, _hv), (tb, te, tf, _tv) = batch[3]
        F0, F1 = len(hb), len(tb)
        for name, src, F in zip(self.LIST_NAMES, (hb, hf, he, tb, te, tf), (F0, F0, F0, F1, F1, F1)):
            _put_front(getattr(st, name), src, F)
        st.graft_live.copy_(torch.tensor([F0, F1], dtype=torch.int32), non_blocking=True)
        _put(st.kb_fact_rel, _host(batch[5], torch.int64).view(st.kb_fact_rel.shape))
        return nbytes + 8 * (3 * F0 + 3 * F1 + st.kb_fact_rel.numel()) + 8

    @staticmethod
    def needs_staging(batch):
        x = batch[3][0][0]
        pageable = (not x.is_cuda) and (not x.is_pinned()) if isinstance(x, torch.Tensor) else True
        return pageable or _KbLayout.needs_staging(batch)

    def stage_host(self, stage, batch):
        le, qe, kb2, qi, sd, _, ad = super().stage_host(stage, batch)
        (hb, hf, he, _hv), (tb, te, tf, _tv) = batch[3]
        F0, F1 = len(hb), len(tb)
        e2f = tuple(_stage_copy(getattr(stage, n), a, F0) for n, a in zip(self.LIST_NAMES[:3], (hb, hf, he)))
        f2e = tuple(_stage_copy(getattr(stage, n), a, F1) for n, a in zip(self.LIST_NAMES[3:], (tb, te, tf)))
        kfr = batch[5]
        kfr = _stage_copy(stage.kb_fact_rel, np.asarray(kfr.numpy() if isinstance(kfr, torch.Tensor) else kfr)
                          .reshape(stage.kb_fact_rel.shape))
        return (le, qe, kb2, (e2f + (None,), f2e + (None,)), qi, kfr, sd, None, ad)

    def run(self, st):
        m = self.step.model
        tup = (st.local_entity, st.query_entities,
               (st.heads, st.rels, st.tails, None, None, st.weight_list, st.weight_rel_list),
               ((st.e2f_b, st.e2f_f, st.e2f_e, None), (st.f2e_b, st.f2e_e, st.f2e_f, None)),
               st.q_input, st.kb_fact_rel, st.seed_dist, None, st.answer_dist)
        db = batching.stage_graft_batch(tup, self.step.device, m.num_relation + 1, m.normalized_gnn, m.norm_rel,
                                        nfacts=st.nfacts, graft_live=st.graft_live)
        with torch.no_grad():        # the status words are read by GraphedStep after the step, not inside the capture
            loss, pred, pred_dist, _ = m._forward_infer(db, check_status=False)
        return db, loss, pred, pred_dist

    @staticmethod
    def status_words(db):
        return [db.graph.status, db.graft.status, db.graft.graph.status]

    @staticmethod
    def raise_for(words):
        kb, graft, graft_csr = (int(w) for w in words)
        ops.GraftGraph.raise_status(graft)
        if graft_csr or kb:
            _KbLayout.raise_for([graft_csr | kb])


def _layout_for(model):
    from .models import GraftNet
    return _GraftLayout if isinstance(model, GraftNet) else _KbLayout


class GraphedStep:
    def __init__(self, model, num_entity, eps=None, max_graphs=8):
        self.model = model
        self.num_entity = num_entity
        self.eps = model.eps if eps is None else eps
        self.device = next(model.parameters()).device
        self.max_graphs = max_graphs
        self._cache = collections.OrderedDict()
        self._copy_stream = None      # H2D stream
        self._d2h_stream = None       # separate: a D2H waiting for graph i must not block the H2D of batch i+1
        self._slot = 0
        self._layout = _layout_for(model)(self)

    # -- the work that gets captured ------------------------------------------------------------------------
    def _run(self, st):
        db, loss, pred, pred_dist = self._layout.run(st)
        cand_idx, cand_count, cand_total = ops.rank_candidates(pred_dist, db.local_entity, db.query_entities,
                                                              self.num_entity, self.eps)
        return db, loss, pred, pred_dist, cand_idx, cand_count, cand_total

    def _fill(self, st, batch):
        self._h2d_bytes = self._layout.fill(st, batch)

    def _entry(self, batch):
        # parameter versions are part of the key: the captured graph holds pre-formatted (split-bf16) weights
        shape_key = self._layout.key(batch)
        key = shape_key + (sum(p._version for p in self.model.parameters()),)
        ent = self._cache.get(key)
        if ent is not None:
            self._cache.move_to_end(key)
            return ent
        while len(self._cache) >= self.max_graphs:          # LRU eviction: graph, static + landing + pinned buffers
            _k, old = self._cache.popitem(last=False)
            torch.cuda.synchronize()
            del old
        st = self._layout.static_inputs(shape_key)
        self._fill(st, batch)
        torch.cuda.synchronize()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):            # warm-up on a side stream (lazy init, allocator, caches)
            for _ in range(2):
                self._run(st)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            outs = self._run(st)
        ent = _Captured()
        ent.st, ent.g, ent.outs = st, g, outs
        ent.pipe = None
        ent.weight_ws = ops.live_weight_workspaces()        # the graph reads these pre-formatted weights: keep them alive
        # ... and these operand planes: a layer drops its cached planes when another (B*N, width) arrives, and the
        # graph still relies on them (and on their zero pad columns) when it replays
        ent.planes = live_plane_buffers()
        self._cache[key] = ent
        return ent

    def _check(self, db):
        self._layout.check(db)

    def __call__(self, batch, check=False):
        ent = self._entry(batch)
        self._fill(ent.st, batch)
        ent.g.replay()
        o = StepOutput()
        o.db, o.loss, o.pred, o.pred_dist, o.cand_idx, o.cand_count, o.cand_total = ent.outs
        o.db.h2d_bytes = self._h2d_bytes
        self.model.last_batch = o.db
        if check:
            self._check(o.db)
        return o

    # -- two-deep pipeline: H2D of batch i+1 and D2H of batch i overlap the graph of batch i -----------------
    def _pipe(self, ent):
        if ent.pipe is None:
            if self._copy_stream is None:
                self._copy_stream = torch.cuda.Stream()
                self._d2h_stream = torch.cuda.Stream()
            db, loss, pred, pred_dist, cand_idx, cand_count, _ = ent.outs
            pipe = _Captured()
            pipe.land, pipe.out_dev, pipe.out_host = [], [], []
            pipe.land_free, pipe.done = [], []
            for _ in range(2):
                land = _Captured()
                for name in self._layout.names():
                    setattr(land, name, torch.empty_like(getattr(ent.st, name)))
                land.weight_list = getattr(land, "weight_list", None)
                land.weight_rel_list = getattr(land, "weight_rel_list", None)
                pipe.land.append(land)
                od = dict(cand_idx=torch.empty_like(cand_idx), pred_dist=torch.empty_like(pred_dist),
                          cand_count=torch.empty_like(cand_count), pred=torch.empty_like(pred),
                          loss=torch.empty_like(loss),
                          status=torch.empty(len(self._layout.status_words(db)), dtype=torch.int32,
                                             device=self.device))
                pipe.out_dev.append(od)
                pipe.out_host.append({k: torch.empty(v.shape, dtype=v.dtype, pin_memory=True)
                                      for k, v in od.items()})
                pipe.land_free.append(None)
                pipe.done.append(None)
                # pinned host staging of the inputs: pageable loader output (numpy, int64 / float64) is cast and copied
                # here by the host (memcpy speed), the DMA to the landing set then runs asynchronously
                stage = _Captured()
                for name in self._layout.names():
                    t = getattr(ent.st, name)
                    setattr(stage, name, torch.empty(t.shape, dtype=t.dtype, pin_memory=True))
                stage.weight_list = getattr(stage, "weight_list", None)
                stage.weight_rel_list = getattr(stage, "weight_rel_list", None)
                pipe.stage = getattr(pipe, "stage", [])
                pipe.stage.append(stage)
                pipe.h2d_done = getattr(pipe, "h2d_done", [])
                pipe.h2d_done.append(None)
            ent.pipe = pipe
        return ent.pipe

    def submit(self, batch):
        """Enqueue one step (H2D of ``batch`` on the copy stream, graph replay, async D2H of the results) and
        return a :class:`Ticket`.  At most two tickets may be outstanding; ``collect`` them in order."""
        ent = self._entry(batch)
        pipe = self._pipe(ent)
        slot, self._slot = self._slot, self._slot ^ 1
        cs, cur = self._copy_stream, torch.cuda.current_stream()
        if pipe.done[slot] is not None:
            pipe.done[slot].synchronize()            # host buffers of this slot have been read out
        if pipe.land_free[slot] is not None:
            cs.wait_event(pipe.land_free[slot])
        land = pipe.land[slot]
        src = batch
        if self._layout.needs_staging(batch):
            if pipe.h2d_done[slot] is not None:
                pipe.h2d_done[slot].synchronize()    # the previous DMA out of this staging set has finished
            src = self._layout.stage_host(pipe.stage[slot], batch)
        with torch.cuda.stream(cs):
            self._fill(land, src)
            h2d_done = torch.cuda.Event()
            h2d_done.record(cs)
        pipe.h2d_done[slot] = h2d_done
        cur.wait_event(h2d_done)
        for name in self._layout.names():            # landing set -> the graph's static inputs (D2D, ~10 us)
            getattr(ent.st, name).copy_(getattr(land, name), non_blocking=True)
        pipe.land_free[slot] = torch.cuda.Event()
        pipe.land_free[slot].record(cur)
        ent.g.replay()
        db, loss, pred, pred_dist, cand_idx, cand_count, _ = ent.outs
        od = pipe.out_dev[slot]
        od["cand_idx"].copy_(cand_idx, non_blocking=True)
        od["pred_dist"].copy_(pred_dist, non_blocking=True)
        od["cand_count"].copy_(cand_count, non_blocking=True)
        od["pred"].copy_(pred, non_blocking=True)
        od["loss"].copy_(loss, non_blocking=True)
        for i, w in enumerate(self._layout.status_words(db)):
            od["status"][i:i + 1].copy_(w, non_blocking=True)
        out_ready = torch.cuda.Event()
        out_ready.record(cur)
        ds = self._d2h_stream
        ds.wait_event(out_ready)
        with torch.cuda.stream(ds):
            for k, v in od.items():
                pipe.out_host[slot][k].copy_(v, non_blocking=True)
            pipe.done[slot] = torch.cuda.Event()
            pipe.done[slot].record(ds)
        db.h2d_bytes = self._h2d_bytes
        self.model.last_batch = db
        t = Ticket()
        t.slot, t.done, t.ent = slot, pipe.done[slot], ent
        le = batch[0]
        t.local_entity_host = le.cpu().numpy() if isinstance(le, torch.Tensor) else np.asarray(le)
        t.B, t.N = db.B, db.N
        return t

    def collect(self, ticket):
        """Wait for a submitted step and return (retrieved, d2h_bytes, loss, pred): the ordered candidate lists
        of every question (like :func:`evaluate.retrieve`), the bytes read back, the loss and the argmax.
        Raises if the CSR build (or, for GraftNet, the graft staging) flagged a malformed fact list."""
        from .evaluate import Retrieved
        ticket.done.synchronize()
        h = ticket.ent.pipe.out_host[ticket.slot]
        self._layout.raise_for(h["status"].tolist())
        idx_h, dist_h = h["cand_idx"].numpy(), h["pred_dist"].numpy()
        counts = h["cand_count"].numpy()
        le = ticket.local_entity_host
        res = []
        for b, c in enumerate(counts.tolist()):
            ix = idx_h[b, :c].astype(np.int64)
            res.append(Retrieved(ix, le[b, ix].astype(np.int64), dist_h[b, ix]))
        nbytes = sum(v.numel() * v.element_size() for v in h.values())
        return res, nbytes, float(h["loss"]), h["pred"].numpy().copy()

    def retrieve(self, out):
        """Ordered candidate lists of a :class:`StepOutput` (one D2H), like evaluate.retrieve."""
        from .evaluate import Retrieved
        counts_h = out.cand_count.cpu().numpy()
        self._check(out.db)
        maxc = int(counts_h.max()) if counts_h.size else 0
        ei, ef = np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.float32)
        if maxc == 0:
            return [Retrieved(ei, ei, ef) for _ in range(out.db.B)], counts_h.size * 4
        idx = out.cand_idx[:, :maxc].long()
        probs = torch.gather(out.pred_dist, 1, idx)
        ents = torch.gather(out.db.local_entity, 1, idx)
        idx_h, probs_h, ents_h = idx.cpu().numpy(), probs.cpu().numpy(), ents.cpu().numpy()
        res = [Retrieved(idx_h[b, :c], ents_h[b, :c], probs_h[b, :c]) for b, c in enumerate(counts_h.tolist())]
        return res, counts_h.size * 4 + idx_h.size * 8 + probs_h.size * 4 + ents_h.size * 8
