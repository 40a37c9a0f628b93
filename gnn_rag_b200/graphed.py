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
``gr_graft_stage``, and ``kb_fact_rel``).  The layout also holds the rest of what differs by model in the training
steps below.  The LRU, the capture routine, the pipeline and the streams are shared.  The status words of the step
(one per CSR build / staging) travel back with the results and are checked on the host after the step.

Training: :class:`GraphedTrainStep` captures ``model(batch, training=True)`` + ``loss.backward()`` + the train-time
metrics (gr_train_metrics) of ReaRev and NSM over the same input side, and :class:`GraphedGraftTrainStep` those of
GraftNet over :class:`_GraftLayout` (the graft fact count stays on the device).  Given a ``torch.optim.Adam``, both
also capture the gradient clipping and the optimizer step (:class:`optim.ClipAdam`); see their docstrings and DESIGN
§4.11.  :meth:`GraphedTrainStep.train_epoch` runs a whole ReaRev / NSM epoch over a ``loader.DeviceSplit``, and
:meth:`GraphedGraftTrainStep.train_epoch` a GraftNet one: each step's graph also assembles its batch (GraftNet: with
its graft lists) from a device cursor into the epoch's question order and records the step's loss and metrics on the
device (csrc/epoch.cu), so the host only replays graphs and reads the device once per epoch.
:meth:`GraphedStep.start_eval` evaluates a whole split the same way, through the same epoch driver (``_split_refusal``,
``_plan_epoch``, ``_epoch_graphs``, ``_warm_up_epoch_step``, ``_epoch_step``, ``_EpochJob``, ``_run_epochs``,
``_raise_epoch_status``): only the step each graph runs and the records it keeps differ.

Sweeps: :class:`Sweep` runs the epochs of several independent runs (distinct models on one GPU) side by side, each
member's graphs replayed on its own stream and drawing from its own CUDA generator and ``np.random.RandomState``, so
that every member computes the bits it computes alone.  A single epoch is a sweep of one job without a member: the same
``_run_epochs``.
"""
import collections
import contextlib
import gc

import numpy as np
import torch

from . import autograd_path, batching, ops, optim
from .modules import live_plane_buffers


class StepOutput:
    __slots__ = ("loss", "pred", "pred_dist", "cand_idx", "cand_count", "cand_total", "db")


class _Captured:
    pass


class Ticket:
    """One in-flight step of the submit/collect pipeline."""
    __slots__ = ("slot", "done", "ent", "local_entity_host", "cand_ent_host", "B", "N")


_INT32_MAX = 2 ** 31 - 1


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
    """What the graphed steps do differently per model family, for ReaRev and NSM: the input side of the 7-tuple of
    ``SingleDataLoader.get_batch``, the serving and training forwards, the training refusals and key scalars, and the
    model's part of an epoch graph."""

    def __init__(self, step):
        from .models import ReaRev
        self.step = step
        m = step.model
        self.weights = bool(m.normalized_gnn), bool(m.norm_rel)
        self.rearev = isinstance(m, ReaRev)

    @staticmethod
    def kb_view(batch):
        """(local_entity, query_entities, kb_adj_mat, q_input, seed_dist, true_batch_id, answer_dist)."""
        return batch[:7]

    @staticmethod
    def _shape_key(B, N, cap, Q, idx_dtype):
        return (B, N, cap, Q, idx_dtype)

    def key(self, batch):
        """The shape part of the capture key of ``batch``: (B, N, fact capacity, Q, index dtype)."""
        le, _qe, kb, qi = self.kb_view(batch)[:4]
        B, N = le.shape
        idx_dtype = torch.int32 if str(kb[0].dtype).endswith("int32") else torch.int64
        return self._shape_key(B, N, fact_capacity(int(kb[0].shape[0])), int(qi.shape[1]), idx_dtype)

    def model_key(self):
        """The Python scalars of the model that its training forward bakes into a graph (none for ReaRev / NSM)."""
        return ()

    def refusal(self, Q):
        """Why the eager training forward would leave the kernels for questions of Q tokens (a message), or None."""
        m = self.step.model
        dev, D = self.step.device, m.entity_dim
        I = m.num_ins if self.rearev else 1
        if not autograd_path.USE_KERNELS:
            return "autograd_path.USE_KERNELS is off: the training forward would run its torch restatement"
        if not ops.aggregate_backward_ok(D, I):
            return ("_kernel_graph is None: entity_dim %d with %d instruction(s) is outside the aggregation backward "
                    "kernel (%s)" % (D, I, ops.aggregate_backward_ok.__doc__.split(": ", 1)[1].rstrip(".")))
        if not autograd_path._instruction_kernels(dev, Q, D, m.instruction.num_ins):
            return ("_instruction_kernels is false: %d question tokens, entity_dim %d and %d instructions are outside "
                    "gr_instructions" % (Q, D, m.instruction.num_ins))
        if self.rearev and not autograd_path._reform_kernels(dev, D, I):
            return "_reform_kernels is false: entity_dim %d with %d instructions is outside gr_query_reform" % (D, I)
        if m.encode_type and not autograd_path._fact_kernels(dev, D):
            return "the TypeLayer kernel does not admit entity_dim %d (ops.fact_train_ok)" % D
        return None

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

    @staticmethod
    def batch_of(st):
        """The 7-tuple over the static buffers ``st``."""
        return (st.local_entity, st.query_entities,
                (st.heads, st.rels, st.tails, None, None, st.weight_list, st.weight_rel_list),
                st.q_input, st.seed_dist, None, st.answer_dist)

    def _stage(self, st):
        m = self.step.model
        return batching.stage_batch(self.batch_of(st), self.step.device, m.num_relation + 1, m.normalized_gnn,
                                    m.norm_rel, nfacts=st.nfacts)

    def run(self, st):
        """The model part of the captured serving step -> (db, loss, pred, pred_dist)."""
        db = self._stage(st)
        loss, pred, pred_dist, _ = self.step.model(db)
        return db, loss, pred, pred_dist

    def train_forward(self, st):
        """The model's training forward over the static buffers ``st`` -> (db, loss, pred, pred_dist)."""
        m = self.step.model
        db = self._stage(st)
        live = autograd_path.LiveBatch(db, st.heads, st.tails, st.weight_list, st.nfacts)
        core = autograd_path.rearev_core if self.rearev else autograd_path.nsm_core
        loss, pred, pred_dist = core(m, live, autograd_path._stage(m, live))
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

    # -- the model's part of an epoch (GraphedTrainStep.start_epoch, GraphedStep.start_eval) -------------------------
    def epoch_refusal(self, split, training):
        """Why ``split`` (a ``loader.DeviceSplit``) does not hold this model family's batches (a message), or None;
        worded for the training epoch with ``training``, else for the evaluation epoch."""
        if split.graft:
            if training:
                return "train_epoch takes a ReaRev / NSM split; this DeviceSplit holds GraftNet's graft lists"
            return "a ReaRev / NSM model evaluates a kb split; this DeviceSplit holds GraftNet's graft lists"
        return None

    @staticmethod
    def epoch_shapes(plan):
        """The graph shape of every step of ``plan``: (B, fact capacity)."""
        return list(zip(plan.B.tolist(), plan.capacity.tolist()))

    def epoch_key(self, split, shape):
        """The shape part of the capture key of an epoch step of ``shape`` (:meth:`epoch_shapes`) over ``split``."""
        return self._shape_key(shape[0], split.N, shape[1], int(split._res["q_input"].shape[1]), split.index_dtype)

    def epoch_inputs(self, key):
        """The static buffers of an epoch graph: :meth:`static_inputs`, plus the head's outputs."""
        st = self.static_inputs(key)
        B, dev = key[0], self.step.device
        st.ids, st.rows, st.kept = (torch.zeros(B, dtype=torch.int64, device=dev) for _ in range(3))
        st.kept_total = torch.zeros(1, dtype=torch.int64, device=dev)
        st.status = torch.zeros(1, dtype=torch.int32, device=dev)
        return st

    def epoch_begin(self, ep, st):
        """The model's head kernels after gr_epoch_step_begin (none for ReaRev / NSM)."""

    def epoch_assemble(self, ep, st, seed):
        """The model's part of the batch assembly after the kb facts' -> its status word (None for ReaRev / NSM)."""
        return None

    @staticmethod
    def epoch_words(st, asm, model_asm, status):
        """The step's words of ``EpochRun.status`` from the assembly word, :meth:`epoch_assemble`'s and the status
        word of :meth:`GraphedTrainStep._run`: assembly, CSR."""
        return [asm, status]


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

    def model_key(self):
        """``pagerank_lambda`` and ``fact_scale``: Python scalars the training forward bakes into a graph."""
        layer = self.step.model.reasoning
        return float(layer.pagerank_lambda), float(layer.fact_scale)

    def refusal(self, Q):
        """Why the eager training forward would leave the kernels (a message), or None.  GraftNet's forward takes the
        kernel path or the per-fact torch ops as a whole (``autograd_path._fact_kernels``); its question encoder has no
        kernel path in training, so Q does not matter."""
        D = self.step.model.entity_dim
        if not autograd_path.USE_KERNELS:
            return "autograd_path.USE_KERNELS is off: the training forward would run its torch restatement"
        if not autograd_path._fact_kernels(self.step.device, D):
            return ("_fact_kernels is false: entity_dim %d is outside the GraftNet training kernels (%s)"
                    % (D, ops.fact_train_ok.__doc__.split(": ", 1)[1].rstrip(".")))
        return None

    def static_inputs(self, key):
        st = super().static_inputs(key)
        B, gcap, max_fact = key[0], key[5], key[6]
        dev = self.step.device
        for name in self.LIST_NAMES:
            setattr(st, name, torch.zeros(gcap, dtype=torch.int64, device=dev))
        st.graft_live = torch.zeros(2, dtype=torch.int32, device=dev)
        st.kb_fact_rel = torch.zeros(B, max_fact, dtype=torch.int64, device=dev)
        return st

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

    @staticmethod
    def batch_of(st):
        """The 9-tuple over the static buffers ``st``."""
        return (st.local_entity, st.query_entities,
                (st.heads, st.rels, st.tails, None, None, st.weight_list, st.weight_rel_list),
                ((st.e2f_b, st.e2f_f, st.e2f_e, None), (st.f2e_b, st.f2e_e, st.f2e_f, None)),
                st.q_input, st.kb_fact_rel, st.seed_dist, None, st.answer_dist)

    def run(self, st):
        m = self.step.model
        db = batching.stage_graft_batch(self.batch_of(st), self.step.device, m.num_relation + 1, m.normalized_gnn,
                                        m.norm_rel, nfacts=st.nfacts, graft_live=st.graft_live)
        with torch.no_grad():        # the status words are read by GraphedStep after the step, not inside the capture
            loss, pred, pred_dist, _ = m._forward_infer(db, check_status=False)
        return db, loss, pred, pred_dist

    def train_forward(self, st):
        m = self.step.model
        tup = self.batch_of(st)
        # the training forward stages without normalized_gnn (GraftNet does not read the kb weights)
        db = batching.stage_graft_batch(tup, self.step.device, m.num_relation + 1, False, m.norm_rel, nfacts=st.nfacts,
                                        graft_live=st.graft_live)
        loss, pred, pred_dist = autograd_path.graftnet_core(m, tup, autograd_path.graft_live_stage(db))
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

    def epoch_refusal(self, split, training):
        if not split.graft:
            if training:
                return ("GraphedGraftTrainStep.train_epoch takes a GraftNet split; this DeviceSplit holds no graft "
                        "lists (GraphedTrainStep.train_epoch covers ReaRev and NSM)")
            return "GraftNet evaluates a GraftNet split; this DeviceSplit holds no graft lists"
        return None

    @staticmethod
    def epoch_shapes(plan):
        """The graph shape of every step of ``plan``: (B, fact capacity, graft capacity)."""
        return list(zip(plan.B.tolist(), plan.capacity.tolist(), plan.graft_capacity.tolist()))

    def epoch_key(self, split, shape):
        return super().epoch_key(split, shape) + (shape[2], split.max_facts)

    def epoch_inputs(self, key):
        st = super().epoch_inputs(key)
        B, gcap, dev = key[0], key[5], self.step.device
        st.kept_g = torch.zeros(B, dtype=torch.int64, device=dev)
        st.graft_status = torch.zeros(1, dtype=torch.int32, device=dev)
        # the graft assembly writes the lists' values (all 1.0); GraftNet's training forward never reads them
        st.e2f_v, st.f2e_v = (torch.zeros(gcap, dtype=torch.float32, device=dev) for _ in range(2))
        return st

    def epoch_begin(self, ep, st):
        """gr_epoch_graft_begin: the graft kept counts and ``graft_live`` of the step's ids."""
        ops.epoch_graft_begin(st.ids, ep.graft_kept_table, ep.split._res["g_off"], st.e2f_b.numel(), st.kept_g,
                              st.graft_live, st.graft_status)

    def epoch_assemble(self, ep, st, seed):
        """The graft lists at their capacity and ``kb_fact_rel``, in the fact order of ``seed``."""
        out = ((st.e2f_b, st.e2f_f, st.e2f_e, st.e2f_v), (st.f2e_b, st.f2e_e, st.f2e_f, st.f2e_v), st.kb_fact_rel)
        _graft, _kfr, _order, gasm = ep.split.assemble_graft(st.ids, st.kept_g, seed, st.e2f_b.numel(),
                                                            ep.graft_n_total, out=out)
        return gasm

    @staticmethod
    def epoch_words(st, asm, model_asm, status):
        """-> assembly (kb, graft head and graft assembly), CSR (kb and graft CSR builds), graft staging."""
        csr, staging, graft_csr = status[0:1], status[1:2], status[2:3]
        return [asm | st.graft_status | model_asm, csr | graft_csr, staging]


def _layout_for(model):
    from .models import GraftNet
    return _GraftLayout if isinstance(model, GraftNet) else _KbLayout


# ---- capture ---------------------------------------------------------------------------------------------------------

def _evict(cache, max_graphs):
    """LRU eviction down to room for one more entry: its graph and every buffer it holds are released."""
    while len(cache) >= max_graphs:
        _k, old = cache.popitem(last=False)
        torch.cuda.synchronize()
        del old


def _warm_up(fn):
    """Run ``fn`` twice on a side stream (lazy init, allocator, caches, cuDNN plans), the device idle around it."""
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()


def _capture(fn, stream=None):
    """Capture ``fn`` into a CUDA graph on ``stream`` (None: torch's capture stream) -> (graph, what ``fn``
    returned).  Graphs that replay side by side are captured on streams of their own: cuBLAS keeps one workspace per
    (handle, stream), and a graph keeps the one of its capture stream."""
    g = torch.cuda.CUDAGraph()
    # no cyclic garbage collection during the capture: collecting a dropped step's graph there (its exec graph and
    # private pool are released) is a CUDA call that invalidates the capture
    gc_on = gc.isenabled()
    gc.disable()
    try:
        with torch.cuda.graph(g, stream=stream):
            outs = fn()
    finally:
        if gc_on:
            gc.enable()
    return g, outs


def _buffers_like(st, make):
    """A buffer set holding ``make(t)`` for every tensor ``t`` of ``st`` (None stays None)."""
    out = _Captured()
    for name, t in vars(st).items():
        setattr(out, name, None if t is None else make(t))
    return out


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
        self._evals = {}              # (id(split), batch size) -> _EvalBuffers

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
        _evict(self._cache, self.max_graphs)
        st = self._layout.static_inputs(shape_key)
        self._fill(st, batch)
        _warm_up(lambda: self._run(st))
        g, outs = _capture(lambda: self._run(st))
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
            nwords = len(self._layout.status_words(db))
            pipe = _Captured()
            pipe.land = [_buffers_like(ent.st, torch.empty_like) for _ in range(2)]
            # pinned host staging of the inputs: pageable loader output (numpy, int64 / float64) is cast and copied
            # here by the host (memcpy speed), the DMA to the landing set then runs asynchronously
            pipe.stage = [_buffers_like(ent.st, lambda t: torch.empty(t.shape, dtype=t.dtype, pin_memory=True))
                          for _ in range(2)]
            pipe.out_dev = [dict(cand_idx=torch.empty_like(cand_idx), pred_dist=torch.empty_like(pred_dist),
                                 cand_count=torch.empty_like(cand_count), pred=torch.empty_like(pred),
                                 loss=torch.empty_like(loss),
                                 status=torch.empty(nwords, dtype=torch.int32, device=self.device))
                            for _ in range(2)]
            pipe.out_host = [{k: torch.empty(v.shape, dtype=v.dtype, pin_memory=True) for k, v in od.items()}
                             for od in pipe.out_dev]
            pipe.land_free, pipe.done, pipe.h2d_done = [None, None], [None, None], [None, None]
            pipe.ents = None                         # device and pinned candidate entity ids, for DeviceSplit batches
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
        le = batch[0]
        on_device = isinstance(le, torch.Tensor) and le.is_cuda     # a loader.DeviceSplit batch
        if on_device:
            cs.wait_stream(cur)                      # the batch was assembled on the current stream
        elif self._layout.needs_staging(batch):
            if pipe.h2d_done[slot] is not None:
                pipe.h2d_done[slot].synchronize()    # the previous DMA out of this staging set has finished
            src = self._layout.stage_host(pipe.stage[slot], batch)
        with torch.cuda.stream(cs):
            self._fill(land, src)
            h2d_done = torch.cuda.Event()
            h2d_done.record(cs)
        pipe.h2d_done[slot] = h2d_done
        cur.wait_event(h2d_done)
        for name, t in vars(land).items():           # landing set -> the graph's static inputs (D2D, ~10 us)
            if t is not None:
                getattr(ent.st, name).copy_(t, non_blocking=True)
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
        ents = None
        if on_device:                                # the candidates' entity ids, gathered here instead of on the host
            if pipe.ents is None:
                pipe.ents = [(torch.empty_like(db.local_entity),
                              torch.empty(db.local_entity.shape, dtype=torch.int64, pin_memory=True)) for _ in range(2)]
            ents = pipe.ents[slot]
            torch.gather(db.local_entity, 1, cand_idx.long(), out=ents[0])
        out_ready = torch.cuda.Event()
        out_ready.record(cur)
        ds = self._d2h_stream
        ds.wait_event(out_ready)
        with torch.cuda.stream(ds):
            for k, v in od.items():
                pipe.out_host[slot][k].copy_(v, non_blocking=True)
            if ents is not None:
                ents[1].copy_(ents[0], non_blocking=True)
            pipe.done[slot] = torch.cuda.Event()
            pipe.done[slot].record(ds)
        db.h2d_bytes = self._h2d_bytes
        self.model.last_batch = db
        t = Ticket()
        t.slot, t.done, t.ent = slot, pipe.done[slot], ent
        if on_device:
            t.local_entity_host, t.cand_ent_host = None, ents[1]
        else:
            t.local_entity_host = le.cpu().numpy() if isinstance(le, torch.Tensor) else np.asarray(le)
            t.cand_ent_host = None
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
        ents = None if ticket.cand_ent_host is None else ticket.cand_ent_host.numpy()
        res = []
        for b, c in enumerate(counts.tolist()):
            ix = idx_h[b, :c].astype(np.int64)
            ent = le[b, ix].astype(np.int64) if ents is None else ents[b, :c].astype(np.int64)
            res.append(Retrieved(ix, ent, dist_h[b, ix]))
        nbytes = sum(v.numel() * v.element_size() for v in h.values())
        if ents is not None:
            nbytes += ents.nbytes
        return res, nbytes, float(h["loss"]), h["pred"].numpy().copy()

    def retrieve(self, out):
        """Ordered candidate lists of a :class:`StepOutput` (one D2H), like evaluate.retrieve."""
        from .evaluate import read_ranked
        self._check(out.db)
        return read_ranked(out.pred_dist, out.db, out.cand_idx, out.cand_count)

    # -- a whole evaluation ------------------------------------------------------------------------------------------
    def evaluate_split(self, split, batch_size):
        """One :meth:`start_eval` and one read: -> :meth:`EvalRun.result`.  Raises :meth:`EvalRun.check`'s errors
        when a batch was malformed."""
        run = self.start_eval(split, batch_size)
        out = run.result()
        run.check()
        return out

    def start_eval(self, split, batch_size, path_targets=None):
        """Start an evaluation of the whole split ``split`` (a ``loader.DeviceSplit``) and return its :class:`EvalRun`
        without waiting for the device.

        As ``evaluate.Evaluator.evaluate`` over the split: ``model.eval()``, ``split.reset_batches(is_sequential=True)``,
        then every batch of ``batch_size`` questions in order, the last one short when ``num_data % batch_size != 0``,
        each assembled as ``split.get_batch(it, batch_size, 0.0)`` assembles it (with ``shuffle``, from a fact-order
        seed drawn in the graph from torch's CUDA generator and recorded in ``EvalRun.seeds``), run through the
        serving step of :meth:`__call__` and ranked, and its questions scored against the split's answer lists
        (``DeviceSplit.answer_table``) as ``evaluate.f1_and_hits`` scores them (gr_eval_step_record).  Each step is
        one graph replay: gr_epoch_step_begin and the assembly from a device cursor (GraftNet: also
        gr_epoch_graft_begin and the graft assembly), the forward, the ranking and the records.  The host picks each
        step's graph, one per (B, fact capacity) and for GraftNet per graft capacity too, from :func:`epoch_plan`;
        the missing ones are captured before the first replay (the LRU grows to hold them all).  Their key holds the
        shapes, ``model_key``, ``eps``, the pad id and the ``data_ptr`` of every parameter but not its version: the
        graphs format the weights they read on each replay (``ops.graph_private_weights``), so they stay valid across
        in-place ``optimizer.step()`` and ``load_state_dict``.  Once the graphs exist nothing here waits on the device.
        Afterwards ``split.loader.sample_ids`` is the last batch's.

        ``path_targets``: an int T >= 1 makes each step's graph also compute the retrieved shortest-path node sets of
        its questions (gr_eval_step_paths, after the ranking): the BFS from each of the question's seeds (its local
        indices with ``query_entities != 0``, ascending, at most ``DeviceSplit.max_seeds()``) and each of its first
        ``min(count, T)`` ranked candidates over the step's kb CSR, the on-path nodes compacted into node records sized
        like the candidate records; :meth:`EvalRun.paths` reads them.  T is part of the graph key; without it the
        graphs are those of an evaluation without paths.

        Refused (``ValueError``): anything but a CUDA ``DeviceSplit`` on the model's device of the model's family,
        ``batch_size <= 0``, a ``q_type`` other than ``"seq"``, fact weights (``normalized_gnn`` / ``norm_rel``) over
        a ``weights="none"`` split, then a ``path_targets`` that is not a positive int or whose BFS workspace
        (B * (max_seeds + T) * N for the largest batch) overflows int32 indexing, and answers that are not
        integers."""
        why = self._eval_refusal(split, batch_size, path_targets)
        if why is not None:
            raise ValueError(why)
        return _run_epochs([self._eval_job(split, batch_size, path_targets)])[0]

    def _eval_refusal(self, split, batch_size, path_targets=None):
        """The ``ValueError`` message :meth:`start_eval` refuses ``(split, batch_size, path_targets)`` with, or
        None."""
        why = _split_refusal(self, split, batch_size, False)
        if why is None and path_targets is not None:
            why = paths_refusal(split, batch_size, path_targets)
        return None if why is None else "start_eval: " + why

    def _eval_job(self, split, batch_size, path_targets=None, member=None):
        """The :class:`_EpochJob` of :meth:`start_eval` (for the sweep member ``member``)."""
        job = _EpochJob(split, member)
        T = None if path_targets is None else int(path_targets)

        def start():
            job.answers = split.answer_table()
            job.plan, job.order, job.batches = _plan_epoch(split, batch_size, False, 0.0, job.rng())

        def begin():
            self.model.eval()
            job.ep = _buffers_for(self._evals, split, batch_size, lambda ep: ep.pad_id != self.num_entity,
                                  lambda: _EvalBuffers(split, batch_size, self.num_entity))
            _upload_order(job.ep, job.order)
            if T is not None and T not in job.ep.paths:
                job.ep.paths[T] = _EvalPaths(split.device, job.ep.num_data, split.max_seeds(), T, job.ep.capacity)

        def capture():
            ep = job.ep
            entries = _epoch_graphs(self, job.plan, lambda shape: self._eval_key(ep, shape, member, T),
                                    lambda shape, s0: self._eval_capture(ep, shape, s0, job.answers, member, T))
            ep.cursor.zero_()
            ep.blob.zero_()
            if T is not None:
                ep.paths[T].blob.zero_()
            return entries

        def finish():
            ep = job.ep
            job.set_sample_ids()
            paths = None
            if T is not None:
                pp = ep.paths[T]
                c, order = split.seed_counts(), job.order
                known = (order >= 0) & (order < c.size)          # an id out of range is check()'s to report
                seeds = np.where(known, c[np.where(known, order, 0)] if c.size else 0, 0)
                paths = (pp.blob.clone(), pp.S, pp.T, pp.capacity, seeds)
            return EvalRun(ep.blob.clone(), ep.cand.clone(), None if ep.seeds is None else ep.seeds.clone(),
                           ep.num_data, ep.order.clone(), paths)
        job.start, job.begin, job.capture, job.finish = start, begin, capture, finish
        return job

    def _eval_key(self, ep, shape, member=None, T=None):
        return (("eval", id(ep)) + self._layout.epoch_key(ep.split, shape) + self._layout.model_key()
                + (float(self.eps), int(self.num_entity)) + tuple(p.data_ptr() for p in self.model.parameters())
                + _rel_text_ptrs(self.model) + _member_key(member) + (() if T is None else ("paths", T)))

    def _eval_capture(self, ep, shape, s0, answers, member=None, T=None):
        """Capture the evaluation graph of ``shape``; ``s0``: a step with that shape, the one the warm-up assembles;
        ``T``: the path targets (None: no node sets)."""
        def body(st, cursor):
            # the serving step of _run, its status words (CSR[, graft staging, graft CSR]) in one tensor
            return _epoch_step(self, ep, st, cursor, self._run,
                               lambda outs: torch.cat(self._layout.status_words(outs[0])))
        with torch.no_grad():
            st = _warm_up_epoch_step(self, ep, shape, s0, body)
        a_off, a_ids = answers

        def captured():
            outs, seed, words = body(st, ep.cursor)
            db, _loss, _pred, pred_dist, cand_idx, cand_count, _total = outs
            if len(words) > 2:                   # gr_eval_step_record ORs the first two words (assembly, CSR)
                ep.status[3:4].bitwise_or_(words[2])
            if T is not None:                    # before gr_eval_step_record, which moves the cursor
                pp = ep.paths[T]
                ops.eval_step_paths(ep.cursor, ep.batch_size, ep.steps, ep.num_data, db.graph,
                                    db.query_entities.contiguous(), cand_idx, cand_count, pp.S, T, pp.node_off,
                                    pp.node_count, pp.pair_dist, pp.nodes, pp.node_total, ep.status[2:3])
            ops.eval_step_record(ep.cursor, ep.batch_size, ep.steps, st.ids, db.local_entity, pred_dist, cand_idx,
                                 cand_count, a_off, a_ids, seed, words[0], words[1], ep.metrics, ep.cases, ep.counts,
                                 ep.cand_off, ep.cand, ep.cand_total, ep.seeds, ep.status[:3])
            return outs
        with torch.no_grad(), ops.graph_private_weights() as private:
            g, outs = _capture(captured, _capture_stream(member))
        ent = _Captured()
        ent.st, ent.g, ent.outs, ent.epoch, ent.pipe = st, g, outs, ep, None
        ent.weights = private                    # the graph formats the weights into these on every replay
        ent.planes = live_plane_buffers()        # as GraphedStep._entry: the operand planes the graph relies on
        ent.draws = _member_draws(member)        # its generator and scratch (and the id in the key) stay alive
        self._cache[self._eval_key(ep, shape, member, T)] = ent


# ---- training ------------------------------------------------------------------------------------------------------

class TrainStepOutput(tuple):
    """``(loss, pred, pred_dist, h1, f1)`` of one :meth:`GraphedTrainStep.step`, all device tensors (views of the
    graph's static outputs, valid until the next step).  ``status`` holds the device int32 status words of the batch's
    staging (ReaRev, NSM: the CSR build's; GraftNet: also the graft staging's); :meth:`check` reads them back and
    raises, with the messages of the input layout that produced them, when a fact list was malformed.  ``grad_norm``:
    the total gradient norm before clipping (device fp32 scalar) of a step with ``max_norm``, else None."""

    def __new__(cls, loss, pred, pred_dist, h1, f1, status, raise_for=_KbLayout.raise_for, grad_norm=None):
        out = super().__new__(cls, (loss, pred, pred_dist, h1, f1))
        out.status, out._raise_for, out.grad_norm = status, raise_for, grad_norm
        return out

    def check(self):
        self._raise_for(self.status.tolist())


class EpochPlan:
    """The host arithmetic of one epoch over a resident split (:func:`epoch_plan`): per step ``B`` (questions),
    ``F`` (live facts: kept facts + self-loops), ``K`` (kept facts) and ``capacity`` (``fact_capacity(F)``), int64
    numpy arrays of ``steps`` entries, and ``starts``, the step's first position in the order.  With graft counts
    also ``G`` (kept graft entries) and ``graft_capacity`` (``fact_capacity(G)``), else None."""
    __slots__ = ("steps", "B", "F", "K", "capacity", "starts", "G", "graft_capacity")


def epoch_plan(order, stored, ents, batch_size, fact_dropout=0.0, graft=None):
    """Per-step counts of an epoch that takes the questions ``order`` (ids, in batch order) ``batch_size`` at a time,
    the last batch short when ``len(order) % batch_size != 0``: what ``DeviceSplit.get_batch(it, batch_size,
    fact_dropout)`` computes on the host for each step, from the split's per-question stored fact counts ``stored``
    and self-loop counts ``ents`` (zeros without ``use_self_loop``), and for GraftNet its stored graft entries per
    question ``graft``.  A question keeps ``loader.kept_counts`` of its stored facts and of its graft entries.  An id
    outside [0, len(stored)) counts as an empty question, as the device assembly counts it."""
    from .loader import kept_counts
    order = np.asarray(order, dtype=np.int64).reshape(-1)
    stored, ents = np.asarray(stored, dtype=np.int64), np.asarray(ents, dtype=np.int64)
    n, bs = order.size, int(batch_size)
    plan = EpochPlan()
    plan.steps = (n + bs - 1) // bs
    plan.starts = np.arange(0, n, bs, dtype=np.int64)
    ok = (order >= 0) & (order < stored.size)
    q = np.where(ok, order, 0)

    def per_step(counts, keep):
        """The sums over each step of ``counts`` per question of the order (their kept counts with ``keep``)."""
        counts = np.asarray(counts, dtype=np.int64)
        c = counts[q] if counts.size else np.zeros(n, np.int64)
        c = np.where(ok, kept_counts(c, fact_dropout) if keep else c, 0)
        return np.add.reduceat(c, plan.starts).astype(np.int64) if n else np.zeros(0, dtype=np.int64)
    plan.K = per_step(stored, True)
    plan.F = plan.K + per_step(ents, False)
    plan.B = np.minimum(bs, n - plan.starts).astype(np.int64)
    plan.capacity = np.array([fact_capacity(f) for f in plan.F.tolist()], dtype=np.int64)
    plan.G = plan.graft_capacity = None
    if graft is not None:
        plan.G = per_step(graft, True)
        plan.graft_capacity = np.array([fact_capacity(g) for g in plan.G.tolist()], dtype=np.int64)
    return plan


class EpochRun:
    """One epoch started by :meth:`GraphedTrainStep.start_epoch`: device tensors, valid once the current stream reaches
    them.  ``losses`` / ``grad_norms`` fp32 [steps] (``grad_norms`` None without ``max_norm``), ``h1`` / ``f1`` fp32
    [num_data] in batch order, ``seeds`` int64 [steps] (the fact-order seed of each step; None without ``shuffle``),
    ``status`` int32 [2]: the OR of every step's batch-assembly status word and of its CSR build's; for GraftNet int32
    [3]: the assembly word (kb and graft sides), the CSR word (kb and graft CSR builds) and the graft staging word.
    :meth:`result` reads them back in one copy; :meth:`check` raises for a nonzero status."""

    def __init__(self, losses, grad_norms, h1, f1, seeds, status):
        self.losses, self.grad_norms, self.h1, self.f1, self.seeds, self.status = \
            losses, grad_norms, h1, f1, seeds, status
        self._words = None

    def result(self):
        """-> ``(np.mean(losses), [0, 0], h1_list_all, f1_list_all)`` as the reference's ``train_epoch`` returns them
        (Python floats in the lists), read back in one device-to-host copy."""
        n, m = self.losses.numel(), self.h1.numel()
        host = torch.cat([self.losses, self.h1, self.f1, self.status.view(torch.float32)]).cpu()
        self._words = host[n + 2 * m:].view(torch.int32).tolist()
        return np.mean(host[:n].tolist()), [0, 0], host[n:n + m].tolist(), host[n + m:n + 2 * m].tolist()

    def check(self):
        """Raise ``DeviceSplit.check``'s message when an assembly flagged an id out of range or an overflow, else (for
        GraftNet) ``GraftGraph``'s when the graft staging rejected a list, else ``TrainStepOutput.check``'s when a CSR
        build flagged ids outside the batch (reads the status unless :meth:`result` has)."""
        words = self._words if self._words is not None else self.status.tolist()
        _raise_epoch_status(words[0], words[1], words[2] if len(words) > 2 else 0)


# ---- the epoch driver: what a training epoch and an evaluation epoch share -----------------------------------------

class _SplitBuffers:
    """The device state the epoch graphs of one (split, batch size) read: the cursor, the question order, the
    kept-count tables (None: every stored fact), the fact-order seed records with ``shuffle`` and the sizes of the
    fact-order workspaces.  Fixed addresses: the graphs hold them."""

    def __init__(self, split, batch_size):
        dev = split.device
        self.split, self.batch_size = split, int(batch_size)
        self.num_data = int(split.num_data)
        self.steps = (self.num_data + self.batch_size - 1) // self.batch_size
        i64 = dict(dtype=torch.int64, device=dev)
        self.cursor = torch.zeros(1, **i64)
        self.order = torch.zeros(self.num_data, **i64)
        self.kept_table = self.graft_kept_table = None
        self.seeds = torch.zeros(self.steps, **i64) if split.shuffle else None
        # the fact-order workspaces of any batch
        self.n_total = _largest(split._stored, self.batch_size)
        self.graft_n_total = _largest(split._graft_count, self.batch_size) if split.graft else None


class _EpochBuffers(_SplitBuffers):
    """:class:`_SplitBuffers` of a training epoch, with the kept-count tables of ``shuffle`` (GraftNet: also the
    graft entries'), the records and the per-step Adam scalars."""

    def __init__(self, split, batch_size, max_norm):
        super().__init__(split, batch_size)
        dev = split.device
        f32 = dict(dtype=torch.float32, device=dev)
        if split.shuffle:
            self.kept_table = torch.zeros(max(split.num_q, 1), dtype=torch.int64, device=dev)
            if split.graft:
                self.graft_kept_table = torch.zeros(max(split.num_q, 1), dtype=torch.int64, device=dev)
        self.losses = torch.zeros(self.steps, **f32)
        self.grad_norms = torch.zeros(self.steps, **f32) if max_norm is not None else None
        self.h1 = torch.zeros(self.num_data, **f32)
        self.f1 = torch.zeros(self.num_data, **f32)
        self.status = torch.zeros(3 if split.graft else 2, dtype=torch.int32, device=dev)
        self.adam = None                 # fp32 [steps, T, 8], made at the first capture (T is known then)


def _largest(counts, batch_size):
    """The stored entries of the ``batch_size`` largest questions of ``counts``: a bound on any batch's."""
    return int(np.sort(counts)[-batch_size:].sum()) if counts.size else 0


def _buffers_for(cache, split, batch_size, stale, make):
    """The buffers ``cache`` holds for (``split``, ``batch_size``), replaced by ``make()`` when there are none, when
    they belong to another split or question count, or when ``stale(buffers)``."""
    k = (id(split), int(batch_size))
    ep = cache.get(k)
    if ep is None or ep.split is not split or ep.num_data != split.num_data or stale(ep):
        ep = cache[k] = make()
    return ep


def _rel_text_ptrs(model):
    """The ``data_ptr`` of the model's relation-text features (``rel_features`` / ``rel_features_inv``) it has."""
    return tuple(t.data_ptr() for t in (getattr(model, "rel_features", None), getattr(model, "rel_features_inv", None))
                 if isinstance(t, torch.Tensor))


def _split_refusal(step, split, batch_size, training, more=None):
    """Why ``step`` runs no epoch (training with ``training``, else evaluation) of ``batch_size`` questions over
    ``split`` (a message), or None.  In this order: anything but a ``loader.DeviceSplit`` of the model's family on its
    device, a ``batch_size`` that is not a positive int, ``more()`` (the caller's own checks -> a message or None),
    a ``q_type`` other than ``"seq"``, fact weights (``normalized_gnn`` / ``norm_rel``) over a ``weights="none"``
    split."""
    from .loader import DeviceSplit, same_device
    if not isinstance(split, DeviceSplit):
        return ("train_epoch takes a loader.DeviceSplit, got %s" if training
                else "the split must be a loader.DeviceSplit, got %s") % type(split).__name__
    why = step._layout.epoch_refusal(split, training)
    if why is not None:
        return why
    if not same_device(split.device, step.device):
        return "the split lives on %s, the model on %s" % (split.device, step.device)
    if isinstance(batch_size, bool) or not isinstance(batch_size, (int, np.integer)) or batch_size <= 0:
        return "batch_size must be a positive int, got %r" % (batch_size,)
    why = None if more is None else more()
    if why is not None:
        return why
    if getattr(split.loader, "q_type", "seq") != "seq":
        return "q_type must be 'seq', got %r" % (split.loader.q_type,)
    m = step.model
    if (m.normalized_gnn or m.norm_rel) and split.weights != "arrays":
        return "normalized_gnn / norm_rel need fact weights: the split was built with weights='none'"
    return None


@contextlib.contextmanager
def _numpy_random(rng):
    """``rng`` (a ``np.random.RandomState``) as the global ``np.random`` stream inside the block: the global state is
    set to ``rng``'s on entry; on exit ``rng`` takes the state the block left and the global state is put back.
    ``rng`` None: the global stream itself."""
    if rng is None:
        yield
        return
    saved = np.random.get_state()
    np.random.set_state(rng.get_state())
    try:
        yield
    finally:
        rng.set_state(np.random.get_state())
        np.random.set_state(saved)


def _plan_epoch(split, batch_size, training, fact_dropout, rng=None):
    """The host side of an epoch's start, before anything reaches the device: ``split.reset_batches`` (the loader's
    ``np.random`` order with ``training``, its stored order without; a sweep member's ``rng`` stands in for
    ``np.random`` there), the :func:`epoch_plan` of that order with ``fact_dropout`` and the refusal of a batch that
    overflows the split's int32 indices -> (the plan, the order as int64, the loader's ``batches``)."""
    with _numpy_random(rng):
        split.reset_batches(is_sequential=not training)
    L = split.loader
    order = np.asarray(L.batches[:L.num_data], dtype=np.int64).reshape(-1)
    plan = epoch_plan(order, split._stored, split._ents, batch_size, fact_dropout,
                      split._graft_count if split.graft else None)
    if split.index_dtype == torch.int32 and plan.steps and (
            int(plan.B.max()) * split.N > _INT32_MAX or int(plan.F.max()) > _INT32_MAX):
        raise ValueError(("train_epoch: " if training else "start_eval: ")
                         + "a batch overflows int32 indices; use index_dtype=torch.int64")
    return plan, order, L.batches


def _upload_order(ep, order):
    ep.order.copy_(torch.from_numpy(order), non_blocking=True)


def _epoch_graphs(step, plan, key, capture):
    """The graph of every step of ``plan`` from ``step``'s LRU (a list), one per step shape
    (``epoch_shapes``): ``capture(shape, s0)`` captures a missing one under ``key(shape)``, ``s0`` being the first step
    of that shape.  The LRU grows to hold them all.  The keys are read again once every graph exists: a training
    capture can create Adam state, which its keys hold."""
    steps = step._layout.epoch_shapes(plan)
    shapes = {}
    for s, shape in enumerate(steps):
        shapes.setdefault(shape, s)
    step.max_graphs = max(step.max_graphs, len(shapes))
    for shape, s in shapes.items():
        k = key(shape)
        if k in step._cache:
            step._cache.move_to_end(k)
        else:
            capture(shape, s)
    ents = {shape: step._cache[key(shape)] for shape in shapes}
    return [ents[shape] for shape in steps]


def _epoch_step(step, ep, st, cursor, run, status):
    """One step of an epoch graph over the static buffers ``st``: gr_epoch_step_begin from the device ``cursor`` into
    ``ep.order``, the model's head kernels, the batch assembly into ``st`` (the fact-order seed drawn from torch's
    CUDA generator with ``shuffle``), then ``outs = run(st)`` -> (outs, seed or None, the step's status words:
    ``epoch_words`` with ``status(outs)``, the CSR / staging words)."""
    split, layout = ep.split, step._layout
    r, cap = split._res, st.heads.numel()
    ops.epoch_step_begin(cursor, ep.order, ep.batch_size, ep.kept_table, r["q_off"], r["q_ents"],
                         split.use_self_loop, cap, st.ids, st.rows, st.kept, st.nfacts, st.kept_total, st.status)
    layout.epoch_begin(ep, st)
    seed = torch.randint(0, 2 ** 62, (1,), device=step.device) if split.shuffle else None
    _rows, _kb, _order, asm = split.assemble(st.ids, st.kept, seed, cap, cap, ep.n_total, rows=st.rows, out=st,
                                             nfacts=st.nfacts)
    asm = st.status | asm
    model_asm = layout.epoch_assemble(ep, st, seed)
    outs = run(st)
    return outs, seed, layout.epoch_words(st, asm, model_asm, status(outs))


def _warm_up_epoch_step(step, ep, shape, s0, body):
    """Make room in ``step``'s LRU for the epoch graph of ``shape`` and warm up its step: ``body(st, cursor)`` over
    new static buffers ``st`` on a cursor at step ``s0`` (the real cursor does not move), torch's CUDA generator
    left where it was -> ``st``."""
    _evict(step._cache, step.max_graphs)
    dev = step.device
    st = step._layout.epoch_inputs(step._layout.epoch_key(ep.split, shape))
    rng = torch.cuda.get_rng_state(dev)
    warm_cursor = torch.full((1,), s0, dtype=torch.int64, device=dev)
    _warm_up(lambda: body(st, warm_cursor))
    torch.cuda.set_rng_state(rng, dev)
    return st


class _EpochJob:
    """One epoch of one step over ``split``, from its refusal to its run, in the phases :func:`_run_epochs` calls:
    ``start()`` (host only: the order and the plan, which may still refuse the epoch; sets ``plan``, ``order`` and
    ``batches``), ``begin()`` (the buffers and the uploads: sets ``ep``), ``capture()`` (the graphs the epoch needs and
    whatever must precede its first replay -> the graph of every step) and, after the replays, ``finish()`` -> the
    run.  ``member``: the :class:`Sweep` member it runs for, None for a solo epoch."""

    def __init__(self, split, member):
        self.split, self.member = split, member
        self.ep = self.plan = self.order = self.batches = None
        self.start = self.begin = self.capture = self.finish = None

    def rng(self):
        return None if self.member is None else self.member.rng

    def set_sample_ids(self):
        """``sample_ids`` of the split's loader := the epoch's last batch (its ids in the order the epoch drew)."""
        if self.plan.steps:
            L, s0 = self.ep.split.loader, int(self.plan.starts[-1])
            L.sample_ids = self.batches[s0:min(s0 + self.ep.batch_size, L.num_data)]


_NO_BATCHES = object()


def _start_all(jobs):
    """Every job's ``start``.  When one refuses, the members' ``RandomState`` objects and their loaders' ``batches``
    are put back as they were, so a refused sweep leaves nothing drawn (a solo job has no member to put back)."""
    saved = [(j.member.rng.get_state(), j.split.loader, vars(j.split.loader).get("batches", _NO_BATCHES))
             for j in jobs if j.member is not None]
    try:
        for j in jobs:
            j.start()
    except BaseException:
        for (state, L, batches), j in zip(saved, [j for j in jobs if j.member is not None]):
            j.member.rng.set_state(state)
            if batches is _NO_BATCHES:
                vars(L).pop("batches", None)
            else:
                L.batches = batches
        raise


def replay_schedule(steps):
    """The replay order of epochs of ``steps`` steps each (one count per job): [(job, step)], step s of every job that
    has one before step s + 1 of any, jobs in their order within a step."""
    steps = [int(n) for n in steps]
    return [(k, s) for s in range(max(steps, default=0)) for k, n in enumerate(steps) if s < n]


def _run_epochs(jobs):
    """Run the epochs ``jobs`` (:class:`_EpochJob`, at most one per step) -> their runs.  Every job's ``start`` (the
    host side, where an epoch can still be refused: :func:`_start_all`), then every job's ``begin``, then every job's
    ``capture``, so that no capture (and none of its device-wide synchronisations) lands between replays; then the
    graphs in :func:`replay_schedule` order, each job's on its member's stream (a solo job's on the current stream),
    then ``finish`` of each job on the current stream, which waits on the members' streams first.  A member's work
    between the two waits (uploads, replays) goes to its own stream, and nothing waits on the device.  Because of
    the two waits, the epochs of one call overlap each other but not the work of an earlier or a later call."""
    _start_all(jobs)
    cur = torch.cuda.current_stream()
    streams = [cur if j.member is None else j.member.stream for j in jobs]
    for s in streams:
        if s != cur:
            s.wait_stream(cur)
    for j, s in zip(jobs, streams):
        with torch.cuda.stream(s):
            j.begin()
    entries = []
    for j, s in zip(jobs, streams):
        with torch.cuda.stream(s), _member_scope(j.member):
            entries.append(j.capture())
    for k, i in replay_schedule([len(e) for e in entries]):
        with torch.cuda.stream(streams[k]):
            entries[k][i].g.replay()
    for s in streams:
        if s != cur:
            cur.wait_stream(s)
    return [j.finish() for j in jobs]


def _member_key(member):
    """The part of an epoch graph's key that names where it draws its random numbers and keeps its scratch: nothing
    for torch's default generator and the shared scratch, the sweep member's :class:`_Draws` otherwise."""
    return () if member is None else ("member", id(member.draws))


def _member_draws(member):
    """What a member's graph holds for as long as it lives: its :class:`_Draws` (None for a solo graph)."""
    return None if member is None else member.draws


def _capture_stream(member):
    return None if member is None else member.draws.capture_stream


def _shared_scratch():
    """The scratch buffers the forwards keep per shape rather than per model, so that models of one shape share them:
    (owner, attribute) of each dict -- the reasoning layers' operand planes, the relation-feature planes and the
    aggregation's tile counter.  A graph writes them on every replay, so graphs that replay side by side need
    copies of their own (:func:`_member_scope`)."""
    from . import modules
    return ((modules._GraphLayerBase, "_plane_cache"), (modules.GraftLayer, "_plane_cache"), (ops.RelFeatures, "_buf"),
            (ops, "_TILE_COUNTER"))


@contextlib.contextmanager
def _member_scope(member):
    """A sweep member's captures: its generator as the graph-safe state of torch's default CUDA generator (each graph
    captured here registers it, so only this member's replays advance it) and its own copies of every
    :func:`_shared_scratch` dict, so that members replaying side by side never write the same buffer.  Nothing for
    None."""
    if member is None:
        yield
        return
    draws = member.draws
    gen = torch.cuda.default_generators[draws.device.index]
    shared = _shared_scratch()
    saved = gen.graphsafe_get_state(), [getattr(owner, name) for owner, name in shared]
    gen.graphsafe_set_state(draws.generator.graphsafe_get_state())
    for (owner, name), mine in zip(shared, draws.scratch):
        setattr(owner, name, mine)
    try:
        yield
    finally:
        for (owner, name), theirs in zip(shared, saved[1]):
            setattr(owner, name, theirs)
        gen.graphsafe_set_state(saved[0])


def _raise_epoch_status(asm, csr, staging):
    """Raise ``DeviceSplit.check``'s message for a nonzero assembly word, else ``GraftGraph``'s for a nonzero graft
    staging word, else the CSR build's for a nonzero CSR word."""
    from .loader import DeviceSplit
    DeviceSplit.raise_status(asm)
    ops.GraftGraph.raise_status(staging)
    if csr:
        _KbLayout.raise_for([csr])


class EvalRun:
    """One evaluation started by :meth:`GraphedStep.start_eval`: device copies of its records, valid once the current
    stream reaches them.  ``seeds``: int64 [steps], the fact-order seed of each step (None without ``shuffle``);
    ``order``: int64 [num_data], the question id of each position.  :meth:`result` and :meth:`records` read the
    records back; :meth:`info` formats the run's ``.info`` rows on the device; :meth:`paths` reads the shortest-path
    node sets of a run started with ``path_targets``; :meth:`check` raises for a nonzero status."""

    def __init__(self, blob, cand, seeds, num_data, order, paths=None):
        self.blob, self.cand, self.seeds, self.num_data, self.order = blob, cand, seeds, num_data, order
        self._paths = paths           # (blob, S, T, capacity, seed count of each position) or None
        self._words = None
        self._host = None

    def _read(self):
        """The per-question records and the status, read back in one copy (once)."""
        if self._host is None:
            self._host = _EvalBuffers.views(self.blob.cpu().numpy(), self.num_data)
            self._words = self._host["status"].tolist()
        return self._host

    def records(self):
        """-> ``(metrics, case)``: float64 [num_data, 5] (precision, recall, f1, hit, em as ``evaluate.f1_and_hits``
        returns them, ``em`` as a float) and the int8 case (0..3) of every question in batch order."""
        v = self._read()
        return v["metrics"], v["cases"]

    def result(self):
        """-> ``(precision, recall, f1, hit, em, case, retrieved)`` of every question in batch order: five float64
        numpy arrays with the values ``evaluate.f1_and_hits`` returns (``em`` as a float), the int8 case (0..3) and
        one :class:`evaluate.Retrieved` per question.  Reads the device twice at most: the per-question records and
        the status in one copy, then the candidates in use."""
        from .evaluate import Retrieved
        v = self._read()
        used = min(int(v["cand_total"][0]), self.cand.shape[0])
        cand = self.cand[:used].cpu().numpy() if used else np.zeros((0, 2), dtype=np.int64)
        ent, pair = cand[:, 0], cand[:, 1:].copy().view(np.int32)
        idx, prob = pair[:, 0].astype(np.int64), pair[:, 1].view(np.float32)
        retrieved = []
        for o, c in zip(v["cand_off"].tolist(), v["counts"].tolist()):
            o, c = (0, 0) if o + c > used else (o, c)          # cut: an overflow, which check() reports
            retrieved.append(Retrieved(idx[o:o + c], ent[o:o + c], prob[o:o + c]))
        m = v["metrics"]
        return m[:, 0].copy(), m[:, 1].copy(), m[:, 2].copy(), m[:, 3].copy(), m[:, 4].copy(), v["cases"].copy(), \
            retrieved

    def paths(self):
        """-> ``(node_sets, pair_dist)`` of a run started with ``path_targets=T``, one entry per question in batch
        order: the sorted list of local indices on a shortest path between one of the question's seeds and one of
        its first ``min(count, T)`` retrieved candidates, as ``evaluate.path_node_sets(db, retrieved, T)`` gives it,
        and the int32 [n_seeds, n_targets] hop distances of those pairs (-1: unreachable).  Calls :meth:`check`
        first.  Reads the device once more at most: the node records, after the records :meth:`result` reads."""
        if self._paths is None:
            raise ValueError("EvalRun.paths: the evaluation was started without path_targets")
        counts = self._read()["counts"]
        self.check()
        blob, S, T, capacity, seeds = self._paths
        v = _EvalPaths.views(blob.cpu().numpy(), self.num_data, S, T, capacity)
        return _EvalPaths.decode(v, np.minimum(seeds, S), np.minimum(counts, T))

    def info(self, tables, file=None):
        """The ``.info`` rows of the run, byte for byte what ``evaluate.Evaluator`` writes for these questions with
        ``json.dumps``: one row per question in batch order, formatted on the device from the records
        (gr_info_rows_size, gr_info_rows_write) with the question prefixes and entity names of ``tables`` (an
        ``evaluate.InfoTables`` of the split, from ``Evaluator.info_tables``).  Calls :meth:`check` first, so a
        malformed run raises its message and formats nothing.  Reads the total size back once, then copies the
        bytes once into pinned memory.  -> the bytes as a uint8 numpy array over that memory, or, with ``file`` (an
        open binary file), None after one ``file.write`` of them.  Raises ``RuntimeError`` when a candidate record
        falls outside the records, a question id outside the tables, or a candidate entity has no name."""
        self.check()
        n, dev = self.num_data, self.blob.device
        v = _EvalBuffers.views(self.blob, n)
        recs = (v["metrics"], v["cases"], v["counts"], v["cand_off"], v["cand_total"])
        row_off = torch.empty(n + 1, dtype=torch.int64, device=dev)
        summary = torch.empty(2, dtype=torch.int64, device=dev)
        ops.info_rows_size(*recs, v["status"], self.cand, self.order, tables, row_off, summary)
        total, flags = summary.tolist()
        if flags:
            raise RuntimeError("EvalRun.info: flags %d (2: a candidate record outside the records or a question id "
                               "outside the tables, 4: a candidate entity without a name)" % flags)
        out = torch.empty(max(total, 1), dtype=torch.uint8, device=dev)
        ops.info_rows_write(*recs, self.cand, self.order, tables, row_off, summary, out)
        host = torch.empty(total, dtype=torch.uint8, pin_memory=True)
        host.copy_(out[:total])
        data = host.numpy()
        if file is None:
            return data
        file.write(data)
        return None

    def check(self):
        """Raise ``DeviceSplit.check``'s message when an assembly flagged an id out of range or an overflow, else (for
        GraftNet) ``GraftGraph``'s when the graft staging rejected a list, else ``GraphedStep``'s when a CSR build
        flagged ids outside the batch, else when the candidate records overflowed, else when the path node records
        did (reads the status unless :meth:`result` or :meth:`records` has)."""
        words = self._words
        if words is None:
            words = _EvalBuffers.views(self.blob, self.num_data)["status"].tolist()
        asm, csr, records, staging = words
        _raise_epoch_status(asm, csr, staging)
        if records & 1:
            raise RuntimeError("EvalRun: more ranked candidates than the %d candidate records of the split"
                               % self.cand.shape[0])
        if records & 2:
            raise RuntimeError("EvalRun: more shortest-path nodes than the %d node records of the split"
                               % self._paths[3])


class _EvalBuffers(_SplitBuffers):
    """:class:`_SplitBuffers` of an evaluation (of one pad id; no kept tables: every stored fact), with the records
    (one byte buffer, so that one copy reads them: float64 [num_data, 5] metrics, int64 [num_data] candidate offsets,
    int64 candidate total, int32 [num_data] candidate counts, int32 [4] status words -- assembly, CSR, candidate
    records, GraftNet's graft staging -- and int8 [num_data] cases) and the candidate records (int64 [capacity, 2],
    see gr_eval_step_record)."""

    def __init__(self, split, batch_size, pad_id):
        super().__init__(split, batch_size)
        dev, n = split.device, self.num_data
        self.pad_id = int(pad_id)
        self.blob = torch.zeros(self.nbytes(n), dtype=torch.uint8, device=dev)
        for name, t in self.views(self.blob, n).items():
            setattr(self, name, t)
        from .loader import candidate_capacity
        self.capacity = candidate_capacity(split.loader.candidate_entities, pad_id)
        self.cand = torch.zeros(max(self.capacity, 1), 2, dtype=torch.int64, device=dev)
        self.paths = {}               # path targets T -> _EvalPaths

    @staticmethod
    def nbytes(n):
        return 53 * n + 24

    @staticmethod
    def views(blob, n):
        """The records of :class:`_EvalBuffers` as views of ``blob`` (a torch uint8 tensor or a numpy uint8 array)."""
        layout = (("metrics", 0, 40 * n, (n, 5), "float64"), ("cand_off", 40 * n, 8 * n, (n,), "int64"),
                  ("cand_total", 48 * n, 8, (1,), "int64"), ("counts", 48 * n + 8, 4 * n, (n,), "int32"),
                  ("status", 52 * n + 8, 16, (4,), "int32"), ("cases", 52 * n + 24, n, (n,), "int8"))
        if isinstance(blob, torch.Tensor):
            return {k: blob[o:o + b].view(getattr(torch, dt)).view(shape) for k, o, b, shape, dt in layout}
        return {k: blob[o:o + b].view(dt).reshape(shape) for k, o, b, shape, dt in layout}


class _EvalPaths:
    """The shortest-path records of an evaluation with ``path_targets=T`` (gr_eval_step_paths), one byte buffer so that
    one copy reads them: int64 [num_data] node offsets, the int64 node total, int32 [num_data] node counts, int32
    [num_data, S, T] pair distances (S: the split's ``max_seeds``) and the int32 [capacity] node records, each
    question's on-path local indices ascending at its offset."""

    def __init__(self, device, n, S, T, capacity):
        self.S, self.T, self.capacity = int(S), int(T), int(capacity)
        self.blob = torch.zeros(self.nbytes(n, S, T, capacity), dtype=torch.uint8, device=device)
        for name, t in self.views(self.blob, n, S, T, capacity).items():
            setattr(self, name, t)

    @staticmethod
    def nbytes(n, S, T, capacity):
        return 12 * n + 8 + 4 * n * S * T + 4 * capacity

    @staticmethod
    def views(blob, n, S, T, capacity):
        """The records of :class:`_EvalPaths` as views of ``blob`` (a torch uint8 tensor or a numpy uint8 array)."""
        pd = 12 * n + 8
        layout = (("node_off", 0, 8 * n, (n,), "int64"), ("node_total", 8 * n, 8, (1,), "int64"),
                  ("node_count", 8 * n + 8, 4 * n, (n,), "int32"), ("pair_dist", pd, 4 * n * S * T, (n, S, T), "int32"),
                  ("nodes", pd + 4 * n * S * T, 4 * capacity, (capacity,), "int32"))
        if isinstance(blob, torch.Tensor):
            return {k: blob[o:o + b].view(getattr(torch, dt)).view(shape) for k, o, b, shape, dt in layout}
        return {k: blob[o:o + b].view(dt).reshape(shape) for k, o, b, shape, dt in layout}

    @staticmethod
    def decode(v, n_seeds, n_targets):
        """Host views ``v`` of the records and the seed / target count of every position -> (node lists, pair
        distance blocks [n_seeds, n_targets])."""
        nodes, pair = v["nodes"], v["pair_dist"]
        sets = [nodes[o:o + c].tolist() for o, c in zip(v["node_off"].tolist(), v["node_count"].tolist())]
        blocks = [pair[p, :s, :t].copy() for p, (s, t) in enumerate(zip(np.asarray(n_seeds).tolist(),
                                                                         np.asarray(n_targets).tolist()))]
        return sets, blocks


def paths_refusal(split, batch_size, path_targets):
    """Why an evaluation of ``split`` in batches of ``batch_size`` refuses ``path_targets`` (a message), or None: a
    value that is not a positive int, or a BFS workspace (B * (``split.max_seeds()`` + T) * N, B the largest batch)
    past int32 indexing."""
    T = path_targets
    if isinstance(T, bool) or not isinstance(T, (int, np.integer)) or T <= 0:
        return "path_targets must be a positive int, got %r" % (T,)
    B = max(min(int(batch_size), int(split.num_data)), 1)
    cells = B * (split.max_seeds() + int(T)) * int(split.N)
    if cells > _INT32_MAX:
        return ("path_targets %d: the BFS workspace of a batch, B * (max_seeds + T) * N = %d * (%d + %d) * %d, "
                "overflows int32 indexing" % (T, B, split.max_seeds(), T, split.N))
    return None


def _release_autograd_history(model, params):
    """Drop the tensors with autograd history that a training forward leaves on the model's modules (``dist_history``,
    the question encoder's states), and the gradients of ``params``, so the next backward allocates them rather than
    accumulating.  While a previous step's graph is alive, the next forward reuses its AccumulateGrad nodes, which stay
    bound to the stream they were made on; one bound to the default stream cannot join a capture."""
    def has_history(v):
        if isinstance(v, (list, tuple)):
            return any(has_history(t) for t in v)
        return isinstance(v, torch.Tensor) and v.grad_fn is not None
    for mod in model.modules():
        for k, v in list(vars(mod).items()):
            if has_history(v):
                setattr(mod, k, None)
    for p in params:
        p.grad = None


def _autocast_dtype():
    return torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else None


class GraphedTrainStep:
    """``model(batch, training=True)`` + ``loss.backward()`` + the train-time hit@1 / F1 as one CUDA graph per batch
    shape, for ReaRev and NSM.

    :meth:`step` copies the ``get_batch`` 7-tuple into static buffers (the input side of :class:`GraphedStep`: facts
    at the front of a ``fact_capacity`` bucket, the live count in ``nfacts``), replays the graph and re-attaches the
    graph's gradient tensors to ``p.grad`` of every trainable parameter.  After a step ``p.grad`` holds this batch's
    gradient, overwritten rather than accumulated (as ``zero_grad(); loss.backward()``), so
    ``optimizer.zero_grad(set_to_none=True)`` between steps is fine.  Without ``optimizer``, clipping and
    ``optimizer.step()`` stay with the caller; they update the parameters in place, and the graph reads every weight
    from the parameter's storage when it replays.

    With a ``torch.optim.Adam`` as ``optimizer``, the graph goes on after the metrics with
    ``clip_grad_norm_(params, max_norm)`` (when ``max_norm`` is given) and ``optimizer.step()`` as two kernels
    (:class:`optim.ClipAdam`), bit-equal to torch's foreach Adam given the norm they compute, which the output returns
    as ``grad_norm``.  ``params`` are the parameters the captured backward gives a gradient; the optimizer updates
    those it holds, as ``Adam.step()`` skips ``grad is None``.  The optimizer state stays torch's (missing state is
    created before the capture, the CPU ``step`` tensors advance on the host), so ``state_dict()``, checkpoints and
    eager steps in between keep working, and ``p.grad`` holds the clipped gradient afterwards.  ``lr`` and the other
    hyperparameters are read on every step, so a scheduler needs no new capture.  :func:`optim.check_optimizer`
    lists what is refused (``ValueError``).

    A graph is keyed on the batch shape (B, N, fact capacity, Q, index dtype) and on the state the forward reads when
    it is captured: ``model.training``, every dropout probability in effect, the autocast dtype, torch's
    deterministic-algorithms flag, the cuDNN / TF32 switches, which parameters are trainable and the ``data_ptr`` of
    every parameter (``p.data = ...`` recaptures; in-place updates do not); with an optimizer also ``max_norm``,
    whether any group has a weight decay and the ``data_ptr`` of every optimizer state tensor (so
    ``optimizer.load_state_dict`` recaptures).  Captured graphs are kept in an LRU of
    ``max_graphs`` entries.  Padding slots past ``nfacts`` contribute nothing: the kernels read live facts through
    the CSR and the torch-side per-fact work masks them (autograd_path.LiveBatch).  Dropout masks come from torch's
    CUDA generator, which a graph advances on every replay, so each replay draws fresh masks.  After the first
    capture of a key a step does no host synchronisation.

    Every kernel path of the eager forward must be available (the aggregation, instruction, query-reform and, with
    ``encode_type``, TypeLayer kernels); otherwise, and for GraftNet or a CPU model, the constructor or the step raises
    ``ValueError``."""

    optimizer = max_norm = None          # without an optimizer the graph ends at the gradients

    def __init__(self, model, max_graphs=8, optimizer=None, max_norm=None):
        from .models import GraftNet
        if isinstance(model, GraftNet):
            raise ValueError("GraphedTrainStep covers ReaRev and NSM; GraftNet trains in GraphedGraftTrainStep")
        self._setup(model, max_graphs, _KbLayout, optimizer, max_norm)

    def _setup(self, model, max_graphs, layout, optimizer, max_norm):
        self.model = model
        self._params = list(model.parameters())
        if not self._params or self._params[0].device.type != "cuda":
            raise ValueError("%s needs a model on a CUDA device (model.cuda()); there is no CPU path"
                             % type(self).__name__)
        optim.check_optimizer(optimizer, self._params, max_norm)
        self.optimizer, self.max_norm = optimizer, None if max_norm is None else float(max_norm)
        self.device = self._params[0].device
        self.max_graphs = max_graphs
        self._cache = collections.OrderedDict()
        self._layout = layout(self)
        self._epochs = {}

    @staticmethod
    def tp_list(h1, f1):
        """The ``tp_list`` of ``model(batch, training=True)``: [h1.tolist(), f1.tolist()] (one device read)."""
        return [h1.tolist(), f1.tolist()]

    # -- capture key and refusals ----------------------------------------------------------------------------------
    def key(self, batch):
        """The capture key of ``batch`` under the current model and torch state (see the class docstring)."""
        return self._layout.key(batch) + self._state_key() + self._layout.model_key()

    def _state_key(self):
        """The part of the capture key that is not the batch shape: the model, torch and optimizer state."""
        m = self.model
        if len(self._params) != sum(1 for _ in m.parameters()):
            raise ValueError("the model's parameters changed after GraphedTrainStep was built: build a new one")
        drops = tuple(float(d.p) if d.training else 0.0 for d in m.modules() if isinstance(d, torch.nn.Dropout))
        backends = (torch.backends.cudnn.enabled, torch.backends.cudnn.allow_tf32,
                    torch.backends.cuda.matmul.allow_tf32)
        opt = self.optimizer
        fused = () if opt is None else (self.max_norm, any(g["weight_decay"] != 0 for g in opt.param_groups),
                                        optim.state_key(opt))
        return (
            m.training, drops, _autocast_dtype(), torch.are_deterministic_algorithms_enabled(), backends,
            tuple(p.requires_grad for p in self._params), tuple(p.data_ptr() for p in self._params),
            _rel_text_ptrs(m)) + fused

    def refusal(self, Q):
        """Why the eager forward would leave the kernels for questions of Q tokens (a message), or None."""
        return self._layout.refusal(Q)

    # -- capture ---------------------------------------------------------------------------------------------------
    def _run(self, st, ac):
        """forward + backward + metrics over the static buffers ``st`` -> (loss, pred, pred_dist, h1, f1, status)."""
        m = self.model
        # Autocast casts every weight once per forward and reuses the copy (its cast cache), so the gradients of a
        # weight's uses are summed in the low-precision dtype, as in the eager step.  The cache is emptied before the
        # forward (an entry made outside the capture would freeze that weight into the graph) and after it (the
        # graph's copies must not serve eager code).
        with torch.autocast("cuda", dtype=ac) if ac is not None else contextlib.nullcontext():
            torch.clear_autocast_cache()
            db, loss, pred, pred_dist = self._layout.train_forward(st)
            torch.clear_autocast_cache()
        loss.backward()
        pred_dist = pred_dist.detach()
        cand_idx, cand_count, _ = ops.rank_candidates(pred_dist, db.local_entity, (db.seed_dist > 0).float(),
                                                      m.num_entity, m.eps)
        h1, f1 = ops.train_metrics(pred_dist, db.answer_dist, db.seed_dist, db.local_entity, cand_idx, cand_count,
                                   m.num_entity)
        words = self._layout.status_words(db)
        return loss.detach(), pred, pred_dist, h1, f1, words[0] if len(words) == 1 else torch.cat(words)

    def _entry(self, batch):
        key = self.key(batch)
        ent = self._cache.get(key)
        if ent is not None:
            self._cache.move_to_end(key)
            return ent
        why = self.refusal(key[3])
        if why is not None:
            raise ValueError("GraphedTrainStep: " + why)
        _evict(self._cache, self.max_graphs)
        ac = _autocast_dtype()
        st = self._layout.static_inputs(key)
        self._layout.fill(st, batch)
        params = [p for p in self._params if p.requires_grad]

        def warm():
            _release_autograd_history(self.model, params)
            self._run(st, ac)
        _warm_up(warm)
        fused = None
        if self.optimizer is not None:
            # the warm-up's gradients show which parameters the backward reaches; their missing Adam state is made
            # now, so the key the next step computes (it holds the state's data_ptrs) is the one stored below
            fused = optim.ClipAdam(self.optimizer, params, [p.grad for p in params], self.max_norm)
            key = self.key(batch)
        _release_autograd_history(self.model, params)    # the captured backward allocates every gradient

        def captured():
            outs = self._run(st, ac)
            if fused is not None:
                fused.launch()
            return outs
        g, outs = _capture(captured)
        return self._store(key, st, g, outs, params, fused)

    def _store(self, key, st, g, outs, params, fused, epoch=None):
        """Cache a captured training graph under ``key`` with everything its replays read and write (``epoch``: the
        epoch buffers of an epoch graph)."""
        ent = _Captured()
        ent.st, ent.g, ent.outs, ent.epoch = st, g, outs, epoch
        ent.params, ent.grads = params, [p.grad for p in params]
        ent.fused = fused
        if fused is not None:                    # the kernels read and clip the captured backward's gradients
            fused.bind([p.grad for p in fused.params])
        self._cache[key] = ent
        return ent

    def step(self, batch):
        """One training step on ``batch`` (the 7-tuple of ``get_batch``, host numpy or pinned) ->
        :class:`TrainStepOutput` ``(loss, pred, pred_dist, h1, f1)``; ``p.grad`` holds this batch's gradients (clipped,
        and the parameters updated, with an optimizer)."""
        ent = self._entry(batch)
        self._layout.fill(ent.st, batch)
        if ent.fused is not None:
            ent.fused.prepare()
        ent.g.replay()
        for p, g in zip(ent.params, ent.grads):
            p.grad = g
        return TrainStepOutput(*ent.outs, raise_for=self._layout.raise_for,
                               grad_norm=None if ent.fused is None else ent.fused.grad_norm)

    # -- a whole epoch -----------------------------------------------------------------------------------------------
    def train_epoch(self, split, batch_size, fact_dropout):
        """The reference's ``Trainer_KBQA.train_epoch`` around the model, over the resident split ``split`` (for
        :class:`GraphedGraftTrainStep` a GraftNet split): one :meth:`start_epoch`, one read.  -> ``(np.mean(losses),
        [0, 0], h1_list_all, f1_list_all)``.  Raises :meth:`EpochRun.check`'s errors after the epoch when a batch was
        malformed."""
        run = self.start_epoch(split, batch_size, fact_dropout)
        out = run.result()
        run.check()
        return out

    def start_epoch(self, split, batch_size, fact_dropout):
        """Start one training epoch over ``split`` (a ``loader.DeviceSplit``) and return its :class:`EpochRun` without
        waiting for the device.

        As the reference's ``train_epoch``: ``model.train()``, ``split.reset_batches(is_sequential=False)`` (the
        loader's ``np.random`` order), then every batch of ``batch_size`` questions in order, the last one short when
        ``num_data % batch_size != 0``, each assembled as ``split.get_batch(it, batch_size, fact_dropout)`` does,
        trained and stepped.  Each step is one graph replay: the graph assembles the batch on the device from a
        cursor into the epoch's question order (gr_epoch_step_begin, ``DeviceSplit.assemble`` at the bucket's fact
        capacity, the fact-order seed drawn from torch's CUDA generator with ``shuffle``; for GraftNet also
        gr_epoch_graft_begin after the first kernel and ``DeviceSplit.assemble_graft`` at the bucket's graft capacity,
        both fact orders drawn from the one seed), runs the step of :meth:`step` with the step's Adam scalars (all
        uploaded at the start of the epoch), then records loss, gradient norm, seed, hit@1 and F1 at the cursor and
        advances it (gr_epoch_step_record).  The host picks each step's graph, one per (B, fact capacity) and for
        GraftNet per graft capacity too, from :func:`epoch_plan`; the graphs the epoch needs and does not hold yet are
        captured before the first replay (the LRU grows to hold them all), without moving the records, the parameters
        or torch's generator.  A GraftNet ``EpochRun.status`` has three words: assembly, CSR and graft staging.

        Afterwards ``p.grad``, the parameters and the Adam state are those of the loop ``get_batch`` + :meth:`step`,
        the CPU ``step`` tensors advanced by the number of steps, and ``split.loader.sample_ids`` is the last batch's.
        Refused (``ValueError``): a step without ``optimizer``, anything but a CUDA ``DeviceSplit`` on the model's
        device of the step's model family (a kb loader for ReaRev / NSM, a GraftNet loader for
        :class:`GraphedGraftTrainStep`), ``batch_size <= 0``, a ``fact_dropout`` ``get_batch`` refuses, and fact
        weights (``normalized_gnn`` / ``norm_rel``) over a ``weights="none"`` split."""
        why = self._train_refusal(split, batch_size, fact_dropout)
        if why is not None:
            raise ValueError(why)
        return _run_epochs([self._train_job(split, batch_size, fact_dropout)])[0]

    def _train_refusal(self, split, batch_size, fact_dropout):
        """The ``ValueError`` message :meth:`start_epoch` refuses ``(split, batch_size, fact_dropout)`` with, or
        None."""
        def dropout_refusal():
            if not split.shuffle and fact_dropout != 0:
                return "fact_dropout must be 0 (facts come in stored order), got %r" % (fact_dropout,)
            if split.shuffle and not 0 <= fact_dropout <= 1:
                return "fact_dropout must be in [0, 1], got %r" % (fact_dropout,)
            return None
        if self.optimizer is None:
            why = "an epoch steps the optimizer in its graphs: build the step with optimizer="
        else:
            why = _split_refusal(self, split, batch_size, True, dropout_refusal)
        return None if why is None else "train_epoch: " + why

    def _train_job(self, split, batch_size, fact_dropout, member=None):
        """The :class:`_EpochJob` of :meth:`start_epoch` (for the sweep member ``member``)."""
        job = _EpochJob(split, member)

        def start():
            job.plan, job.order, job.batches = _plan_epoch(split, batch_size, True,
                                                           fact_dropout if split.shuffle else 0.0, job.rng())

        def begin():
            self.model.train()
            ep = job.ep = _buffers_for(self._epochs, split, batch_size, lambda ep: False,
                                       lambda: _EpochBuffers(split, batch_size, self.max_norm))
            _upload_order(ep, job.order)
            if ep.kept_table is not None:
                from .loader import kept_counts
                ep.kept_table[:split.num_q].copy_(torch.from_numpy(kept_counts(split._stored, fact_dropout)),
                                                  non_blocking=True)
                if ep.graft_kept_table is not None:
                    ep.graft_kept_table[:split.num_q].copy_(
                        torch.from_numpy(kept_counts(split._graft_count, fact_dropout)), non_blocking=True)

        def capture():
            ep, plan = job.ep, job.plan
            entries = _epoch_graphs(self, plan, lambda shape: self._epoch_key(ep, shape, member),
                                    lambda shape, s0: self._epoch_capture(ep, shape, s0, member))
            if len({ent.fused.layout() for ent in entries if ent.fused is not None}) > 1:
                raise RuntimeError("train_epoch: the epoch's graphs update different parameter sets")
            fused = entries[0].fused if entries else None
            if fused is not None and plan.steps:
                ep.adam.copy_(torch.from_numpy(fused.epoch_scalars(plan.steps)), non_blocking=True)
            ep.cursor.zero_()
            ep.status.zero_()
            job.entries = entries
            return entries

        def finish():
            ep, entries = job.ep, job.entries
            job.set_sample_ids()
            if entries:
                last = entries[-1]
                for p, g in zip(last.params, last.grads):
                    p.grad = g
                if entries[0].fused is not None:
                    entries[0].fused.advance(job.plan.steps)
            return EpochRun(ep.losses.clone(), None if ep.grad_norms is None else ep.grad_norms.clone(),
                            ep.h1.clone(), ep.f1.clone(), None if ep.seeds is None else ep.seeds.clone(),
                            ep.status.clone())
        job.start, job.begin, job.capture, job.finish = start, begin, capture, finish
        return job

    def _epoch_key(self, ep, shape, member=None):
        return (self._layout.epoch_key(ep.split, shape) + self._state_key() + self._layout.model_key()
                + ("epoch", id(ep)) + _member_key(member))

    def _epoch_capture(self, ep, shape, s0, member=None):
        """Capture the epoch graph of ``shape`` (``_KbLayout.epoch_shapes``); ``s0``: a step of the epoch with that
        shape, the one the warm-up assembles."""
        why = self.refusal(self._layout.epoch_key(ep.split, shape)[3])
        if why is not None:
            raise ValueError("GraphedTrainStep: " + why)
        ac = _autocast_dtype()
        params = [p for p in self._params if p.requires_grad]

        def body(st, cursor):
            return _epoch_step(self, ep, st, cursor, lambda st: self._run(st, ac), lambda outs: outs[5])

        def warm(st, cursor):
            _release_autograd_history(self.model, params)
            body(st, cursor)
        st = _warm_up_epoch_step(self, ep, shape, s0, warm)
        fused = optim.ClipAdam(self.optimizer, params, [p.grad for p in params], self.max_norm)
        T = fused._scalars.shape[0]
        if ep.adam is None:
            ep.adam = torch.zeros(ep.steps, T, 8, dtype=torch.float32, device=self.device)
        elif ep.adam.shape[1] != T:
            raise RuntimeError("train_epoch: the epoch's graphs update different parameter sets")
        key = self._epoch_key(ep, shape, member)
        _release_autograd_history(self.model, params)

        def captured():
            outs, seed, words = body(st, ep.cursor)
            torch.index_select(ep.adam, 0, ep.cursor, out=fused._scalars.view(1, T, 8))
            fused.launch()
            loss, _pred, _pd, h1, f1, _words = outs
            for i in range(2, len(words)):       # gr_epoch_step_record ORs the first two words (assembly, CSR)
                ep.status[i:i + 1].bitwise_or_(words[i])
            ops.epoch_step_record(ep.cursor, ep.batch_size, ep.num_data, loss.float(), fused.grad_norm, seed, h1, f1,
                                  words[0], words[1], ep.losses, ep.grad_norms, ep.seeds, ep.h1, ep.f1, ep.status[:2])
            return outs
        g, outs = _capture(captured, _capture_stream(member))
        ent = self._store(key, st, g, outs, params, fused, ep)
        ent.draws = _member_draws(member)        # its generator and scratch (and the id in the key) stay alive
        return ent


class GraphedGraftTrainStep(GraphedTrainStep):
    """:class:`GraphedTrainStep` for GraftNet: ``model(batch, training=True)`` + ``loss.backward()`` + the train-time
    hit@1 / F1 as one CUDA graph per batch shape, with the same :meth:`step`, :meth:`tp_list`, LRU, gradients and
    optional clip + Adam step (``optimizer``, ``max_norm``).

    :meth:`step` takes the 9/10-tuple of ``GraftSingleDataLoader.get_batch`` (host numpy, pinned tensors or a
    ``loader.DeviceSplit`` batch) and copies it into the static buffers of :class:`_GraftLayout`: kb facts at a
    ``fact_capacity`` bucket with their live count in ``nfacts``, both graft lists at their own bucket with their live
    counts in ``graft_live``, ``kb_fact_rel``.  In the graph gr_graft_stage stages the live graft facts and writes
    their count on the device, and the forward runs ``autograd_path.graftnet_core`` over capacity-length per-fact
    vectors (``autograd_path.graft_live_stage``), so nothing reads a count on the host.  The three status words (kb CSR,
    graft staging, graft CSR) come back in the output; ``out.check()`` raises ``GraftGraph``'s messages.

    The capture key is :class:`GraphedTrainStep`'s plus the graft capacity, ``max_fact``, and the two Python scalars
    the forward bakes into the graph: ``pagerank_lambda`` and ``fact_scale``.  A CPU model, ``USE_KERNELS`` off or an
    ``entity_dim`` the GraftNet training kernels do not admit (``ops.fact_train_ok``) raises ``ValueError``, as does a
    batch that is not a graft tuple."""

    def __init__(self, model, max_graphs=8, optimizer=None, max_norm=None):
        from .models import GraftNet
        if not isinstance(model, GraftNet):
            raise ValueError("GraphedGraftTrainStep covers GraftNet; ReaRev and NSM train in GraphedTrainStep")
        self._setup(model, max_graphs, _GraftLayout, optimizer, max_norm)

    def key(self, batch):
        if len(batch) not in (9, 10):
            raise ValueError("GraphedGraftTrainStep takes the 9/10-tuple of GraftSingleDataLoader.get_batch, not a "
                             "%d-tuple" % len(batch))
        return super().key(batch)


# ---- several runs side by side on one GPU ----------------------------------------------------------------------------

class _Draws:
    """What a sweep member's graphs hold for as long as they live, and nothing more (no step: a graph cached in a step's
    LRU must not keep its step alive through a cycle): the member's CUDA generator, its device, its copies of the
    :func:`_shared_scratch` dicts and the stream its graphs are captured on.  Its ``id`` is part of their keys."""

    def __init__(self, generator, device):
        self.generator, self.device = generator, device
        self.scratch = tuple({} for _ in _shared_scratch())
        self.capture_stream = torch.cuda.Stream(device=device)


class _Member:
    """One run of a :class:`Sweep`: its step, its ``np.random.RandomState`` (``rng``), the stream its uploads and
    replays go to, its :class:`_Draws` (the CUDA generator, the scratch and the capture stream its graphs keep) and the
    :class:`GraphedStep` its evaluations run through."""

    def __init__(self, step, generator, rng):
        self.step, self.rng = step, rng
        self.draws = _Draws(generator, step.device)
        self.stream = torch.cuda.Stream(device=step.device)
        self._eval_step = step if isinstance(step, GraphedStep) else None

    @property
    def generator(self):
        return self.draws.generator

    def eval_step(self):
        """The member's :class:`GraphedStep`: the step itself, or for a training step one over its model (the model's
        ``num_entity`` and ``eps``), made at the first use."""
        if self._eval_step is None:
            m = self.step.model
            self._eval_step = GraphedStep(m, m.num_entity)
        return self._eval_step


def _check_members(steps):
    """Refuse (``ValueError``) sweep members that are not graphed steps, that share a model or that are not on one
    CUDA device."""
    if not steps:
        raise ValueError("Sweep: no members")
    for i, s in enumerate(steps):
        if not isinstance(s, (GraphedStep, GraphedTrainStep)):
            raise ValueError("Sweep: member %d is a %s; members are GraphedTrainStep, GraphedGraftTrainStep or "
                             "GraphedStep objects" % (i, type(s).__name__))
    seen = {}
    for i, s in enumerate(steps):
        j = seen.setdefault(id(s.model), i)
        if j != i:
            raise ValueError("Sweep: members %d and %d hold the same model; each run needs a model of its own" % (j, i))
    devices = [torch.device(s.device) for s in steps]
    if any(d.type != "cuda" for d in devices):
        raise ValueError("Sweep: the members' models are on %s; a sweep runs on one CUDA device"
                         % ", ".join(sorted({str(d) for d in devices})))
    if len({d.index for d in devices}) > 1:
        raise ValueError("Sweep: members on different devices (%s); a sweep runs on one CUDA device"
                         % ", ".join(sorted({str(d) for d in devices})))


def _job_refusal(member, job, training):
    """Why the sweep refuses ``job`` for ``member`` (a message), or None: what :meth:`GraphedTrainStep.start_epoch`
    (with ``training``) or :meth:`GraphedStep.start_eval` refuses, with their messages, a job that is not their
    argument tuple (an evaluation job of three is one over a ``loader.DeviceSplit``), and a training job for a
    :class:`GraphedStep`.  ``job`` None: the member sits this one out."""
    if job is None:
        return None
    from .loader import DeviceSplit
    if training:
        shaped = isinstance(job, (tuple, list)) and len(job) == 3
    else:                             # (split, batch_size) or (split, batch_size, path_targets) over a DeviceSplit
        shaped = isinstance(job, (tuple, list)) and (len(job) == 2 or len(job) == 3 and isinstance(job[0], DeviceSplit))
    if not shaped:
        return "Sweep.%s: a job is %s or None, got %r" % (
            "start_epochs" if training else "start_evals",
            "(split, batch_size, fact_dropout)" if training else "(split, batch_size[, path_targets])", job)
    if training:
        if not isinstance(member.step, GraphedTrainStep):
            return ("Sweep.start_epochs: a GraphedStep member evaluates only; a training member is a "
                    "GraphedTrainStep / GraphedGraftTrainStep built with optimizer=")
        return member.step._train_refusal(*job)
    return member.eval_step()._eval_refusal(*job)


class Sweep:
    """Several independent runs on one GPU, their epochs side by side: each member replays its epoch graphs on a
    stream of its own, so the small launches of one run fill the SMs the others leave idle.  Each member's results are
    bit for bit those of the same epochs run alone (:meth:`GraphedTrainStep.start_epoch`,
    :meth:`GraphedStep.start_eval`) with torch's default CUDA generator at the member's generator state and
    ``np.random`` at its ``RandomState``, whatever the other members run (DESIGN §4.14).

    ``steps``: the members, each a :class:`GraphedTrainStep` / :class:`GraphedGraftTrainStep` built with
    ``optimizer=`` or a :class:`GraphedStep` that only evaluates; each over a model of its own, all on one CUDA device.
    ``generators``: one ``torch.Generator`` per member on that device, else each member gets a generator seeded with
    one draw from torch's default CUDA generator when the sweep is built.  A member's graphs are captured with its
    generator as the default generator's graph-safe state, so they draw its fact-order seeds, its dropout masks and
    GraftNet's dropout seeds from it, and only its own replays advance it.  ``rngs``: one ``np.random.RandomState``
    per member, else each seeded with one draw from ``np.random`` when the sweep is built; it stands in for
    ``np.random`` while the member's ``reset_batches`` draws its epoch order, and nowhere else.

    :meth:`start_epochs` and :meth:`start_evals` take one job per member -- the arguments of ``start_epoch`` /
    ``start_eval``, or None for a member that sits it out -- and return one :class:`EpochRun` / :class:`EvalRun` per
    member (None for those) without waiting for the device.  Every job is checked first, with the messages of the
    single-run methods; then every member's host start and uploads, then every capture any member needs, and only
    then the replays: step s of every member, then step s + 1, members with fewer steps dropping out.  Between
    epochs, LR schedulers, ``optimizer.state_dict()`` and checkpoints work per member as they do for a single run.
    Members may share a ``DeviceSplit``: the split holds no scratch its steps write.  A shared split's
    ``loader.sample_ids`` ends as the last batch of the last member (in member order) that ran over it.  A refused
    job raises before any member's order is drawn: a refusal found while planning (an int32 overflow, answers that
    are not integers) puts every member's ``RandomState`` and its loader's ``batches`` back.

    The epochs of one call overlap each other.  Consecutive calls do not overlap: each call's members wait for the
    caller's stream first, and the caller's stream waits for them at the end, so ``start_evals`` right after
    ``start_epochs`` runs the evaluations after the training replays.

    Build a sweep once and keep it.  A graph is bound to the generator it was captured with, so each sweep captures
    its members' graphs anew; they stay in the steps' LRUs (``max_graphs``) and are released by its eviction."""

    def __init__(self, steps, generators=None, rngs=None):
        steps = list(steps)
        _check_members(steps)
        K, dev = len(steps), torch.device(steps[0].device)
        if generators is None:
            seeds = torch.randint(0, 2 ** 62, (K,), dtype=torch.int64, device=dev).tolist()
            generators = [torch.Generator(device=dev) for _ in range(K)]
            for g, s in zip(generators, seeds):
                g.manual_seed(s)
        generators = list(generators)
        from .loader import same_device
        if len(generators) != K or any(not isinstance(g, torch.Generator) or not same_device(g.device, dev)
                                       for g in generators):
            raise ValueError("Sweep: generators must be %d torch.Generator objects on %s" % (K, dev))
        if len({id(g) for g in generators}) != K:
            raise ValueError("Sweep: two members share a generator; each run needs its own")
        if rngs is None:
            rngs = [np.random.RandomState(s) for s in np.random.randint(0, 2 ** 31 - 1, size=K).tolist()]
        rngs = list(rngs)
        if len(rngs) != K or any(not isinstance(r, np.random.RandomState) for r in rngs):
            raise ValueError("Sweep: rngs must be %d np.random.RandomState objects" % K)
        if len({id(r) for r in rngs}) != K:
            raise ValueError("Sweep: two members share a RandomState; each run needs its own")
        self.members = [_Member(s, g, r) for s, g, r in zip(steps, generators, rngs)]

    @property
    def generators(self):
        return [m.generator for m in self.members]

    @property
    def rngs(self):
        return [m.rng for m in self.members]

    def eval_step(self, i):
        """The :class:`GraphedStep` member ``i`` evaluates through."""
        return self.members[i].eval_step()

    def start_epochs(self, jobs):
        """One training epoch per member with a job ``(split, batch_size, fact_dropout)`` -> one :class:`EpochRun`
        per member (None where the job is None), as :meth:`GraphedTrainStep.start_epoch` returns it."""
        return self._start(jobs, True)

    def start_evals(self, jobs):
        """One evaluation per member with a job ``(split, batch_size)`` or ``(split, batch_size, path_targets)`` -> one
        :class:`EvalRun` per member (None where the job is None), as :meth:`GraphedStep.start_eval` returns it.  A training member evaluates its model
        through :meth:`eval_step`."""
        return self._start(jobs, False)

    def _start(self, jobs, training):
        jobs = list(jobs)
        if len(jobs) != len(self.members):
            raise ValueError("Sweep.%s: %d jobs for %d members (None: a member sits this one out)"
                             % ("start_epochs" if training else "start_evals", len(jobs), len(self.members)))
        for m, job in zip(self.members, jobs):
            why = _job_refusal(m, job, training)
            if why is not None:
                raise ValueError(why)
        todo = [(k, m, job) for k, (m, job) in enumerate(zip(self.members, jobs)) if job is not None]
        made = [m.step._train_job(*job, member=m) if training else m.eval_step()._eval_job(*job, member=m)
                for _k, m, job in todo]
        runs = [None] * len(jobs)
        for (k, _m, _job), run in zip(todo, _run_epochs(made)):
            runs[k] = run
        return runs
