"""Differentiable forward for ``model(batch, training=True)`` (gnn/train_model.py:209-233).

The inference path runs hand-written CUDA kernels; ``Trainer_KBQA.train_epoch`` needs
``loss.backward()`` through the same parameters.  This module evaluates the same math with torch ops on the model's
device (CUDA when the model lives there -- no CPU fallback is involved) so that autograd provides the gradients:

  * the relation projection ``rel_linear_k`` is hoisted from the F facts to the R1 relation rows (one GEMM per layer);
  * messages are formed per fact (``relu(P[rel] * ins[batch]) * w^2 * prior[src]``) and reduced with ``index_add_``
    (deterministic order is not needed for training);
  * dropouts are applied where the reference applies them (``linear_drop`` before e2e / score / instruction linears,
    ``lstm_drop`` on the word embeddings), active only under ``model.train()``;
  * on CUDA with ``USE_KERNELS`` the aggregations, the TypeLayer and GraftNet's fact attention and fact messages run
    in hand-written kernels with their own backward (the ``torch.autograd.Function``s below); the per-fact torch
    restatement is the CPU reference under ``HOST_CHECK`` and the ``USE_KERNELS = False`` path;
  * on CUDA with ``USE_KERNELS``, at the shapes the forward kernels admit, the instruction steps (ReaRev, NSM) and
    ReaRev's query reform run in the question-side kernels with their own backward (_InstructionsFn, _QueryReformFn);
    the instruction dropout is drawn in the kernel from a seed of torch's CUDA generator;
  * under ``torch.use_deterministic_algorithms(True)`` (``warn_only`` included), read by each Function at forward,
    those backward kernels are the fixed-order, atomic-free variants: every gradient they produce is a pure function
    of the inputs.  The torch restatement's ``index_add`` is made deterministic by torch itself under the same flag;
  * under ``torch.autocast("cuda", dtype=torch.bfloat16)``, read by each Function at forward as well, the kernels take
    and produce their node-sized tensors ([B*N, D] outputs and gradients) in bf16: the same fp32 arithmetic, with each
    stored value rounded to nearest even.  Their small operands (relation tables, instructions, priors, per-fact
    scalars) are cast to fp32 inside the Functions.  Under fp16 autocast the Functions cast to fp32 and run the fp32
    kernels.  The torch restatement accumulates its scatters in fp32.

Reference: ReaRev.forward gnn/models/ReaRev/rearev.py:163-243, ReasonGNNLayer.forward gnn/modules/kg_reasoning/
reasongnn.py:61-174, TypeLayer.forward gnn/modules/layer_init.py:25-62, BaseInstruction.get_instruction
gnn/modules/question_encoding/base_encoder.py:82-102, QueryReform / Fusion gnn/modules/query_update.py:6-44,
NSM.forward gnn/models/NSM/nsm.py:179-254, NSMLayer gnn/modules/kg_reasoning/nsm_gnn.py:54-112, the loss
gnn/models/base_model.py:193-215 and the train-time metrics get_eval_metric gnn/models/base_model.py:236-298.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import ops

VERY_NEG_NUMBER = -100000000000


class _Facts:
    """Fact arrays of one ``get_batch`` tuple on the device (the COO operators of build_matrix, base_gnn.py:19-51,
    as index vectors)."""

    def __init__(self, kb_adj_mat, device, normalized_gnn, norm_rel):
        heads, rels, tails, bids, _fids, weight_list, weight_rel_list = kb_adj_mat

        def idx(a):
            if isinstance(a, torch.Tensor):
                return a.to(device=device, dtype=torch.int64)
            return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.int64))).to(device)
        self.heads, self.rels, self.tails = idx(heads), idx(rels), idx(tails)
        if bids is None:
            raise ValueError("training needs the batch_ids array of kb_adj_mat (dataset_load.py:521)")
        self.bids = idx(bids)
        def weights(w):       # host lists / float64 arrays, or the fp32 tensors of a loader.DeviceSplit batch
            if isinstance(w, torch.Tensor):
                return w.to(device=device, dtype=torch.float32)
            return torch.as_tensor(np.asarray(w, dtype=np.float32), device=device)
        self.w = self.wr = None
        if normalized_gnn:
            if weight_list is None:
                raise ValueError("normalized_gnn needs kb_adj_mat's weight_list")
            self.w = weights(weight_list)
        if norm_rel:
            if weight_rel_list is None:
                raise ValueError("norm_rel needs kb_adj_mat's weight_rel_list")
            self.wr = weights(weight_rel_list)
        self.live = None          # every slot is a fact (cf. _LiveFacts)


class _LiveFacts:
    """Fact arrays of a :class:`LiveBatch`: fixed-capacity buffers whose first ``nfacts`` slots are facts.  ``live``
    marks those slots; the padding slots read node 0 (ids are clamped into the batch, as gr_csr_build clamps them) and
    the users of ``live`` zero what they contribute.  Only the per-fact torch work that the kernels do not cover reads
    these (NSM's reason_kb mask); the aggregations see live facts through the CSR."""

    def __init__(self, heads, tails, weight_list, nfacts, Nt):
        self.live = torch.arange(heads.numel(), device=heads.device) < nfacts
        self.heads, self.tails = (torch.where(self.live, a.long().clamp(0, Nt - 1), 0) for a in (heads, tails))
        self.rels = self.bids = self.wr = None
        self.w = weight_list


class LiveBatch:
    """A training batch already on the device in fixed-capacity buffers (graphed.GraphedTrainStep): the [B, N] and
    [B, Q] tensors and the CSR of a :class:`batching.DeviceBatch` built with ``nfacts``, plus the raw fact buffers for
    :class:`_LiveFacts`.  ``model(batch, training=True)``'s forward takes it in place of the ``get_batch`` tuple."""

    def __init__(self, db, heads, tails, weight_list, nfacts):
        self.db = db
        self._raw = (heads, tails, weight_list, nfacts)
        self._facts = None

    @property
    def facts(self):
        if self._facts is None:
            heads, tails, w, nfacts = self._raw
            self._facts = _LiveFacts(heads, tails, w, nfacts, self.db.B * self.db.N)
        return self._facts


def _scatter_rows(values, dst, rows):
    """Row sums in fp32 (bf16 / fp16 values under autocast are widened; fp32 values are used as they are)."""
    out = torch.zeros(rows, values.shape[1], dtype=torch.float32, device=values.device)
    return out.index_add_(0, dst, values.float())


def _type_layer(layer, facts, rel_features, Nt, graph=None):
    """layer_init.py:44-59: relu(sum over facts into tails + sum over facts into heads) of kb_self_linear(rel).
    With the batch's CsrGraph (kernel path) the sums and their backward run in gr_type_layer /
    gr_type_layer_backward (_TypeLayerFn); otherwise per fact with index_add."""
    if graph is not None:
        wt, wh = (graph.wr_t, graph.wr_h) if layer.norm_rel else (None, None)
        return _TypeLayerFn.apply(layer.kb_self_linear(rel_features), graph, wt, wh)
    fact_val = layer.kb_self_linear(rel_features)[facts.rels]
    if facts.wr is not None:
        fact_val = fact_val * facts.wr.unsqueeze(1)
    return F.relu(_scatter_rows(fact_val, facts.tails, Nt) + _scatter_rows(fact_val, facts.heads, Nt))


def _aggregate(table, ins_j, prior_flat, facts, src, dst, Nt):
    """reasongnn.py:61-89 (src = heads, dst = tails) / :91-116 (src = tails, dst = heads)."""
    fact_val = F.relu(table[facts.rels] * ins_j[facts.bids])
    prior = prior_flat[src]
    if facts.w is not None:
        prior = prior * facts.w * facts.w          # head2fact and fact2tail both carry the weight (base_gnn.py:38-48)
    return _scatter_rows(fact_val * prior.unsqueeze(1), dst, Nt)


USE_KERNELS = True      # CUDA tensors: aggregation forward / backward through the hand-written kernels (below)
HOST_CHECK = False      # tests only: let a CPU-resident model evaluate this restatement with torch CPU ops, so that the
                        # ``-m "not gpu"`` suite can hold it against the reference's gradients.  Off (the product):
                        # ``model(batch, training=True)`` on a CPU model raises, like the inference path.


def _autocast_bf16():
    """True under torch.autocast("cuda", dtype=torch.bfloat16): the training kernels then produce their node-sized
    outputs in bf16.  Read by each Function at forward, like the deterministic flag."""
    return torch.is_autocast_enabled("cuda") and torch.get_autocast_dtype("cuda") == torch.bfloat16


def _node_dtype():
    return torch.bfloat16 if _autocast_bf16() else torch.float32


def _require_cuda(dev):
    if dev.type != "cuda" and not HOST_CHECK:
        raise RuntimeError("gnn_rag_b200 runs on CUDA only: move the model to an H100 (model.cuda()); there is no CPU "
                           "path (training=True included)")


class _AggregateFn(torch.autograd.Function):
    """out[n, j, :] = sum_{e -> n} w_e^2 p[src_e] relu(table[rel_e] * ins[b, j]) for all instructions j of one direction:
    forward = gr_aggregate (csrc/aggregate.cu), backward = gr_aggregate_backward (csrc/aggregate_bwd.cu).  The output
    is bf16 under bf16 autocast; the backward reads grad_out in its own dtype."""

    @staticmethod
    def forward(ctx, table, ins, prior, graph, direction, w):
        ctx.dtypes = (table.dtype, ins.dtype, prior.dtype)
        table, ins, prior = table.detach().float(), ins.detach().float(), prior.detach().float()
        out = ops.aggregate(graph, direction, prior, table, ins, w=w, dtype=_node_dtype())
        ctx.save_for_backward(table, ins, prior)
        ctx.graph, ctx.direction, ctx.w = graph, direction, w
        ctx.det = torch.are_deterministic_algorithms_enabled()
        return out

    @staticmethod
    def backward(ctx, grad_out):
        table, ins, prior = ctx.saved_tensors
        # the kernel accumulates into dense row-major buffers: zeros_like alone would keep a transposed input's strides
        gt, gi, gp = (torch.zeros_like(t, memory_format=torch.contiguous_format) for t in (table, ins, prior))
        ops.aggregate_backward(ctx.graph, ctx.direction, prior, table.contiguous(), ins.contiguous(),
                               grad_out.contiguous(), gt, gi, gp, ctx.w, deterministic=ctx.det)
        return (*(g.to(dt) for g, dt in zip((gt, gi, gp), ctx.dtypes)), None, None, None)


class _TypeLayerFn(torch.autograd.Function):
    """out = relu(sum_{tail CSR} w_e table[rel_e] + sum_{head CSR} w_e table[rel_e]) (TypeLayer, layer_init.py:46-57):
    forward = gr_type_layer (csrc/aggregate.cu), backward = gr_type_layer_backward (csrc/aggregate_bwd.cu); saves the
    [B*N, D] output (bf16 under bf16 autocast) for the relu mask."""

    @staticmethod
    def forward(ctx, table, graph, w_t, w_h):
        out = torch.empty(graph.B * graph.N, table.shape[1], dtype=_node_dtype(), device=table.device)
        ops.type_layer(graph, table.detach().float(), out, w_t, w_h)
        ctx.save_for_backward(out)
        ctx.graph, ctx.w, ctx.rows, ctx.dtype = graph, (w_t, w_h), table.shape[0], table.dtype
        ctx.det = torch.are_deterministic_algorithms_enabled()
        return out

    @staticmethod
    def backward(ctx, grad_out):
        out, = ctx.saved_tensors
        if grad_out.dtype != out.dtype:      # widening is exact: same gradients as with grad_out in out's dtype
            out, grad_out = out.float(), grad_out.float()
        gt = torch.zeros(ctx.rows, out.shape[1], dtype=torch.float32, device=out.device)
        ops.type_layer_backward(ctx.graph, grad_out.contiguous(), out, gt, *ctx.w, deterministic=ctx.det)
        return gt.to(ctx.dtype), None, None, None


def _fact_kernels(device, D):
    """True when the TypeLayer and GraftNet's fact-level work run in the training kernels: CUDA, ``USE_KERNELS`` and
    a width they admit (:func:`ops.fact_train_ok`); the per-fact torch ops otherwise."""
    return bool(USE_KERNELS and device.type == "cuda" and ops.fact_train_ok(D))


def _type_layer_graph(model, batch, device, D):
    """The batch's CSR for the TypeLayer kernels, or None (no TypeLayer, or a shape / device they do not cover)."""
    return _batch_graph(model, batch, device) if model.encode_type and _fact_kernels(device, D) else None


def _batch_graph(model, batch, device):
    """CSR of the batch for the kernel path (with the normalized_gnn / norm_rel weights the model uses), or None (CPU
    tensors, or ``USE_KERNELS`` off)."""
    if not (USE_KERNELS and device.type == "cuda"):
        return None
    if isinstance(batch, LiveBatch):
        return batch.db.graph
    from . import batching
    return batching.stage_batch(batch, device, model.num_relation + 1, model.normalized_gnn, model.norm_rel).graph


def _kernel_graph(model, batch, device, D, I, graph=None):
    """CSR of the batch for the aggregation kernels, or None (CPU tensors / shapes the backward kernel does not admit,
    :func:`ops.aggregate_backward_ok`).  ``graph``: the batch's CSR if it was already staged (for the TypeLayer)."""
    if not (USE_KERNELS and device.type == "cuda" and ops.aggregate_backward_ok(D, I)):
        return None
    return graph if graph is not None else _batch_graph(model, batch, device)


def _neighbours(table_f, table_i, ins, dist, facts, graph, Nt):
    """[Nt, I, n_dir, D] neighbour messages of one layer (reasongnn.py:150-156), kernel or torch path."""
    I = ins.shape[1]
    if graph is not None:
        outs = [_AggregateFn.apply(table_f.contiguous(), ins, dist, graph, "fwd", graph.w_t).view(Nt, I, 1, -1)]
        if table_i is not None:
            outs.append(_AggregateFn.apply(table_i.contiguous(), ins, dist, graph, "inv", graph.w_h).view(Nt, I, 1, -1))
        return torch.cat(outs, dim=2)
    pf = dist.reshape(-1)
    reps = []
    for j in range(I):
        r = [_aggregate(table_f, ins[:, j], pf, facts, facts.heads, facts.tails, Nt)]
        if table_i is not None:
            r.append(_aggregate(table_i, ins[:, j], pf, facts, facts.tails, facts.heads, Nt))
        reps.append(torch.stack(r, dim=1))
    return torch.stack(reps, dim=1)


def _instruction_kernels(device, Q, D, I):
    """True when the instruction steps run in gr_instructions_train / gr_instructions_backward: CUDA, ``USE_KERNELS``
    and a shape gr_instructions admits (:func:`ops.instructions_ok`)."""
    return bool(USE_KERNELS and device.type == "cuda" and ops.instructions_ok(Q, D, I))


def _reform_kernels(device, D, I):
    """True when the query reform runs in gr_query_reform(_ex) / gr_query_reform_backward: CUDA, ``USE_KERNELS`` and
    a shape gr_query_reform admits (:func:`ops.query_reform_ok`)."""
    return bool(USE_KERNELS and device.type == "cuda" and ops.query_reform_ok(D, I))


def _weight_grads(G, X):
    """(G^T X, column sums of G) over the rows of the per-question operands: one GEMM per weight, fp32 outside
    autocast.  Deterministic under use_deterministic_algorithms (torch's cuBLAS path and reductions)."""
    with torch.autocast("cuda", enabled=False):
        G2 = G.reshape(-1, G.shape[-1])
        return G2.t() @ X.reshape(G2.shape[0], -1), G2.sum(0)


class _InstructionsFn(torch.autograd.Function):
    """All num_ins steps of get_instruction (base_encoder.py:73-114) with the reference's three linear_drop sites:
    forward = gr_instructions_train, backward = gr_instructions_backward (csrc/question.cu), which redraws the Philox
    mask from the saved seed.  The kernels write the per-question gradient operands; each weight gradient is one torch
    GEMM over them.  The question tensors are not node-sized: under autocast everything here is fp32, and each
    gradient is returned in its input's dtype.  Inputs after the data: wca, bca, Wcq, bcq, then (W_i, b_i) of every
    question_linear_i."""

    @staticmethod
    def forward(ctx, hidden, qnode, qtext, pad_id, seed, p, wca, bca, Wcq, bcq, *wq):
        ctx.dtypes = (hidden.dtype, qnode.dtype) + tuple(t.dtype for t in (wca, bca, Wcq, bcq) + wq)
        hidden, qnode = hidden.detach().float().contiguous(), qnode.detach().float().contiguous()
        wts = [t.detach().float().contiguous() for t in (wca, bca, Wcq, bcq) + wq]
        Wq, bq = wts[4::2], wts[5::2]
        out, attn = ops.instructions_train(hidden, qnode, qtext, pad_id, Wq, bq, wts[2], wts[3], wts[0], wts[1],
                                           seed, p)
        ctx.save_for_backward(hidden, qnode, qtext, seed, out, attn, *wts)
        ctx.pad_id, ctx.p = pad_id, p
        return out

    @staticmethod
    def backward(ctx, grad_out):
        hidden, qnode, qtext, seed, out, attn, *wts = ctx.saved_tensors
        wca, bca, Wcq, bcq = wts[:4]
        Wq, bq = wts[4::2], wts[5::2]
        gh, gqn, Gq, Xq, Gcq, Xcq, Gca, Xca = ops.instructions_backward(
            hidden, qnode, qtext, ctx.pad_id, Wq, bq, Wcq, bcq, wca, bca, seed, ctx.p, out, attn, grad_out.float())
        gwca, gbca = _weight_grads(Gca.unsqueeze(-1), Xca)       # rows (b, i, q)
        gWcq, gbcq = _weight_grads(Gcq, Xcq)                     # rows (b, i)
        gq = []
        for i in range(len(Wq)):
            gq.extend(_weight_grads(Gq[:, i], Xq[:, i]))          # rows b
        grads = [gh, gqn, gwca.view(wca.shape), gbca.view(bca.shape), gWcq, gbcq] + gq
        dts = ctx.dtypes
        return (grads[0].to(dts[0]), grads[1].to(dts[1]), None, None, None, None,
                *(g.to(dt) for g, dt in zip(grads[2:], dts[2:])))


def _instructions_kernel(enc, hidden, qnode, q_input):
    """The instruction steps through _InstructionsFn; the dropout seed is one int64 from torch's CUDA generator,
    drawn on the device (no host sync), when the encoder's linear_drop is active."""
    drop = enc.linear_drop
    p = float(drop.p) if drop.training else 0.0
    seed = torch.randint(0, 2 ** 62, (1,), dtype=torch.int64, device=hidden.device) if p > 0.0 else None
    lins = [getattr(enc, "question_linear" + str(i)) for i in range(enc.num_ins)]
    wq = [t for lin in lins for t in (lin.weight, lin.bias)]
    return _InstructionsFn.apply(hidden, qnode.reshape(qnode.shape[0], -1), q_input, enc.pad_val, seed, p,
                                 enc.ca_linear.weight, enc.ca_linear.bias, enc.cq_linear.weight, enc.cq_linear.bias,
                                 *wq)


class _QueryReformFn(torch.autograd.Function):
    """QueryReform + Fusion for every instruction (query_update.py:6-44, rearev.py:214-221): forward =
    gr_query_reform(_ex) (one seed retrieve serves all I reforms), backward = gr_query_reform_backward, which adds the
    seed-row gradient into a zero [B*N, D] grad_h in h's dtype (only the seed rows are written).  h is read in its own
    dtype (bf16 under bf16 autocast); everything else is fp32.  Inputs after the data: (Wr_j, Wg_j) of every reform."""

    @staticmethod
    def forward(ctx, seed_info, h, ins, B, N, *wts):
        ctx.dtypes = (h.dtype, ins.dtype) + tuple(t.dtype for t in wts)
        h = h.detach()
        if h.dtype not in (torch.float32, torch.bfloat16):
            h = h.float()
        ins = ins.detach().float().contiguous()
        wts = [t.detach().float().contiguous() for t in wts]
        out = ops.query_reform(seed_info, h, ins, wts[0::2], wts[1::2], B, N, op="question_train")
        ctx.save_for_backward(seed_info, h, ins, *wts)
        ctx.BN = (B, N)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        seed_info, h, ins, *wts = ctx.saved_tensors
        B, N = ctx.BN
        grad_h = torch.zeros(h.shape, dtype=h.dtype, device=h.device)
        gins, Gr, Gg, Z = ops.query_reform_backward(seed_info, h, ins, wts[0::2], wts[1::2], B, N, grad_out.float(),
                                                    grad_h)
        gw = []
        for j in range(len(wts) // 2):
            gw.append(_weight_grads(Gr[:, j], Z[:, j])[0])
            gw.append(_weight_grads(Gg[:, j], Z[:, j])[0])
        dts = ctx.dtypes
        return (None, grad_h.to(dts[0]), gins.to(dts[1]), None, None, *(g.to(dt) for g, dt in zip(gw, dts[2:])))


def _instructions(enc, q_input):
    """base_encoder.py:73-114 on top of encode_question; returns [B, num_ins, D].  The steps run in the question-side
    kernels (_InstructionsFn) on CUDA with ``USE_KERNELS`` at the shapes gr_instructions admits; otherwise as torch ops
    below."""
    enc.encode_question_train(q_input)
    hidden, qnode, qmask = enc.query_hidden_emb, enc.query_node_emb, enc.query_mask_train
    if _instruction_kernels(hidden.device, hidden.shape[1], hidden.shape[2], enc.num_ins):
        return _instructions_kernel(enc, hidden, qnode, q_input)
    drop = enc.linear_drop
    rel_ins = torch.zeros(q_input.size(0), enc.entity_dim, device=q_input.device)
    out = []
    for i in range(enc.num_ins):
        ri = rel_ins.unsqueeze(1)
        q_i = getattr(enc, "question_linear" + str(i))(drop(qnode))
        cq = enc.cq_linear(drop(torch.cat((ri, q_i, q_i - ri, q_i * ri), dim=-1)))
        ca = enc.ca_linear(drop(cq * hidden))
        attn = F.softmax(ca + (1 - qmask.unsqueeze(2)) * VERY_NEG_NUMBER, dim=1)
        rel_ins = torch.sum(attn * hidden, dim=1)
        out.append(rel_ins)
    return torch.stack(out, dim=1)


def _loss(model, pred_dist, answer_dist):
    case_valid = (torch.sum(answer_dist, dim=1, keepdim=True) > 0).float()
    return model.calc_loss_label(pred_dist, answer_dist, case_valid)


def _retrieved_sets_host(pred_dist, local_entity, seeds, num_entity, eps):
    """Candidate cut of f1_and_hits (base_model.py:216-234) with torch ops on the tensors' own device: used when the
    training tensors do not live on a GPU (the CUDA path uses the ranking kernel)."""
    B, N = pred_dist.shape
    # p < (1 - eps) / N in float64, as the reference compares Python floats: against the fp32 tensor torch would round
    # the bound to fp32 and keep a p just below it
    ignore_prob = (1 - eps) / N
    keep = (seeds == 0) & (local_entity != num_entity) & ~(pred_dist.double() < ignore_prob)
    p = torch.where(keep, pred_dist, torch.full_like(pred_dist, float("-inf")))
    order = torch.sort(p, dim=1, descending=True, stable=True)[1]
    kept = torch.gather(keep, 1, order)
    ps = torch.gather(pred_dist, 1, order)
    csum = torch.cumsum(torch.where(kept, ps, torch.zeros_like(ps)).double(), dim=1)
    total = keep.sum(1)
    crossed = (csum > eps) & kept
    first = torch.where(crossed.any(1), crossed.float().argmax(1) + 1, total)
    count = torch.minimum(first, total)
    return order, count


@torch.no_grad()
def eval_metric(model, pred_dist, answer_dist, seed_dist, local_entity):
    """get_eval_metric (base_model.py:281-298): hit@1 per question, and F1 of the eps-mass retrieval for the questions
    that have hit@1 (0 for the others, :250-253).  The retrieval runs in the ranking kernel when the tensors are on the
    GPU; answers = non-seed, non-pad candidates with answer mass (:266-271)."""
    top1 = pred_dist.argmax(dim=-1, keepdim=True)
    h1 = ((torch.zeros_like(pred_dist).scatter_(1, top1, 1.0) * (answer_dist > 1e-10).float()).sum(-1) > 0).float()
    f1 = torch.zeros_like(h1)
    if bool(h1.any()):
        seeds = (seed_dist > 0).float()
        if pred_dist.is_cuda:
            cand_idx, cand_count, _ = ops.rank_candidates(pred_dist.contiguous(), local_entity, seeds,
                                                          model.num_entity, model.eps)
        else:
            cand_idx, cand_count = _retrieved_sets_host(pred_dist, local_entity, seeds, model.num_entity, model.eps)
        counts = cand_count.cpu().tolist()
        idx_h = cand_idx.cpu().numpy()
        ans_ok = ((answer_dist > 0) & (seeds == 0) & (local_entity != model.num_entity)).cpu().numpy()
        le_h = local_entity.cpu().numpy()
        h1_h = h1.cpu().tolist()
        vals = []
        for b, c in enumerate(counts):
            if h1_h[b] == 0.0:
                vals.append(0.0)
                continue
            ans_ids = le_h[b][ans_ok[b]]                  # answers are ENTITY ids (a list: :266-271), as are candidates
            n_ans = len(ans_ids)
            correct = int(np.isin(le_h[b][idx_h[b, :c]], ans_ids).sum()) if c else 0
            if n_ans == 0:
                vals.append(1.0 if c == 0 else 0.0)
            elif c == 0 or correct == 0:
                vals.append(0.0)
            else:
                p, r = correct / c, correct / n_ans
                vals.append(2.0 / (1.0 / p + 1.0 / r))
        f1 = torch.tensor(vals, dtype=torch.float32, device=pred_dist.device)
    return h1, f1


def _stage(model, batch):
    """(local_entity, query_entities, facts, q_input, seed_dist, answer_dist) on the model's device."""
    dev = model.word_embedding.weight.device
    _require_cuda(dev)
    if isinstance(batch, LiveBatch):
        db = batch.db
        return db.local_entity, db.query_entities, batch.facts, db.q_input, db.seed_dist, db.answer_dist
    local_entity, query_entities, kb_adj_mat, q_input, seed_dist, _tb, answer_dist = batch[:7]

    def t(x, dtype):
        x = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x))
        return x.to(device=dev, dtype=dtype)
    facts = _Facts(kb_adj_mat, dev, model.normalized_gnn, model.norm_rel)
    return (t(local_entity, torch.int64), t(query_entities, torch.float32), facts, t(q_input, torch.int64),
            t(seed_dist, torch.float32), t(answer_dist, torch.float32))


def _tp_list(model, pred_dist, staged):
    local_entity, _qe, _facts, _qi, seed_dist, answer_dist = staged
    h1, f1 = eval_metric(model, pred_dist.detach(), answer_dist, seed_dist, local_entity)
    return [h1.tolist(), f1.tolist()]


def rearev_forward(model, batch):
    """ReaRev forward with autograd (rearev.py:163-243) -> (loss, pred, pred_dist, [h1, f1])."""
    staged = _stage(model, batch)
    loss, pred, pred_dist = rearev_core(model, batch, staged)
    return loss, pred, pred_dist, _tp_list(model, pred_dist, staged)


def rearev_core(model, batch, staged):
    """The differentiable part of :func:`rearev_forward` over the inputs of :func:`_stage` -> (loss, pred, pred_dist)."""
    local_entity, query_entities, facts, q_input, seed_dist, answer_dist = staged
    B, N = local_entity.shape
    Nt, D, I = B * N, model.entity_dim, model.num_ins
    layer = model.reasoning
    rel_f, rel_f_inv = model.get_rel_feature_train()
    graph = _type_layer_graph(model, batch, local_entity.device, D)
    if model.encode_type:
        h = _type_layer(model.type_layer, facts, rel_f, Nt, graph)
    else:
        h = model.entity_linear(model.entity_embedding(local_entity)).view(Nt, D)
    instructions = _instructions(model.instruction, q_input)           # [B, I, D]
    ins_list = [instructions[:, j] for j in range(I)]
    mask = (local_entity != model.num_entity).float()
    drop = layer.linear_drop_train
    tables = []
    for k in range(model.num_gnn):
        lin = getattr(layer, "rel_linear" + str(k))
        tf, ti = lin(rel_f), lin(rel_f_inv)
        if layer.use_posemb:
            pe, pei = getattr(layer, "pos_emb" + str(k)).weight, getattr(layer, "pos_emb_inv" + str(k)).weight
            tf = torch.cat([tf[: pe.shape[0]] + pe, tf[pe.shape[0]:]])
            ti = torch.cat([ti[: pei.shape[0]] + pei, ti[pei.shape[0]:]])
        tables.append((tf, ti))
    dist_history = [seed_dist]
    dist = seed_dist
    graph = _kernel_graph(model, batch, h.device, D, I, graph)
    reform_kernels = _reform_kernels(h.device, D, I)
    fusion_w = [w for j in range(I) for w in (getattr(model, "reform" + str(j)).fusion.r.weight,
                                               getattr(model, "reform" + str(j)).fusion.g.weight)]
    for _t in range(model.num_iter):
        dist = seed_dist
        ins = torch.stack(ins_list, dim=1)                                  # [B, I, D]
        for k in range(model.num_gnn):
            tf, ti = tables[k]
            nb = _neighbours(tf, ti, ins, dist, facts, graph, Nt)           # [Nt, I, 2, D]: (j, direction) as in :150-156
            h = F.relu(getattr(layer, "e2e_linear" + str(k))(drop(torch.cat([h, nb.reshape(Nt, -1)], dim=1))))
            score = layer.score_func(drop(h)).view(B, N) + (1 - mask) * VERY_NEG_NUMBER
            dist = F.softmax(score, dim=1)
        dist_history.append(dist)
        if reform_kernels:                                                # one seed retrieve for all I reforms
            new = _QueryReformFn.apply(query_entities, h, torch.stack(ins_list, dim=1), B, N, *fusion_w)
            ins_list = [new[:, j] for j in range(I)]
            continue
        hB = h.view(B, N, D)
        new = []
        for j in range(I):
            reform = getattr(model, "reform" + str(j))
            seed_retrieve = torch.bmm(query_entities.unsqueeze(1), hB).squeeze(1)
            new.append(reform.fusion(ins_list[j], seed_retrieve))
        ins_list = new
    pred_dist = dist_history[-1]
    loss = _loss(model, pred_dist, answer_dist)
    pred = torch.max(pred_dist, dim=1)[1]
    model.dist_history = dist_history
    return loss, pred, pred_dist


def nsm_forward(model, batch):
    """NSM forward with autograd (nsm.py:179-254, forward reasoning only)."""
    staged = _stage(model, batch)
    loss, pred, pred_dist = nsm_core(model, batch, staged)
    return loss, pred, pred_dist, _tp_list(model, pred_dist, staged)


def nsm_core(model, batch, staged):
    """The differentiable part of :func:`nsm_forward` over the inputs of :func:`_stage` -> (loss, pred, pred_dist)."""
    local_entity, _qe, facts, q_input, seed_dist, answer_dist = staged
    B, N = local_entity.shape
    Nt, D = B * N, model.entity_dim
    layer = model.reasoning
    rel_f = model.get_rel_feature_train()
    graph = _type_layer_graph(model, batch, local_entity.device, D)
    if model.encode_type:
        h = _type_layer(model.type_layer, facts, rel_f, Nt, graph)
    else:
        h = model.entity_linear(model.entity_embedding(local_entity)).view(Nt, D)
    instructions = _instructions(model.instruction, q_input)
    mask = (local_entity != model.num_entity).float()
    drop = layer.linear_drop_train
    dist = seed_dist
    dist_history = [dist]
    graph = _kernel_graph(model, batch, h.device, D, 1, graph)
    for k in range(model.num_step):
        table = getattr(layer, "rel_linear" + str(k))(rel_f)
        pf = dist.reshape(-1)
        nb = _neighbours(table, None, instructions[:, k:k + 1], dist, facts, graph, Nt).reshape(Nt, D)
        h = F.relu(getattr(layer, "e2e_linear" + str(k))(drop(torch.cat([h, nb], dim=1))))
        m = mask
        if layer.reason_kb:                                                # nsm_gnn.py:98-101
            prior = pf[facts.heads]
            if facts.w is not None:
                prior = prior * facts.w * facts.w
            if facts.live is not None:                                     # padding slots of a LiveBatch
                prior = torch.where(facts.live, prior, 0.0)
            possible = torch.zeros(Nt, device=h.device).index_add_(0, facts.tails, prior)
            m = mask * (possible > 1e-10).float().view(B, N)
        score = layer.score_func(drop(h)).view(B, N) + (1 - m) * VERY_NEG_NUMBER
        dist = F.softmax(score, dim=1)
        dist_history.append(dist)
    pred_dist = dist_history[-1]
    loss = _loss(model, pred_dist, answer_dist)
    pred = torch.max(pred_dist, dim=1)[1]
    model.dist_history = dist_history
    return loss, pred, pred_dist


def _graft_facts(graft, kb_fact_rel, B, N, dev):
    """kb_adj_mat_graft -> (slot, head, tail) index vectors ordered by slot b*max_fact + f (build_adj_facts,
    base_gnn.py:56-75: the head list (b, f, head) and the tail list (b, tail, f) paired by slot)."""
    (e2f_b, e2f_f, e2f_e, _v0), (f2e_b, f2e_e, f2e_f, _v1) = graft

    def idx(a):
        if isinstance(a, torch.Tensor):
            return a.to(device=dev, dtype=torch.int64)
        return torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.int64))).to(dev)
    M = kb_fact_rel.shape[1]
    kh, kt = idx(e2f_b) * M + idx(e2f_f), idx(f2e_b) * M + idx(f2e_f)
    oh, ot = torch.argsort(kh), torch.argsort(kt)
    slot = kh[oh]
    if not torch.equal(slot, kt[ot]):
        raise ValueError("kb_adj_mat_graft: the head and tail lists do not hold the same fact slots")
    return slot, (idx(e2f_b) * N + idx(e2f_e))[oh], (idx(f2e_b) * N + idx(f2e_e))[ot]


class _GraftAttentionFn(torch.autograd.Function):
    """W [B, max_fact] of compute_attention (graft_gnn.py:64-87) for every slot: forward = gr_graft_attention,
    backward = gr_graft_attention_backward (csrc/graft.cu), which recomputes the per-slot softmax."""

    @staticmethod
    def forward(ctx, qh, rel, qmask, gg):
        ctx.dtypes = (qh.dtype, rel.dtype)
        qh, rel, qmask = qh.detach().float(), rel.detach().float().contiguous(), qmask.float()
        W, _wt, _e = ops.graft_attention(gg, qh, qmask, rel, out_w=True)
        ctx.save_for_backward(qh, rel, qmask)
        ctx.gg = gg
        ctx.det = torch.are_deterministic_algorithms_enabled()
        return W.view(gg.B, gg.max_fact)

    @staticmethod
    def backward(ctx, grad_W):
        qh, rel, qmask = ctx.saved_tensors
        gq = torch.zeros(qh.shape, dtype=torch.float32, device=qh.device)
        gr = torch.zeros(rel.shape, dtype=torch.float32, device=rel.device)
        ops.graft_attention_backward(ctx.gg, qh, qmask, rel.contiguous(), grad_W.float().reshape(-1), gq, gr,
                                     deterministic=ctx.det)
        return gq.to(ctx.dtypes[0]), gr.to(ctx.dtypes[1]), None, None


class _GraftAggregateFn(torch.autograd.Function):
    """sum_out[n] = sum_{f -> n} drop_f(relu(self_tab[r_f] + head_tab[head_f])) * s_f over the staged graft facts
    (graft_gnn.py:103-107 before kb_tail_linear): forward = gr_graft_aggregate_train, backward =
    gr_graft_aggregate_backward.  The dropout mask is recomputed from the saved seed, never stored.  Under bf16
    autocast head_tab, sum_out and their gradients are bf16 (self_tab and s fp32)."""

    @staticmethod
    def forward(ctx, self_tab, head_tab, s, gg, seed, p):
        ctx.dtypes = (self_tab.dtype, head_tab.dtype, s.dtype)
        self_tab, s = self_tab.detach().float().contiguous(), s.detach().float()
        head_tab = head_tab.detach().to(_node_dtype()).contiguous()
        out = ops.graft_aggregate_train(gg, s, self_tab, head_tab, seed, p)
        ctx.save_for_backward(self_tab, head_tab, s, seed)
        ctx.gg, ctx.p = gg, p
        ctx.det = torch.are_deterministic_algorithms_enabled()
        return out

    @staticmethod
    def backward(ctx, grad_out):
        self_tab, head_tab, s, seed = ctx.saved_tensors
        if grad_out.dtype != head_tab.dtype:     # widening is exact: same gradients as with grad_out in head_tab's dtype
            head_tab, grad_out = head_tab.float(), grad_out.float()
        gs = torch.zeros(s.shape, dtype=torch.float32, device=s.device)
        gself = torch.zeros(self_tab.shape, dtype=torch.float32, device=s.device)
        ghead = torch.zeros(head_tab.shape, dtype=head_tab.dtype, device=s.device)
        ops.graft_aggregate_backward(ctx.gg, s, self_tab, head_tab, grad_out.contiguous(), gs, gself, ghead, seed,
                                     ctx.p, deterministic=ctx.det)
        return (*(g.to(dt) for g, dt in zip((gself, ghead, gs), ctx.dtypes)), None, None, None)


def _graft_kernel_batch(model, batch, dev):
    """Stage a graft batch for the kernel path (slot order, both graft CSRs, the kb CSRs with the norm_rel weights);
    raises on malformed graft or kb fact lists with the messages of model(batch)."""
    from . import batching
    db = batching.stage_graft_batch(batch, dev, model.num_relation + 1, False, model.norm_rel)
    db.graft.check_status()
    db.graph.check_status()
    return db


def graft_live_stage(db):
    """The inputs of :func:`graftnet_core` for a graft batch staged from fixed-capacity buffers
    (graphed.GraphedGraftTrainStep): the (slot, head, tail) index vectors over the whole capacity of ``db.graft``,
    with its first ``nfacts`` entries live.  ``GraftGraph``'s buffers are written only in their live front, so each
    padding entry is replaced by a spare index before anything gathers through it: slot B*max_fact and node B*N, one
    past the end.  The core gathers 0 there and drops what is summed there, so a padding entry contributes nothing
    and shares no sum with a live one: torch's deterministic index_add groups the terms of one row, and how it adds
    them up depends on how many there are."""
    gg = db.graft
    live = torch.arange(gg.cap, device=gg.nfacts.device) < gg.nfacts
    Nt = db.B * db.N
    facts = tuple(torch.where(live, a[: gg.cap].long(), spare)
                  for a, spare in ((gg.slot_of, gg.B * gg.max_fact), (gg.heads, Nt), (gg.tails, Nt)))
    return db.local_entity, db.q_input, db.seed_dist, db.answer_dist, gg.kb_fact_rel, db, facts


def _stage_graft(model, batch):
    """(local_entity, q_input, seed_dist, answer_dist, kb_fact_rel, db, None) of a ``get_batch`` tuple on the model's
    device; ``db`` is the staged graft batch of the kernel path (None otherwise), whose malformed fact lists raise."""
    (local_entity, _qe, _kb, _graft, q_input, kb_fact_rel, seed_dist, _tb, answer_dist) = batch[:9]
    dev = model.word_embedding.weight.device
    _require_cuda(dev)

    def t(x, dtype):
        x = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x))
        return x.to(device=dev, dtype=dtype)
    local_entity, q_input = t(local_entity, torch.int64), t(q_input, torch.int64)
    seed_dist, answer_dist = t(seed_dist, torch.float32), t(answer_dist, torch.float32)
    kb_fact_rel = t(kb_fact_rel, torch.int64)
    db = _graft_kernel_batch(model, batch, dev) if _fact_kernels(dev, model.entity_dim) else None
    return local_entity, q_input, seed_dist, answer_dist, kb_fact_rel, db, None


def graftnet_forward(model, batch):
    """GraftNet forward with autograd (graftnet.py:135-183, graft_gnn.py:64-153) -> (loss, pred, pred_dist, [h1, f1]).

    Kernel path (CUDA, ``USE_KERNELS``, ``ops.fact_train_ok(D)``): the fact attention, the fact messages and the TypeLayer run in the kernels of
    csrc/graft.cu and csrc/aggregate*.cu with their own backward (_GraftAttentionFn, _GraftAggregateFn, _TypeLayerFn),
    so nothing of shape [facts, D] is formed or saved; kb_tail_linear is applied after the per-node sum (by linearity:
    sum_f kb_tail(v_f) = kb_tail.weight @ sum_f v_f + indeg * kb_tail.bias).  The per-fact scalars (W~, E, s, d') stay
    in torch autograd on [F] vectors.  The fact-message dropout is drawn in the kernels (Philox keyed by fact slot, one
    seed per layer from torch's CUDA generator).
    Otherwise (CPU under ``HOST_CHECK``, or ``USE_KERNELS`` off): per-fact messages are gathered and reduced with
    ``index_add_``; dropout sits where the reference applies it."""
    staged = _stage_graft(model, batch)
    loss, pred, pred_dist = graftnet_core(model, batch, staged)
    local_entity, _qi, seed_dist, answer_dist = staged[:4]
    h1, f1 = eval_metric(model, pred_dist.detach(), answer_dist, seed_dist, local_entity)
    return loss, pred, pred_dist, [h1.tolist(), f1.tolist()]


def graftnet_core(model, batch, staged):
    """The differentiable part of :func:`graftnet_forward` -> (loss, pred, pred_dist).  ``staged``: the inputs of
    :func:`_stage_graft` (the live graft fact count is then read on the host and the per-fact vectors have that length)
    or of :func:`graft_live_stage` (capacity-length vectors whose padding entries hold the spare indices)."""
    (_le, _qe, kb_adj_mat, graft) = batch[:4]
    local_entity, q_input, seed_dist, answer_dist, kb_fact_rel, db, live_facts = staged
    dev = local_entity.device
    B, N = local_entity.shape
    Nt, D = B * N, model.entity_dim
    layer = model.reasoning
    drop = layer.linear_drop_train
    kernels = db is not None
    spare = live_facts is not None

    def pad(v):               # v and, past its end, the 0 the spare index gathers
        return F.pad(v, (0, 1)) if spare else v

    def node_sums(idx, v):    # per-node sums; the spare row's is dropped
        if spare:
            return torch.zeros(Nt + 1, device=dev).index_add(0, idx, v)[:Nt]
        return torch.zeros(Nt, device=dev).index_add(0, idx, v)
    rel = model.get_rel_feature_train()
    if model.encode_type and kernels:
        h = _type_layer(model.type_layer, None, rel, Nt, db.graph)
    elif model.encode_type:
        h = _type_layer(model.type_layer, _Facts(kb_adj_mat, dev, False, model.norm_rel), rel, Nt)
    else:
        h = model.entity_linear(model.entity_embedding(local_entity)).view(Nt, D)
    enc = model.instruction
    enc.encode_question_train(q_input)
    qh, qnode, qmask = enc.query_hidden_emb, enc.query_node_emb, enc.query_mask_train
    if kernels:
        gg = db.graft
        if spare:
            slot, head, tail = live_facts
        else:
            nf = int(gg.nfacts.item())
            slot, head, tail = (t[:nf].long() for t in (gg.slot_of, gg.heads, gg.tails))
        W = _GraftAttentionFn.apply(qh, rel, qmask.float(), gg)                  # [B, max_fact]
    else:
        slot, head, tail = _graft_facts(graft, kb_fact_rel, B, N, dev)
        # compute_attention (graft_gnn.py:64-87) over every slot
        fact_emb = rel[kb_fact_rel]                                               # [B, max_fact, D]
        div = float(np.sqrt(D))
        sim = torch.bmm(qh, fact_emb.transpose(1, 2)) / div
        sim = F.softmax(sim + (1 - qmask.unsqueeze(2)) * VERY_NEG_NUMBER, dim=1)  # [B, Q, max_fact]
        W = torch.sum(torch.bmm(sim.transpose(1, 2), qh) * fact_emb, dim=2) / div
    W_tilde = pad(torch.exp(W - torch.max(W, dim=1, keepdim=True)[0]).reshape(-1))[slot]
    E = torch.clamp(node_sums(head, W_tilde), min=1e-10)
    mask = (local_entity != model.num_entity).float()
    d = seed_dist.reshape(-1)
    query = qnode                                                                 # [B, 1, D]
    dist_history, pagerank = [seed_dist], [seed_dist]
    lam = layer.pagerank_lambda
    if kernels:
        indeg = node_sums(tail, torch.ones_like(W_tilde)).unsqueeze(1)
    else:
        fact_rel = kb_fact_rel.reshape(-1)[slot]
    for i in range(model.num_layer):
        q2e = layer.lin("q2e_linear", i)(drop(query)).expand(B, N, D).reshape(Nt, D)
        s = W_tilde * pad(d / E)[head]
        if kernels:
            kt = layer.lin("kb_tail_linear", i)
            p = float(drop.p) if drop.training else 0.0
            seed = torch.randint(0, 2 ** 62, (1,), dtype=torch.int64, device=dev) if p > 0.0 else None
            sum_v = _GraftAggregateFn.apply(layer.lin("kb_self_linear", i)(rel),
                                            layer.lin("kb_head_linear", i)(drop(h)), s, gg, seed, p)
            f2e = F.relu(layer.lin("kb_self_linear", i)(h) + F.linear(sum_v, kt.weight) + indeg * kt.bias)
        else:
            v = F.relu(layer.lin("kb_self_linear", i)(rel)[fact_rel] + layer.lin("kb_head_linear", i)(drop(h))[head])
            v = v * s.unsqueeze(1)
            f2e = F.relu(layer.lin("kb_self_linear", i)(h) + torch.zeros(Nt, D, device=dev).index_add(
                0, tail, layer.lin("kb_tail_linear", i)(drop(v)).float()))
        d = lam * node_sums(tail, s) + (1 - lam) * d
        x = torch.cat([h, q2e, layer.fact_scale * f2e], dim=1)
        query = torch.bmm(d.view(B, 1, N), layer.lin("e2q_linear", i)(drop(x)).view(B, N, D))
        h = F.relu(layer.lin("e2e_linear", i)(drop(x)))
        logit = layer.score_func(drop(h)).view(B, N)
        dist_history.append(F.softmax(logit + (1 - mask) * VERY_NEG_NUMBER, dim=1))
        pagerank.append(d.view(B, N))
    pred_dist = dist_history[-1]
    case_valid = (torch.sum(answer_dist, dim=1, keepdim=True) > 0).float()
    loss = model.calc_loss_label(logit, answer_dist, case_valid)
    pred = torch.max(pred_dist, dim=1)[1]
    model.dist_history, model.pagerank_history = dist_history, pagerank
    return loss, pred, pred_dist
